"""The power-of-two operand scaling of the 3xFP16 split (DESIGN.md section 2.1) across magnitudes, and non-finite
values through it.

Every tensor-core activation and gradient is multiplied by its own power of two s before the fp16 split, s derived
from a (max|x|, 1/s) scale pair that the producing kernel or tc_amax fills.  The parity tests feed tensors of similar
magnitude and compare normwise, so a pair that is shared, stale or never reset, a max|x| over part of a tensor, or an
operand split with s = 1 stays within ~2x of the right scale and passes them.  This file checks what such bugs break:
 1. homogeneity: scaling an input (or the incoming gradient) by 2^k changes only the exponent, the scale pair takes
    it back out exactly, so every linear map below returns BITWISE 2^k times its unscaled result;
 2. history independence: calls whose operands differ by 2^60 in size, interleaved on one context, give the bits the
    same call gives on a fresh context;
 3. range against float64: per-sample spreads of 1 .. 2^-24 (a saturated D's gradients) and single outliers 2^16
    above the rest, judged per sample / per channel block, not only tensor-wide;
 4. non-finite values: a NaN or Inf in an activation, a gradient or a weight makes exactly its receptive field
    non-finite (as on the fp32 path and in float64) and leaves every other output's bits alone.
Each check runs with the default options (mma_f16 = 1) and with mma_f16 = 0 (3xTF32: no scaling, the same claims hold).

Bars: KTOL = 1e-5 per sample / per block for one launch against float64 on identical inputs, the tensor-wide launch
bar of tests/test_gpu_headline.py.  The split represents an element to 2^-22 of itself down to 2^-29 of its tensor's
max|x| (section 2.1), so a sample 2^-24 below the largest keeps the full-tensor accuracy.  DTOL = 2e-5 per sample for
a whole D backward's input gradient; TOL = 1e-4 per parameter tensor for whole-net gradients (the existing bar).

Deliberate bugs each of which turns tests here red (mma_f16 = 1 cases):
 - G's scale pairs not reset in the G backward: test_history_independence;
 - amax_kernel skipping its last vector: test_lop_conv_single_outlier;
 - the BatchNorm backward's max|dz| over the first half of the channels only: test_G_gradient_with_one_dominant_channel
   (last channel);
 - D's pooled activations' (d_act_pool_fwd) or gradients' (d_act_pool_bwd) max|x| over the first half of the channels
   only: test_D_gradient_with_one_dominant_channel (last channel, fwd / bwd);
 - no scale pair for the L-op dgrad operand: test_lop_conv_per_sample_range;
 - the FP16 split clamping NaN / Inf to +-65504, and max|x| dropping NaN / taking Inf: the non-finite tests.
A TcOp's amax_ready left set after tc_op_split turns nothing red: every consumer that reads it runs after the producer
that sets it, in the same pass, so a flag left set is overwritten before it is read.
"""
import numpy as np
import pytest

import c2f_utils as CU
import parity_utils as PU
import s16_utils as SU
from oracle import oracle as O
from oracle import oracle_c2f as OC
from oracle import oracle_s16 as OS
from test_gpu_headline import dev, rel

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = torch.nn.functional
TOL = 1e-4   # whole net
KTOL = 1e-5  # one launch against fp64 on identical inputs (measured worst per sample / per block: see each test)
DTOL = 2e-5  # a whole D backward's input gradient, per sample: each of its launches holds KTOL per sample (section 2.1)
C = 3
F16 = [1, 0]


def f32(a):
    return np.ascontiguousarray(a, np.float32)


def same_bits(got, want, what):
    """bitwise equality (signed zeros equal); the message names the worst element"""
    got, want = np.asarray(got), np.asarray(want)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if bad.any():
        i = int(np.flatnonzero(bad.ravel())[0])
        d = np.abs(got.astype(np.float64) - want).ravel()
        pytest.fail("%s: %d of %d elements differ (first at %d: %r vs %r; max |diff| %.3e, max |want| %.3e)" % (
            what, int(bad.sum()), bad.size, i, got.ravel()[i], want.ravel()[i], np.nanmax(d), np.nanmax(np.abs(want))))


def scaled(a, k):
    return f32(np.asarray(a, np.float32) * np.float32(2.0 ** k))


def _context(B, f16, **opts):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_option("mma_f16", f16)
    for key, v in opts.items():
        ctx.set_option(key, v)
    return ctx


# ================================================================================================ L-op convolutions
class Lop:
    """fg_conv2d_* / fg_scu_* on one context, NCHW numpy in and out (factor 1 = fg_conv2d_*)"""

    def __init__(self, ctx, factor=1):
        from face_generator_b200.lib import _ptr
        self.lib, self.h, self.p, self.f = ctx.lib, ctx.h, _ptr, factor

    def _ok(self, rc):
        assert rc == 0, self.lib.fg_last_error()

    def _geom(self, x_shape, w):
        N, Cin, H, W = x_shape
        return N, Cin, H, W, w.shape[0] // (self.f * self.f), w.shape[2]

    def fwd(self, x, w, b=None):
        N, Cin, H, W, nout, k = self._geom(x.shape, w)
        y = np.empty((N, w.shape[0], H, W), np.float32)
        p = self.p
        if self.f == 1:
            self._ok(self.lib.fg_conv2d_forward(self.h, p(x), p(w), p(b), p(y), N, Cin, H, W, nout, k))
        else:
            self._ok(self.lib.fg_scu_forward(self.h, p(x), p(w), p(b), p(y), N, Cin, H, W, nout, k, self.f))
        return y

    def dgrad(self, dy, w, Cin):
        N, _, H, W = dy.shape
        _, _, _, _, nout, k = self._geom((N, Cin, H, W), w)
        dx = np.empty((N, Cin, H, W), np.float32)
        p = self.p
        if self.f == 1:
            self._ok(self.lib.fg_conv2d_backward_data(self.h, p(dy), p(w), p(dx), N, Cin, H, W, nout, k))
        else:
            self._ok(self.lib.fg_scu_backward_data(self.h, p(dy), p(w), p(dx), N, Cin, H, W, nout, k, self.f))
        return dx

    def wgrad(self, x, dy, w_shape):
        N, Cin, H, W = x.shape
        nout, k = w_shape[0] // (self.f * self.f), w_shape[2]
        dw, db = np.zeros(w_shape, np.float32), np.zeros(w_shape[0], np.float32)
        p = self.p
        if self.f == 1:
            self._ok(self.lib.fg_conv2d_backward_filter(self.h, p(x), p(dy), p(dw), p(db), N, Cin, H, W, nout, k))
        else:
            self._ok(self.lib.fg_scu_backward_filter(self.h, p(x), p(dy), p(dw), p(db), N, Cin, H, W, nout, k, self.f))
        return dw, db


def lop_case(N, Cin, H, Cout, k, seed):
    rng = np.random.default_rng(seed)
    x = f32(rng.standard_normal((N, Cin, H, H)))
    w = f32(rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k))
    return x, w, f32(rng.standard_normal(Cout)), f32(rng.standard_normal((N, Cout, H, H)))


# the shapes of test_gpu_parity.test_tc_conv_lop and the D.C2-C4 launches at batch 256 and 130
LOP_SHAPES = [(8, 64, 16, 128, 3), (3, 128, 8, 256, 3), (5, 256, 4, 512, 3), (2, 32, 32, 64, 5), (3, 64, 16, 128, 7),
              (1, 128, 32, 128, 1), (256, 64, 16, 128, 3), (256, 128, 8, 256, 3), (256, 256, 4, 512, 3),
              (130, 64, 16, 128, 3), (130, 128, 8, 256, 3), (130, 256, 4, 512, 3)]


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("N,Cin,H,Cout,k", LOP_SHAPES)
def test_lop_conv_is_exactly_homogeneous(N, Cin, H, Cout, k, f16):
    """(2^k x, w, 2^k b) -> 2^k y; 2^k dy -> 2^k dx, 2^k dw, 2^k db; 2^k x -> 2^k dw, all bitwise"""
    x, w, b, dy = lop_case(N, Cin, H, Cout, k, 500 + N + Cin + k)
    ctx = _context(8, f16, conv_impl=2)
    op = Lop(ctx)
    y, dx, (dw, db) = op.fwd(x, w, b), op.dgrad(dy, w, Cin), op.wgrad(x, dy, w.shape)
    for e in (-48, -24, 24, 48):
        t = np.float32(2.0 ** e)
        same_bits(op.fwd(scaled(x, e), w, scaled(b, e)), t * y, "forward 2^%d" % e)
        same_bits(op.dgrad(scaled(dy, e), w, Cin), t * dx, "dgrad 2^%d" % e)
        dwe, dbe = op.wgrad(x, scaled(dy, e), w.shape)
        same_bits(dwe, t * dw, "wgrad dy 2^%d" % e)
        same_bits(dbe, t * db, "bias grad dy 2^%d" % e)
        same_bits(op.wgrad(scaled(x, e), dy, w.shape)[0], t * dw, "wgrad x 2^%d" % e)
    ctx.close()


@pytest.mark.parametrize("f16", F16)
def test_scu_is_exactly_homogeneous(f16):
    """fg_scu_* (SpatialConvolutionUpsample, factor 2): the same convolution on nOut*4 planes"""
    N, Cin, H, nout, k = 130, 64, 8, 32, 3
    x, w, b, dy = lop_case(N, Cin, H, nout * 4, k, 77)
    ctx = _context(8, f16, conv_impl=2)
    op = Lop(ctx, factor=2)
    y, dx, (dw, db) = op.fwd(x, w, b), op.dgrad(dy, w, Cin), op.wgrad(x, dy, w.shape)
    xt, wt = dev(x), dev(w)
    assert rel(y, F.conv2d(xt, wt, dev(b), padding=1)) < KTOL
    for e in (-24, 24):
        t = np.float32(2.0 ** e)
        same_bits(op.fwd(scaled(x, e), w, scaled(b, e)), t * y, "scu forward 2^%d" % e)
        same_bits(op.dgrad(scaled(dy, e), w, Cin), t * dx, "scu dgrad 2^%d" % e)
        dwe, dbe = op.wgrad(x, scaled(dy, e), w.shape)
        same_bits(dwe, t * dw, "scu wgrad 2^%d" % e)
        same_bits(dbe, t * db, "scu bias grad 2^%d" % e)
    ctx.close()


def per_block_err(got, ref, axes):
    """normwise relative error of every block (max over `axes`), as a float64 numpy array"""
    d = (dev(got) - ref).abs().amax(dim=axes)
    return (d / (ref.abs().amax(dim=axes) + 1e-300)).cpu().numpy()


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("N,Cin,H,Cout", [(256, 64, 16, 128), (130, 128, 8, 256), (130, 256, 4, 512)])
def test_lop_conv_per_sample_range(N, Cin, H, Cout, f16):
    """samples of x and dy scaled from 1 down to 2^-24 (the saturated-D regime: logits above ~17 send back gradients
    of ~1e-8): forward and dgrad per sample, wgrad with dy's output channels spread the same way per (co, ci) block,
    all against float64 at KTOL.  A tensor split unscaled (s = 1) loses such samples to fp16 subnormals."""
    x, w, _, dy = lop_case(N, Cin, H, Cout, 3, 900 + N + Cin)
    spread = lambda n: (2.0 ** (-24.0 * np.arange(n) / (n - 1))).astype(np.float32)
    xs, dys = f32(x * spread(N)[:, None, None, None]), f32(dy * spread(N)[:, None, None, None])
    dyc = f32(dy * spread(Cout)[None, :, None, None])
    ctx = _context(8, f16, conv_impl=2)
    op = Lop(ctx)
    y, dx, (dw, _) = op.fwd(xs, w), op.dgrad(dys, w, Cin), op.wgrad(x, dyc, w.shape)
    ctx.close()
    xt, wt = dev(xs), dev(w)
    e_y = per_block_err(y, F.conv2d(xt, wt, padding=1), (1, 2, 3))
    e_dx = per_block_err(dx, torch.nn.grad.conv2d_input(xt.shape, wt, dev(dys), padding=1), (1, 2, 3))
    e_dw = per_block_err(dw, torch.nn.grad.conv2d_weight(dev(x), wt.shape, dev(dyc), padding=1), (2, 3))
    worst = dict(fwd=e_y.max(), dgrad=e_dx.max(), wgrad=e_dw.max())
    # measured on an H100 (80 GB HBM3, 700 W), worst over the shapes and both mma_f16: forward 1.6e-6, dgrad 1.6e-6
    # per sample, wgrad 3.3e-6 per (co, ci) block
    assert max(worst.values()) < KTOL, (worst, int(e_y.argmax()), int(e_dx.argmax()), np.unravel_index(e_dw.argmax(), e_dw.shape))


def outlier_positions(N, Cc, H):
    """flat NCHW indices: first element, last element, a middle pixel of the last sample, of the last channel"""
    at = lambda n, c, i, j: ((n * Cc + c) * H + i) * H + j
    return {"first": 0, "last": N * Cc * H * H - 1, "last_sample": at(N - 1, Cc // 3, H // 2, H // 3),
            "last_channel": at(N // 2, Cc - 1, H // 3, H // 2)}


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("N,Cin,H,Cout", [(130, 64, 16, 128), (130, 256, 4, 512)])
def test_lop_conv_single_outlier(N, Cin, H, Cout, f16):
    """one element 2^16 above the rest, in x (forward, wgrad) and in dy (dgrad, wgrad), at the first and last index,
    in the last sample of the batch tail and in the last channel: a max|x| that misses it clamps it to 65504 / s"""
    x, w, b, dy = lop_case(N, Cin, H, Cout, 3, 1300 + Cin)
    ctx = _context(8, f16, conv_impl=2)
    op = Lop(ctx)
    wt = dev(w)
    errs = {}
    for where, i in outlier_positions(N, Cin, H).items():
        xo = x.copy()
        xo.flat[i] = 65536.0 * (1.0 if i % 2 else -1.0)
        xt = dev(xo)
        errs["fwd " + where] = rel(op.fwd(xo, w, b), F.conv2d(xt, wt, dev(b), padding=1))
        errs["wgrad(x) " + where] = rel(op.wgrad(xo, dy, w.shape)[0], torch.nn.grad.conv2d_weight(xt, wt.shape, dev(dy), padding=1))
    for where, i in outlier_positions(N, Cout, H).items():
        dyo = dy.copy()
        dyo.flat[i] = 65536.0 * (1.0 if i % 2 else -1.0)
        dyt = dev(dyo)
        errs["dgrad " + where] = rel(op.dgrad(dyo, w, Cin), torch.nn.grad.conv2d_input(x.shape, wt, dyt, padding=1))
        dw, db = op.wgrad(x, dyo, w.shape)
        errs["wgrad(dy) " + where] = rel(dw, torch.nn.grad.conv2d_weight(dev(x), wt.shape, dyt, padding=1))
        errs["bias grad " + where] = rel(db, dyt.sum((0, 2, 3)))
    ctx.close()
    # measured on an H100 (80 GB HBM3, 700 W): worst 2.4e-6
    assert max(errs.values()) < KTOL, errs


def conv64(x, w):
    """the zero-padded "same" convolution in float64 as its definition: im2col (F.unfold, the padding as explicit
    zeros) times the weight matrix, so a non-finite element meets every weight and every padding zero it is
    multiplied with (0 * NaN = NaN, 0 * Inf = NaN)"""
    N, _, H, W = x.shape
    k = w.shape[2]
    return (w.reshape(w.shape[0], -1) @ F.unfold(x, k, padding=k // 2)).reshape(N, w.shape[0], H, W)


def dgrad64(dy, w):
    return conv64(dy, w.transpose(0, 1).flip(2, 3))


def wgrad64(x, dy, k):
    N, Cout = dy.shape[:2]
    cols = F.unfold(x, k, padding=k // 2)
    return torch.einsum("nol,nkl->ok", dy.reshape(N, Cout, -1), cols).reshape(Cout, x.shape[1], k, k)


def nonfinite64(t):
    return (~torch.isfinite(t)).cpu().numpy()


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("bad", [np.nan, np.inf])
@pytest.mark.parametrize("N,Cin,H,Cout", [(130, 64, 16, 128), (5, 256, 4, 512)])
def test_lop_conv_nonfinite(N, Cin, H, Cout, bad, f16):
    """one NaN / +Inf in x (forward, wgrad) and in dy (dgrad, wgrad): the non-finite outputs are exactly those of the
    same operation in float64 (conv64 and friends: the element's receptive field; for the weight gradient of a bad dy
    element, every tap of its channel, the taps past the image edge through 0 * NaN), and every other output is
    bitwise the run with that element set to 0"""
    x, w, b, dy = lop_case(N, Cin, H, Cout, 3, 1700 + Cin)
    ctx = _context(8, f16, conv_impl=2)
    op = Lop(ctx)
    wt = dev(w)

    def check(got, clean, expect, what):
        fin = np.isfinite(got)
        assert np.array_equal(~fin, expect), "%s: %d non-finite outputs, %d expected (%d of them in the set)" % (
            what, int((~fin).sum()), int(expect.sum()), int((~fin & expect).sum()))
        same_bits(got[fin], clean[fin], what + " (finite outputs)")

    i = ((N - 1) * Cin + 1) * H * H + 3 * H + H - 1  # last sample, channel 1, right edge
    xb = x.copy()
    xb.flat[i] = bad
    x0 = x.copy()
    x0.flat[i] = 0.0
    check(op.fwd(xb, w, b), op.fwd(x0, w, b), nonfinite64(conv64(dev(xb), wt) + dev(b).view(1, -1, 1, 1)), "forward, x")
    dwb, dbb = op.wgrad(xb, dy, w.shape)
    dw0, db0 = op.wgrad(x0, dy, w.shape)
    check(dwb, dw0, nonfinite64(wgrad64(dev(xb), dev(dy), 3)), "wgrad, x")
    same_bits(dbb, db0, "bias grad, x")

    j = (2 * Cout + 7) * H * H + H - 1  # sample 2, channel 7, top right corner
    dyb = dy.copy()
    dyb.flat[j] = bad
    dy0 = dy.copy()
    dy0.flat[j] = 0.0
    check(op.dgrad(dyb, w, Cin), op.dgrad(dy0, w, Cin), nonfinite64(dgrad64(dev(dyb), wt)), "dgrad, dy")
    dwb, dbb = op.wgrad(x, dyb, w.shape)
    dw0, db0 = op.wgrad(x, dy0, w.shape)
    check(dwb, dw0, nonfinite64(wgrad64(dev(x), dev(dyb), 3)), "wgrad, dy")
    check(dbb, db0, nonfinite64(dev(dyb).sum((0, 2, 3))), "bias grad, dy")
    ctx.close()


# ================================================================================================ the three net pairs
class Net:
    """one G/D pair behind a uniform interface: "32" (fg_*), "c2f" (fg_c2f_*), "s16" (fg_s16_*)"""

    def __init__(self, kind, B, f16, seed=0, init=None, ctx=None, **opts):
        """ctx: share that context (this pair's own scale-pair block on it) instead of creating one"""
        import face_generator_b200 as fg
        self.kind, self.B, self.own = kind, B, ctx is None
        self.ctx = _context(B, f16, **opts) if ctx is None else ctx
        if kind == "32":
            self.case = PU.make_case(2 * B, C, seed, init=init or "trained")
            self.net, self.side, self.GL, self.DL = self.ctx, 32, O.G_layout(C), O.D_layout(C)
        elif kind == "c2f":
            self.case = CU.make_case(2 * B, C, seed, init=init or "trained")
            self.net, self.side, self.GL, self.DL = fg.C2f(self.ctx), 32, OC.G_layout(C), OC.D_layout(C)
        else:
            self.case = SU.make_case(2 * B, C, seed, init=init or "near")
            self.net, self.side, self.GL, self.DL = fg.S16(self.ctx), 16, OS.G_layout(C), OS.D_layout(C)
        self.set_params()

    def set_params(self, PG=None, PD=None):
        from face_generator_b200.lib import NET_D, NET_G
        self.net.set_params(NET_G, self.case["PG"] if PG is None else PG)
        self.net.set_params(NET_D, self.case["PD"] if PD is None else PD)

    def close(self):
        if self.net is not self.ctx:
            self.net.close()
        if self.own:
            self.ctx.close()

    # ---- G ----
    def g_inputs(self):
        B = self.B
        if self.kind == "c2f":
            return [self.case["noise_G"][:B], self.case["cond_G"][:B]]
        return [self.case["noise_G"][:B]]

    def G_forward(self, ins):
        return self.net.G_forward(*ins)

    def G_backward(self, d):
        """G's gradients (and d_noise where the entry point returns it) of the last G forward"""
        from face_generator_b200.lib import NET_G
        self.net.zero_grads(NET_G)
        if self.kind == "c2f":
            self.net.G_backward(d)
            return [self.net.get_grads(NET_G)]
        dn = self.net.G_backward(d, want_dnoise=True)
        return [self.net.get_grads(NET_G), dn]

    # ---- D ----
    def d_inputs(self):
        B = self.B
        if self.kind == "c2f":
            return [f32(self.case["real_diff"][:B]), self.case["cond_D"][:B]]
        return [np.random.default_rng(B).random((B, C, self.side, self.side)).astype(np.float32)]

    def masks(self):
        return self.case["masks_D"][:self.B]

    def D_forward(self, ins):
        """D.logit (the pre-sigmoid output) of a training-mode forward with explicit dropout masks"""
        self.net.D_forward(*ins, masks=self.masks())
        return self.net.debug_tensor("D.logit")[:self.B].copy()

    def D_backward(self, d_out):
        from face_generator_b200.lib import NET_D
        self.net.zero_grads(NET_D)
        di = self.net.D_backward(d_out)
        return [self.net.get_grads(NET_D), di]


def bias_keys(layout):
    return [k for k in layout if k.endswith("b") and not k.startswith("be")]


def scale_biases(P, layout, e):
    P = P.copy()
    for k in bias_keys(layout):
        o, s = layout[k]
        P[o:o + int(np.prod(s))] *= np.float32(2.0 ** e)
    return P


NET_CONFIGS = {"32": [{}, {"conv_impl": 1}, {"bwd_merge": 0}, {"bwd_merge": 2}], "c2f": [{}, {"conv_impl": 1}],
               "s16": [{}, {"conv_impl": 1}]}
G_CASES = [(kind, B, f16, opts) for kind in ("32", "c2f", "s16") for B in (256, 130) for f16 in F16
           for opts in NET_CONFIGS[kind] if f16 == 1 or not opts]
G_IDS = ["%s-B%d-f16_%d%s" % (k, B, f, "".join("-%s_%d" % kv for kv in o.items())) for k, B, f, o in G_CASES]
D_CASES = [(kind, B, f16) for kind in ("32", "c2f", "s16") for B in (256, 130) for f16 in F16]
D_IDS = ["%s-B%d-f16_%d" % c for c in D_CASES]


@pytest.mark.parametrize("kind,B,f16,opts", G_CASES, ids=G_IDS)
def test_G_backward_is_exactly_homogeneous(kind, B, f16, opts):
    """G_backward(2^k d): G's gradients and d_noise are 2^k times those of G_backward(d), bitwise (one forward)"""
    n = Net(kind, B, f16, seed=5000 + B, **opts)
    n.G_forward(n.g_inputs())
    d = np.random.default_rng(B + 1).standard_normal((B, C, n.side, n.side)).astype(np.float32)
    base = n.G_backward(d)
    for e in (-24, 24):
        for i, (got, want) in enumerate(zip(n.G_backward(scaled(d, e)), base)):
            same_bits(got, np.float32(2.0 ** e) * want, "%s G backward output %d at 2^%d" % (kind, i, e))
    n.close()


@pytest.mark.parametrize("kind,B,f16,opts", G_CASES, ids=G_IDS)
def test_G_forward_is_exactly_homogeneous(kind, B, f16, opts):
    """inputs and every bias scaled by 2^k: c2f G's output (no BatchNorm) and the 32x32 / s16 G's first convolution
    output G.z1 (BatchNorm's eps breaks exactness after it) scale by 2^k, bitwise"""
    n = Net(kind, B, f16, seed=5100 + B, **opts)
    ins = n.g_inputs()

    def run(e):
        n.set_params(PG=scale_biases(n.case["PG"], n.GL, e))
        out = n.G_forward([scaled(a, e) for a in ins])
        return out if kind == "c2f" else n.net.debug_tensor("G.z1")

    base = run(0)
    for e in (-24, 24):
        same_bits(run(e), np.float32(2.0 ** e) * base, "%s G forward at 2^%d" % (kind, e))
    n.close()


@pytest.mark.parametrize("kind,B,f16", D_CASES, ids=D_IDS)
def test_D_is_exactly_homogeneous(kind, B, f16):
    """D_backward(2^k d_out): D's gradients and the input gradients scale by 2^k; D.logit with the inputs and every
    bias scaled by 2^k (PReLU, pooling and dropout are positively homogeneous) scales by 2^k; all bitwise"""
    n = Net(kind, B, f16, seed=5200 + B)
    ins = n.d_inputs()
    base_logit = n.D_forward(ins)
    d = np.random.default_rng(B + 2).standard_normal(B).astype(np.float32)
    base = n.D_backward(d)
    for e in (-24, 24):
        for i, (got, want) in enumerate(zip(n.D_backward(scaled(d, e)), base)):
            same_bits(got, np.float32(2.0 ** e) * want, "%s D backward output %d at 2^%d" % (kind, i, e))
    for e in (-24, 24):
        n.set_params(PD=scale_biases(n.case["PD"], n.DL, e))
        same_bits(n.D_forward([scaled(a, e) for a in ins]), np.float32(2.0 ** e) * base_logit, "%s D.logit at 2^%d" % (kind, e))
    n.close()


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("B", [256, 130])
@pytest.mark.parametrize("kind", ["32", "s16"])
def test_D_input_gradient_per_sample(kind, B, f16):
    """D_backward with d_out spanning 1 .. 1e-8 across the samples: d_images of every sample against float64 on its
    own scale ("smooth" init: PReLU slopes 1, no kink ambiguity)"""
    import torch_ref as R
    import torch_ref_s16 as RS
    n = Net(kind, B, f16, seed=5300 + B, init="smooth")
    img = n.d_inputs()[0]
    d_out = f32(np.random.default_rng(B + 3).choice([-1.0, 1.0], B) * np.logspace(0, -8, B))
    n.D_forward([img])
    di = n.D_backward(d_out)[1]
    n.close()
    P, x = dev(n.case["PD"]), dev(img).requires_grad_(True)
    ref = (R.D_forward if kind == "32" else RS.torch_D16)(P, x, dev(n.masks()), C)
    ref.backward(dev(d_out))
    err = per_block_err(di, x.grad, (1, 2, 3))
    # bar DTOL per sample; measured on an H100 (80 GB HBM3, 700 W): worst sample 4.1e-6
    assert err.max() < DTOL, (float(err.max()), int(err.argmax()))


DOM_CASES = [(kind, B, f16, w) for kind in ("32", "s16") for B in (256, 130) for f16 in F16 for w in ("first", "last")]
DOM_IDS = ["%s-B%d-f16_%d-%s" % c for c in DOM_CASES]


def whole_net_errs(got, ref, layout, skip=()):
    """per parameter tensor, normwise; a shared PReLU slope is one heavily cancelling sum and is held to 3 TOL as in
    the other whole-net tests, so it is reported here divided by 3"""
    errs = {}
    for k, (o, s) in layout.items():
        if k in skip:
            continue
        m = int(np.prod(s))
        errs[k] = PU.relerr(got[o:o + m], ref[o:o + m]) / (3 if k[0] == "a" else 1)
    return errs


@pytest.mark.parametrize("kind,B,f16,where", DOM_CASES, ids=DOM_IDS)
def test_G_gradient_with_one_dominant_channel(kind, B, f16, where):
    """In each BatchNorm, gamma of one channel (channel 1, or the last but one) multiplied by 2^10, so that dz1 and
    dz2 -- the BatchNorm backward's outputs, whose max|x| their producers reduce -- are each dominated by one channel.
    G.C3's weights of the BatchNorm-2 channel are divided by 2^6 so that the sigmoid output does not saturate (without
    it 84 % of the outputs have a derivative below 1e-6); dz2's channel still stands 2^4 above the others.  G's
    gradients and d_noise against float64 at the whole-net bar ("smooth" init: PReLU slopes 1, no kink ambiguity)."""
    import torch_ref as R
    import torch_ref_s16 as RS
    n = Net(kind, B, f16, seed=5600 + B, init="smooth")
    PG = n.case["PG"].copy()
    c1, c2 = (1, 1) if where == "first" else (254, 126)
    PG[n.GL["g1"][0] + c1] *= 1024.0
    PG[n.GL["g2"][0] + c2] *= 1024.0
    o, s = n.GL["C3W"]
    PG[o:o + int(np.prod(s))].reshape(s)[:, c2] *= 2.0 ** -6
    n.set_params(PG=PG)
    noise = n.g_inputs()[0]
    d = np.random.default_rng(B + 5).standard_normal((B, C, n.side, n.side)).astype(np.float32)
    n.G_forward([noise])
    gG, dn = n.G_backward(d)
    n.close()
    P, nz = dev(PG).requires_grad_(True), dev(noise).requires_grad_(True)
    out = R.G_forward(P, nz, C)[0] if kind == "32" else RS.torch_G16(P, nz, C)
    out.backward(dev(d))
    errs = whole_net_errs(gG, P.grad.cpu().numpy(), n.GL, skip=("C1b", "C2b"))  # those two: analytically zero
    errs["d_noise"] = rel(dn, nz.grad)
    # measured on an H100 (80 GB HBM3, 700 W): worst 1.8e-5 (be1), over both channel positions
    assert max(errs.values()) < TOL, errs


# D: (producer weight, producer bias, consumer weight, the consumer's input columns of producer channel c)
D_CHAINS = {
    "32": [("c1W", "c1b", "c2W", "conv"), ("c2W", "c2b", "c3W", "conv"), ("c3W", "c3b", "c4W", "conv"),
           ("c4W", "c4b", "L1W", "2x2"), ("L1W", "L1b", "L2W", 0), ("L2W", "L2b", "L3W", 0)],
    "s16": [("c1W", "c1b", "c2W", "conv"), ("c2W", "c2b", "c3W", "conv"), ("c3W", "c3b", "c4W", "conv"),
            ("c4W", "c4b", "F1W", "2x2"), ("F1W", "F1b", "JW", 0), ("E1W", "E1b", "E2W", 0), ("E2W", "E2b", "JW", 1024)]}


def dominant_D_factors(layout, count, chain, where, up):
    """per-parameter powers of two: one output channel of every layer scaled by 2^10 (up) or 2^-10, its input columns
    in the next layer by the inverse.  With D's parameters multiplied by them the logits stay O(1) while the forward
    activations (up) or the backward gradients (not up) of that channel stand 2^10 above the rest of their tensor."""
    P = np.ones(count, np.float32)
    view = lambda k: P[layout[k][0]:layout[k][0] + int(np.prod(layout[k][1]))].reshape(layout[k][1])
    f = np.float32(1024.0 if up else 1.0 / 1024.0)
    for wk, bk, nk, cols in chain:
        c = 1 if where == "first" else layout[bk][1][0] - 2
        view(wk)[c] *= f
        view(bk)[c] *= f
        nxt = view(nk)
        if cols == "conv":
            nxt[:, c] /= f
        elif cols == "2x2":  # the Linear after the last convolution reads (c, h, w)-ordered 2x2 maps
            nxt[:, 4 * c:4 * c + 4] /= f
        else:
            nxt[:, cols + c] /= f
    return P


DDOM_CASES = [(kind, B, f16, w, up) for kind in ("32", "s16") for B in (256, 130) for f16 in F16
              for w in ("first", "last") for up in ("fwd", "bwd")]


@pytest.mark.parametrize("kind,B,f16,where,up", DDOM_CASES, ids=["%s-B%d-f16_%d-%s-%s" % c for c in DDOM_CASES])
def test_D_gradient_with_one_dominant_channel(kind, B, f16, where, up):
    """every D layer with one output channel (channel 1, or the last but one) whose weights and bias are scaled by 2^10
    ("fwd": its activations dominate the tensor the next layer splits) or by 2^-10 ("bwd": its gradients dominate dz),
    the next layer's weights of that channel scaled inversely.  D's gradients and d_images against float64 at the
    whole-net bars ("smooth" init).  The gradients are compared in the units of the unscaled parameters (both sides
    multiplied by the same powers of two, chain rule): an entry of the next layer's weight gradient sums terms 2^10
    above its neighbours, and where those cancel (one case here: a sum of terms ~1e4 comes to 43) its fp32 rounding
    would otherwise be judged against the small neighbours."""
    import torch_ref as R
    import torch_ref_s16 as RS
    from face_generator_b200.lib import NET_D
    n = Net(kind, B, f16, seed=5700 + B, init="smooth")
    fac = dominant_D_factors(n.DL, n.net.count(NET_D), D_CHAINS[kind], where, up == "fwd")
    PD = n.case["PD"] * fac
    n.set_params(PD=PD)
    img = n.d_inputs()[0]
    d_out = np.random.default_rng(B + 7).standard_normal(B).astype(np.float32)
    n.D_forward([img])
    gD, di = n.D_backward(d_out)
    n.close()
    P, x = dev(PD).requires_grad_(True), dev(img).requires_grad_(True)
    ref = (R.D_forward if kind == "32" else RS.torch_D16)(P, x, dev(n.masks()), C)
    ref.backward(dev(d_out))
    errs = whole_net_errs(gD * fac, P.grad.cpu().numpy() * fac, n.DL)
    errs["d_images"] = rel(di, x.grad)
    # measured on an H100 (80 GB HBM3, 700 W): worst 3.2e-6 over weights, biases and d_images;
    # every tensor, the shared PReLU slopes included, below 1.8e-5
    assert max(errs.values()) < TOL, errs


NF_CASES = [(kind, B, f16, bad) for kind in ("32", "s16") for B in (256, 130) for f16 in F16 for bad in (np.nan, np.inf)]


@pytest.mark.parametrize("kind,B,f16,bad", NF_CASES, ids=["%s-B%d-f16_%d-%s" % c for c in NF_CASES])
def test_D_nonfinite_stays_in_its_sample(kind, B, f16, bad):
    """a NaN / +Inf in one pixel of sample i makes D.logit[i] non-finite and leaves every other logit's bits; a NaN in
    d_out[i] makes d_images[i] non-finite and leaves every other sample's input gradient's bits"""
    n = Net(kind, B, f16, seed=5400 + B)
    img = n.d_inputs()[0]
    clean = n.D_forward([img])
    i = B - 2
    bad_img = img.copy()
    bad_img[i, 1, n.side // 2, 3] = bad
    logit = n.D_forward([bad_img])
    assert not np.isfinite(logit[i]), logit[i]
    rest = np.arange(B) != i
    same_bits(logit[rest], clean[rest], "%s D.logit of the other samples" % kind)
    n.D_forward([img])
    d = np.random.default_rng(B + 4).standard_normal(B).astype(np.float32)
    di0 = n.D_backward(d)[1]
    d[i] = np.nan
    di = n.D_backward(d)[1]
    assert (~np.isfinite(di[i])).any(), "d_images of sample %d is finite" % i
    same_bits(di[rest], di0[rest], "%s d_images of the other samples" % kind)
    n.close()


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("B", [256, 130])
def test_D_nan_weight_reaches_the_output(B, f16):
    """a NaN in one D.C2 weight (set through set_params) makes every logit non-finite"""
    n = Net("32", B, f16, seed=5500 + B)
    o, _ = n.DL["c2W"]
    PD = n.case["PD"].copy()
    PD[o + 1234] = np.nan
    n.set_params(PD=PD)
    logit = n.D_forward(n.d_inputs())
    n.close()
    assert not np.isfinite(logit).any(), int(np.isfinite(logit).sum())


# ================================================================================================ history independence
def _history_ops(B, f16):
    """(name, fn(state) -> list of arrays) in call order; fn may scale its operands (the state: the nets, the L-op
    wrapper, the data).  The unscaled calls are the ones compared."""
    rng = np.random.default_rng(B + 6000)
    x, w, b, dy = lop_case(B, 64, 16, 128, 3, 6001)
    d32 = rng.standard_normal((B, C, 32, 32)).astype(np.float32)
    d16 = rng.standard_normal((B, C, 16, 16)).astype(np.float32)
    dout = rng.standard_normal(B).astype(np.float32)
    ops = []
    for e in (30, -30, 0):
        ops += [("lop fwd %d" % e, lambda s, e=e: [s["op"].fwd(scaled(x, e), w, scaled(b, e))]),
                ("lop dgrad %d" % e, lambda s, e=e: [s["op"].dgrad(scaled(dy, -e), w, 64)]),
                ("lop wgrad %d" % e, lambda s, e=e: list(s["op"].wgrad(scaled(x, -e), scaled(dy, e), w.shape)))]
        for kind, d in (("32", d32), ("c2f", d32), ("s16", d16)):
            ops += [("%s G backward %d" % (kind, e), lambda s, e=e, kind=kind, d=d: s[kind].G_backward(scaled(d, e))),
                    ("%s D backward %d" % (kind, e), lambda s, e=e, kind=kind: s[kind].D_backward(scaled(dout, -e)))]
        if e == 30:
            ops += [("mma_f16 toggled", lambda s: s["ctx"].set_option("mma_f16", 1 - f16) or []),
                    ("lop fwd toggled", lambda s: [s["op"].fwd(x, w, b)]),
                    ("mma_f16 back", lambda s: s["ctx"].set_option("mma_f16", f16) or [])]
    return ops


def _history_state(B, f16):
    """the three pairs on one context, each after one training-mode G and D forward"""
    n32 = Net("32", B, f16, seed=6100 + B)
    s = {"ctx": n32.ctx, "op": Lop(n32.ctx), "32": n32, "c2f": Net("c2f", B, f16, 6200 + B, ctx=n32.ctx),
         "s16": Net("s16", B, f16, 6300 + B, ctx=n32.ctx)}
    for kind in ("32", "c2f", "s16"):
        s[kind].G_forward(s[kind].g_inputs())
        s[kind].D_forward(s[kind].d_inputs())
    return s


def _close_state(s):
    for kind in ("c2f", "s16", "32"):
        s[kind].close()


def _train(s, B, real_scale):
    """one fg_train_step from the case's initial state (parameters, zero Adam moments, BatchNorm running state)"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    n, ctx, case = s["32"], s["ctx"], s["32"].case
    n.set_params()
    for net in (NET_D, NET_G):
        ctx.set_adam_state(net, np.zeros(ctx.count(net), np.float32), np.zeros(ctx.count(net), np.float32), 0)
    ctx.set_bn_state(PU.fresh_state(case, np.float32)["bnG"])
    st = ctx.train_step(fg.hyper_default(), B, scaled(case["real"][:B // 2], real_scale), case["noise_D"][:B // 2],
                        case["noise_G"][:B], case["masks_D"][:B], case["masks_G"][:B])
    return [ctx.get_params(NET_D), ctx.get_params(NET_G), np.float32([st["loss_D"], st["loss_G"]])]


@pytest.mark.parametrize("f16", F16)
@pytest.mark.parametrize("B", [256, 130])
def test_history_independence(B, f16):
    """on one context: L-op convolutions, G / D backward of all three pairs with operands 2^30 and 2^-30 in size,
    mma_f16 switched to the other value (one L-op call there) and back, a train step on images 2^-30 in
    size and then the same step again (a graph replay): every unscaled call returns the bits that a fresh context
    making only the unscaled calls returns"""
    ops = _history_ops(B, f16)
    s = _history_state(B, f16)
    got = {name: fn(s) for name, fn in ops}
    _train(s, B, -30)
    got["train step"] = _train(s, B, 0)
    _close_state(s)
    f = _history_state(B, f16)
    want = {name: fn(f) for name, fn in ops if name.endswith(" 0")}
    want["train step"] = _train(f, B, 0)
    _close_state(f)
    for name, w in want.items():
        for i, (a, b) in enumerate(zip(got[name], w)):
            same_bits(a, b, "%s, output %d" % (name, i))
