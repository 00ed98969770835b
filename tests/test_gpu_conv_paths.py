"""Every convolution and Linear kernel the layer ABI (fg_conv2d_*, fg_scu_*, fg_linear_*: what the Lua b200.* modules
call) can launch, held to float64 at the shapes where such kernels go wrong, with a witness of the kernel that ran.

Each row of ROWS names a shape on an edge of one kernel variant -- non-square images, batch tails of boxes that hold
several images, strips of the 32-wide edge kernels at H != 32, tile counts one past a wave, split-K with even and
ragged K ranges, FFMA tiles at every Cout / Cin threshold, Linear at K = 16384 and N = 1 -- and the kernel the
forward, data-gradient and weight-gradient calls must launch there: (kind, tile m, tile n, operand format, K splits),
read back through fg_get_option("last_conv_*").  So a dispatch that quietly sends a row elsewhere fails the row.

Each pass is compared with a float64 PyTorch convolution on the GPU (the checker test_gpu_headline.py pins to the C++
oracle), measured locally: forward and data gradient per image, the weight gradient per output channel, so that one
wrong batch-tail tile, N tile or K split cannot hide behind the rest of the tensor.  The bar is KTOL = 1e-5, as for
every isolated launch.  dW and db start from random nonzero buffers: the layer ABI accumulates (accGradParameters).

The last test checks that the witnessed variants are exactly the declared ones, and that the declared ones cover
every kernel instantiation the launchers can choose (INSTANTIATIONS).
"""
import ctypes as C
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KTOL = 1e-5  # one launch against fp64 on identical inputs
KIND = {"tapconv": 1, "wgrad_tc": 2, "reduce": 3, "expand": 4, "simt": 5, "flatk": 6, "wgrad_simt": 7}
FMT = {"fp32": 0, "tf32": 1, "f16": 2}

# every kernel instantiation the layer ABI's launchers choose from, (kind, tile m, tile n, format):
# launch_tapconv / tc_conv_wgrad: tapconv_tc_kernel / wgrad_tc_kernel<BN 64 | 128, F16 0 | 1>; launch_reduce<NS, VEC>,
# launch_expand<CS, N> (k_conv_edge.cu); k_conv_simt: conv_simt_kernel / conv_simt_flatk_kernel<8, TN 8 | 4 | 1>;
# k_wgrad_simt: wgrad_simt_kernel<TM, TN>, TM, TN in {8, 4, 1}
INSTANTIATIONS = (
    {(k, 128, bn, f) for k in ("tapconv", "wgrad_tc") for bn in (64, 128) for f in ("tf32", "f16")}
    | {("reduce", ns, vec, "fp32") for ns in (1, 3) for vec in (2, 4)}
    | {("expand", cs, n, "fp32") for cs in (1, 3, 4) for n in (64, 128)}
    | {(k, 8, tn, "fp32") for k in ("simt", "flatk") for tn in (8, 4, 1)}
    | {("wgrad_simt", tm, tn, "fp32") for tm in (8, 4, 1) for tn in (8, 4, 1)})


def W(kind, m, n, fmt="fp32", splits=1):
    return (kind, m, n, fmt, splits)


def tap(bn, fmt):
    return W("tapconv", 128, bn, fmt)


def wtc(bn, fmt, splits):
    return W("wgrad_tc", 128, bn, fmt, splits)


def simt(tn):
    return W("simt", 8, tn)


def flatk(tn):
    return W("flatk", 8, tn)


def wsimt(tm, tn, splits):
    return W("wgrad_simt", tm, tn, "fp32", splits)


class Row:
    """op "conv": (N, Cin, H, W, Cout, k); "scu": (N, Cin, H, W, nOutputPlane, k, factor); "linear": (N, in, out).
    N may be a function of the GPU's SM count (rows placed one tile past a wave).  mma_f16: the context option.
    want: the kernel of the forward, data-gradient and weight-gradient call.  Split counts are those of an H100 SXM
    (132 SMs)."""

    def __init__(self, name, op, shape, want, mma_f16=1):
        self.name, self.op, self.shape, self.mma_f16 = name, op, shape, mma_f16
        self.want = dict(zip(("fwd", "dgrad", "wgrad"), want))


ROWS = [
    # wgmma forward / data gradient, 3xFP16: k = 1 .. 9, N = 1, 3, 129, non-square images
    Row("tap_f16_k1_16x8", "conv", (3, 64, 16, 8, 128, 1), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 6))),
    Row("tap_f16_bn64_k3_4x32", "conv", (1, 64, 4, 32, 192, 3), (tap(64, "f16"), tap(64, "f16"), wsimt(8, 4, 1))),
    Row("tap_f16_k5_2x64", "conv", (3, 128, 2, 64, 64, 5), (tap(64, "f16"), tap(64, "f16"), wsimt(4, 8, 2))),
    Row("tap_f16_k7_1x128", "conv", (1, 64, 1, 128, 128, 7), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 2))),
    Row("tap_f16_k9_8x256", "conv", (1, 64, 8, 256, 128, 9), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 1))),
    Row("tap_f16_bn128_n129", "conv", (129, 64, 8, 16, 256, 3), (tap(128, "f16"), tap(64, "f16"), wtc(64, "f16", 7))),
    # persistent tiles: BN 128 at 2.5 waves, BN 64 (Cout = 64) and BN 64 by the wave heuristic one tile past a wave
    Row("tap_f16_bn128_2.5waves", "conv", (lambda S: 2 * S + S // 2, 64, 8, 16, 128, 3),
        (tap(128, "f16"), tap(64, "f16"), wtc(64, "f16", 14))),
    Row("tap_f16_bn64_sm+1", "conv", (lambda S: S + 1, 64, 8, 16, 64, 3),
        (tap(64, "f16"), tap(64, "f16"), wsimt(4, 4, 56))),
    Row("tap_f16_bn64_wave_heuristic_sm+1", "conv", (lambda S: S + 1, 64, 8, 16, 128, 1),
        (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 89))),
    # 3xTF32: Cin % 64 != 0, or the option mma_f16 = 0; the same image shapes
    Row("tap_tf32_cin32_16x8", "conv", (3, 32, 16, 8, 128, 3), (tap(64, "tf32"), simt(4), wsimt(8, 4, 2))),
    Row("tap_tf32_cin96_4x32", "conv", (3, 96, 4, 32, 64, 3), (tap(64, "tf32"), simt(8), wsimt(4, 8, 2))),
    Row("tap_tf32_2x64", "conv", (1, 64, 2, 64, 128, 5), (tap(64, "tf32"), tap(64, "tf32"), wtc(64, "tf32", 4)), mma_f16=0),
    Row("tap_tf32_1x128", "conv", (3, 128, 1, 128, 64, 3), (tap(64, "tf32"), tap(64, "tf32"), wsimt(4, 8, 2)), mma_f16=0),
    Row("tap_tf32_cin96_8x256", "conv", (1, 96, 8, 256, 128, 1), (tap(64, "tf32"), simt(8), wsimt(8, 8, 8))),
    Row("tap_tf32_bn128_n129", "conv", (129, 64, 8, 16, 256, 3), (tap(128, "tf32"), tap(64, "tf32"), wtc(64, "tf32", 7)),
        mma_f16=0),
    Row("tap_tf32_sm+1", "conv", (lambda S: S + 1, 32, 8, 16, 64, 3), (tap(64, "tf32"), simt(4), wsimt(4, 4, 56))),
    # several images per 128-pixel box: bb = 2, 8, 32, 128 at N = bb + 1 (TMA zero fill, predicated epilogue)
    Row("bb2_8x8_n3", "conv", (3, 64, 8, 8, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 3))),
    Row("bb8_4x4_n9", "conv", (9, 128, 4, 4, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(128, "f16", 3))),
    Row("bb32_2x2_n33", "conv", (33, 64, 2, 2, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 3))),
    Row("bb128_1x1_n129", "conv", (129, 64, 1, 1, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 3))),
    Row("bb8_4x4_n9_tf32", "conv", (9, 64, 4, 4, 128, 5), (tap(64, "tf32"), tap(64, "tf32"), wtc(64, "tf32", 5)), mma_f16=0),
    Row("bb128_1x1_n129_tf32", "conv", (129, 128, 1, 1, 64, 1), (tap(64, "tf32"), tap(64, "tf32"), wsimt(4, 8, 1)),
        mma_f16=0),
    # wgmma weight gradient: unsplit (k = 9: one split per SM is already more than a wave), split into K ranges that
    # divide evenly (24 K blocks, 12 splits of 2) and with a ragged last split (25 K blocks, 13 splits, the last of 1)
    Row("wg_f16_bn64_unsplit", "conv", (3, 64, 16, 16, 128, 9), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 1))),
    Row("wg_f16_bn128_unsplit", "conv", (2, 128, 8, 16, 128, 9), (tap(64, "f16"), tap(64, "f16"), wtc(128, "f16", 1))),
    Row("wg_f16_bn64_even", "conv", (24, 64, 8, 8, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 12))),
    Row("wg_f16_bn64_ragged", "conv", (25, 64, 8, 8, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 13))),
    Row("wg_f16_bn128_even", "conv", (24, 128, 8, 8, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(128, "f16", 12))),
    Row("wg_f16_bn128_ragged", "conv", (25, 128, 8, 8, 128, 3), (tap(64, "f16"), tap(64, "f16"), wtc(128, "f16", 13))),
    Row("wg_tf32_bn64_unsplit", "conv", (2, 64, 8, 16, 128, 9), (tap(64, "tf32"), tap(64, "tf32"), wtc(64, "tf32", 1)),
        mma_f16=0),
    Row("wg_tf32_bn128_unsplit", "conv", (2, 128, 8, 16, 128, 9), (tap(64, "tf32"), tap(64, "tf32"), wtc(128, "tf32", 1)),
        mma_f16=0),
    Row("wg_tf32_bn64_even", "conv", (24, 64, 4, 8, 128, 3), (tap(64, "tf32"), tap(64, "tf32"), wtc(64, "tf32", 12)),
        mma_f16=0),
    Row("wg_tf32_bn64_ragged", "conv", (25, 64, 4, 8, 128, 3), (tap(64, "tf32"), tap(64, "tf32"), wtc(64, "tf32", 13)),
        mma_f16=0),
    Row("wg_tf32_bn128_even", "conv", (24, 128, 4, 8, 128, 3), (tap(64, "tf32"), tap(64, "tf32"), wtc(128, "tf32", 12)),
        mma_f16=0),
    Row("wg_tf32_bn128_ragged", "conv", (25, 128, 4, 8, 128, 3), (tap(64, "tf32"), tap(64, "tf32"), wtc(128, "tf32", 13)),
        mma_f16=0),
    # the 32-wide edge kernels at H = 8, 24, 40, 64 (strip counts, the halo of the last strip), N = 1 and odd
    Row("edge_reduce_3x4_h8_n1", "conv", (1, 128, 8, 32, 3, 3),
        (W("reduce", 3, 4), W("expand", 3, 128), wsimt(1, 8, 1))),
    Row("edge_reduce_1x2_h24_n5", "conv", (5, 64, 24, 32, 1, 3),
        (W("reduce", 1, 2), W("expand", 1, 64), wsimt(1, 4, 15))),
    Row("edge_reduce_1x4_h40_n3", "conv", (3, 128, 40, 32, 1, 3),
        (W("reduce", 1, 4), W("expand", 1, 128), wsimt(1, 8, 15))),
    Row("edge_reduce_3x2_h64_n1", "conv", (1, 64, 64, 32, 3, 3),
        (W("reduce", 3, 2), W("expand", 3, 64), wsimt(1, 4, 8))),
    Row("edge_expand_4x64_h24_n7", "conv", (7, 4, 24, 32, 64, 3), (W("expand", 4, 64), simt(1), wsimt(4, 1, 21))),
    Row("edge_expand_4x128_h8_n1", "conv", (1, 4, 8, 32, 128, 3), (W("expand", 4, 128), simt(1), wsimt(8, 1, 1))),
    Row("edge_expand_1x128_h64_n3", "conv", (3, 1, 64, 32, 128, 3),
        (W("expand", 1, 128), W("reduce", 1, 4), wsimt(8, 1, 24))),
    Row("edge_expand_3x64_h40_n1", "conv", (1, 3, 40, 32, 64, 3),
        (W("expand", 3, 64), W("reduce", 3, 2), wsimt(4, 1, 5))),
    # FFMA: Cout 7 / 33 / 65 / 129, Cin 15 (taps x channels flattened) vs 16, k = 11, boxes that do not tile
    Row("simt_cin15_cout7_12x12", "conv", (3, 15, 12, 12, 7, 3), (flatk(1), flatk(1), wsimt(1, 1, 2))),
    Row("simt_cin16_cout33_12x12", "conv", (2, 16, 12, 12, 33, 3), (simt(4), simt(1), wsimt(4, 1, 2))),
    Row("simt_cin15_cout65_6x10_k5", "conv", (3, 15, 6, 10, 65, 5), (flatk(8), simt(1), wsimt(8, 1, 1))),
    Row("simt_cin16_cout129_6x10_k11", "conv", (1, 16, 6, 10, 129, 11), (simt(8), simt(1), wsimt(8, 1, 1))),
    Row("simt_cin3_cout33_k11", "conv", (3, 3, 12, 12, 33, 11), (flatk(4), simt(1), wsimt(4, 1, 2))),
    Row("simt_k11_16x16", "conv", (1, 64, 16, 16, 64, 11), (simt(4), simt(4), wsimt(4, 4, 1))),
    Row("simt_cin32_cout65_8x8", "conv", (2, 32, 8, 8, 65, 3), (simt(8), simt(4), wsimt(8, 4, 1))),
    Row("simt_cin65_cout33_12x12", "conv", (2, 65, 12, 12, 33, 3), (simt(4), simt(8), wsimt(4, 8, 2))),
    Row("simt_cin100_cout100_6x10", "conv", (2, 100, 6, 10, 100, 3), (simt(8), simt(8), wsimt(8, 8, 1))),
    # SpatialConvolutionUpsample: the convolution with nOutputPlane * factor^2 planes
    Row("scu_f2_8x16", "scu", (3, 64, 8, 16, 32, 3, 2), (tap(64, "f16"), tap(64, "f16"), wtc(64, "f16", 6))),
    Row("scu_f3_6x10", "scu", (2, 16, 6, 10, 5, 3, 3), (simt(4), simt(1), wsimt(4, 1, 1))),
    # Linear: N = 1 / 130, in = 1 / 100 / 16384, out = 1 / 37 / 513; the weight gradient with dx = NULL
    Row("lin_n1_in1_out1", "linear", (1, 1, 1), (simt(1), simt(1), wsimt(1, 1, 1))),
    Row("lin_n130_in100_out37", "linear", (130, 100, 37), (simt(4), simt(8), wsimt(4, 8, 1))),
    # K = 16384 on FFMA (one sequential fp32 sum per output) holds KTOL: measured 4.5e-6 per image (513 outputs) and
    # 8.6e-6 for the single output of N = 1, out = 1 (H100 80GB HBM3)
    Row("lin_n130_in16384_out513", "linear", (130, 16384, 513), (simt(8), simt(8), wsimt(8, 8, 1))),
    Row("lin_n1_in16384_out1", "linear", (1, 16384, 1), (simt(1), simt(8), wsimt(1, 8, 1))),
    Row("lin_n130_in1_out513", "linear", (130, 1, 513), (simt(8), simt(1), wsimt(8, 1, 1))),
    Row("lin_n1_in100_out513", "linear", (1, 100, 513), (simt(8), simt(8), wsimt(8, 8, 1))),
]


def coverage_key(w):
    kind, m, n, fmt, splits = w
    return (kind, m, n, fmt, "split" if splits > 1 else "unsplit")


DECLARED = {coverage_key(w) for r in ROWS for w in r.want.values()}
WITNESSED = set()
ATTEMPTED = set()


@pytest.fixture(scope="module")
def ctx():
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=8, channels=3)
    yield c
    c.close()


def p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def call(ctx, fn, *args):
    torch.cuda.synchronize()  # the library runs on its own stream: inputs written by torch must have landed
    rc = getattr(ctx.lib, fn)(ctx.h, *args)
    assert rc == 0, "%s: %s" % (fn, ctx.lib.fg_last_error().decode())
    ctx.sync()


def witness(ctx):
    get = lambda k: ctx.get_option("last_conv_" + k)
    kind = {v: k for k, v in KIND.items()}.get(get("kind"), "none")
    fmt = {v: k for k, v in FMT.items()}[get("format")]
    return (kind, get("tile_m"), get("tile_n"), fmt, get("splits"))


def check_witness(ctx, row, what):
    got = witness(ctx)
    WITNESSED.add(coverage_key(got))
    assert got == row.want[what], "%s %s ran %s, the row wants %s" % (row.name, what, got, row.want[what])


def local_err(got, ref):
    """max over the slices along dim 0 (images, or output channels) of max|got - ref| / max|ref| of that slice.
    A slice of one or a few sums that happen to cancel (a Linear layer with in = 1: one dot product per image) is
    measured against the rms of the whole tensor instead: its rounding error is set by the size of its terms, which
    it shares with the other slices.  A slice of many values always has max|ref| above the rms."""
    d = (got.double() - ref).abs().flatten(1).amax(1)
    s = ref.abs().flatten(1).amax(1).clamp_min(float(ref.square().mean().sqrt()))
    return float((d / s.clamp_min(1e-300)).max())


def slice_scale(ref):
    """max|ref| of each slice along dim 0, shaped to broadcast against ref"""
    return ref.abs().flatten(1).amax(1).view(-1, *[1] * (ref.dim() - 1)).float()


def rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g, device="cuda", dtype=torch.float64) * scale).float()


@pytest.mark.parametrize("row", ROWS, ids=[r.name for r in ROWS])
def test_conv_path(ctx, row):
    ATTEMPTED.add(row.name)
    F = torch.nn.functional
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(row.name.encode()))
    ctx.set_option("mma_f16", row.mma_f16)
    S = ctx.get_option("sm_count")
    shape = list(row.shape)
    if callable(shape[0]):
        shape[0] = shape[0](S)
    if row.op == "linear":
        N, fi, fo = shape
        x, w, b, dy = rand(g, N, fi), rand(g, fo, fi, scale=fi ** -0.5), rand(g, fo), rand(g, N, fo)
        x64, w64, dy64 = x.double(), w.double(), dy.double()
        ref = {"y": F.linear(x64, w64, b.double()), "dx": dy64 @ w64, "dw": dy64.t() @ x64, "db": dy64.sum(0)}
        y, dx = torch.empty(N, fo, device="cuda"), torch.empty_like(x)
        call(ctx, "fg_linear_forward", p(x), p(w), p(b), p(y), N, fi, fo)
        check_witness(ctx, row, "fwd")
        call(ctx, "fg_linear_backward", p(x), p(w), p(dy), p(dx), None, None, N, fi, fo)
        check_witness(ctx, row, "dgrad")
        dw0, db0 = rand(g, fo, fi) * slice_scale(ref["dw"]), rand(g, fo, scale=float(ref["db"].abs().max()))
        dw, db = dw0.clone(), db0.clone()
        call(ctx, "fg_linear_backward", p(x), p(w), p(dy), None, p(dw), p(db), N, fi, fo)  # Lin:accGradParameters
        check_witness(ctx, row, "wgrad")
    else:
        N, Cin, H, Wd, Cout, k = shape[:6]
        planes = Cout * shape[6] ** 2 if row.op == "scu" else Cout
        x, w = rand(g, N, Cin, H, Wd), rand(g, planes, Cin, k, k, scale=(Cin * k * k) ** -0.5)
        b, dy = rand(g, planes), rand(g, N, planes, H, Wd)
        x64, w64, dy64, pad = x.double(), w.double(), dy.double(), (k - 1) // 2
        ref = {"y": F.conv2d(x64, w64, b.double(), padding=pad),
               "dx": torch.nn.grad.conv2d_input(x.shape, w64, dy64, padding=pad),
               "dw": torch.nn.grad.conv2d_weight(x64, w.shape, dy64, padding=pad), "db": dy64.sum((0, 2, 3))}
        pre, extra = ("fg_scu_", (shape[6],)) if row.op == "scu" else ("fg_conv2d_", ())
        y, dx = torch.empty(N, planes, H, Wd, device="cuda"), torch.empty_like(x)
        call(ctx, pre + "forward", p(x), p(w), p(b), p(y), N, Cin, H, Wd, Cout, k, *extra)
        check_witness(ctx, row, "fwd")
        call(ctx, pre + "backward_data", p(dy), p(w), p(dx), N, Cin, H, Wd, Cout, k, *extra)
        check_witness(ctx, row, "dgrad")
        dw0, db0 = rand(g, *w.shape) * slice_scale(ref["dw"]), rand(g, planes, scale=float(ref["db"].abs().max()))
        dw, db = dw0.clone(), db0.clone()
        call(ctx, pre + "backward_filter", p(x), p(dy), p(dw), p(db), N, Cin, H, Wd, Cout, k, *extra)
        check_witness(ctx, row, "wgrad")
    # dW starts at a random buffer of the size of each channel's gradient, so the rounding of the += stays ~2^-24
    errs = {"y": local_err(y, ref["y"]), "dx": local_err(dx, ref["dx"]),
            "dw": local_err(dw.double() - dw0.double(), ref["dw"]),
            "db": float((db.double() - db0.double() - ref["db"]).abs().max() / ref["db"].abs().max())}
    print("%s N=%d %s" % (row.name, shape[0], " ".join("%s %.2e" % kv for kv in errs.items())))
    assert max(errs.values()) < KTOL, (row.name, errs)


def test_host_pointers_accumulate(ctx):
    """the same accumulation through host pointers (scratch copies in and out, dW / db loaded before the add)"""
    from face_generator_b200.lib import _ptr
    rng = np.random.default_rng(5)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    ctx.set_option("mma_f16", 1)
    for N, Cin, H, Wd, Cout, k in [(3, 64, 8, 16, 128, 3), (2, 15, 6, 10, 33, 5)]:  # wgrad_tc, wgrad_simt
        x, dy = f(rng.standard_normal((N, Cin, H, Wd))), f(rng.standard_normal((N, Cout, H, Wd)))
        dw0, db0 = f(rng.standard_normal((Cout, Cin, k, k)) * 10), f(rng.standard_normal(Cout) * 10)
        dw, db = dw0.copy(), db0.copy()
        assert ctx.lib.fg_conv2d_backward_filter(ctx.h, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), N, Cin, H, Wd, Cout, k) == 0
        x64, dy64 = torch.as_tensor(x, dtype=torch.float64), torch.as_tensor(dy, dtype=torch.float64)
        rdw = torch.nn.grad.conv2d_weight(x64, dw.shape, dy64, padding=(k - 1) // 2).numpy()
        rdb = dy64.sum((0, 2, 3)).numpy()
        assert np.abs(dw - dw0 - rdw).max() < KTOL * np.abs(rdw).max() + 4e-6  # + the rounding of the add at |dw0| ~ 10
        assert np.abs(db - db0 - rdb).max() < KTOL * np.abs(rdb).max() + 4e-6
    N, fi, fo = 5, 100, 37
    x, dy = f(rng.standard_normal((N, fi))), f(rng.standard_normal((N, fo)))
    dw0, db0 = f(rng.standard_normal((fo, fi))), f(rng.standard_normal(fo))
    dw, db = dw0.copy(), db0.copy()
    w = f(rng.standard_normal((fo, fi)))
    assert ctx.lib.fg_linear_backward(ctx.h, _ptr(x), _ptr(w), _ptr(dy), None, _ptr(dw), _ptr(db), N, fi, fo) == 0
    rdw, rdb = dy.astype(np.float64).T @ x.astype(np.float64), dy.astype(np.float64).sum(0)
    assert np.abs(dw - dw0 - rdw).max() < KTOL * np.abs(rdw).max() + 1e-6
    assert np.abs(db - db0 - rdb).max() < KTOL * np.abs(rdb).max() + 1e-6


BAD_CALLS = [
    ("fg_conv2d_forward", "xwby", (2, 16, 8, 8, 16, 2)),   # even k
    ("fg_conv2d_forward", "xwby", (2, 16, 8, 8, 16, -1)),  # negative k
    ("fg_conv2d_forward", "xwby", (0, 16, 8, 8, 16, 3)),   # zero batch
    ("fg_conv2d_backward_data", "ywx", (2, 16, 8, 8, 16, 4)),
    ("fg_conv2d_backward_data", "ywx", (2, 0, 8, 8, 16, 3)),   # zero input channels
    ("fg_conv2d_backward_data", "ywx", (2, 16, 8, 8, 16, -1)),
    ("fg_conv2d_backward_filter", "xyww", (2, 16, 8, 8, 16, 2)),
    ("fg_conv2d_backward_filter", "xyww", (2, 16, 0, 8, 16, 3)),  # zero height
    ("fg_conv2d_backward_filter", "xyww", (2, 16, 8, 8, 0, 3)),   # zero output channels
    ("fg_scu_forward", "xwby", (2, 16, 8, 8, 4, 3, 0)),  # factor 0
    ("fg_scu_backward_data", "ywx", (2, 16, 8, 8, 4, 3, -1)),
    ("fg_scu_backward_filter", "xyww", (2, 16, 8, 8, 4, 3, 0)),
    ("fg_linear_forward", "xwby", (2, 0, 4)),
    ("fg_linear_backward", "xwyxww", (2, 4, 0)),
    ("fg_linear_backward", "xwyxww", (2, 0, 4)),
]


def test_refusals_leave_the_context_usable(ctx):
    """even or negative k, zero sizes and an SCU factor < 1 are refused with an error (no kernel recorded), and the
    next call on the same context runs"""
    buf = torch.zeros(1 << 16, device="cuda")
    for fn, ptrs, args in BAD_CALLS:
        call(ctx, "fg_conv2d_forward", p(buf), p(buf), None, p(buf[4096:]), 1, 16, 8, 8, 16, 3)  # a good call first
        assert ctx.get_option("last_conv_kind") != 0
        rc = getattr(ctx.lib, fn)(ctx.h, *[p(buf)] * len(ptrs), *args)
        assert rc == -1, (fn, args, rc)  # FG_ERR_INVALID
        assert ctx.get_option("last_conv_kind") == 0, (fn, args)
    y = torch.empty(2, 16, 8, 8, device="cuda")
    x, w = torch.randn(2, 16, 8, 8, device="cuda"), torch.randn(16, 16, 3, 3, device="cuda")
    call(ctx, "fg_conv2d_forward", p(x), p(w), None, p(y), 2, 16, 8, 8, 16, 3)
    ref = torch.nn.functional.conv2d(x.double(), w.double(), padding=1)
    assert local_err(y, ref) < KTOL


def test_every_declared_variant_was_witnessed():
    """runs last: the variants the rows reached == the variants the table declares, and the declared ones cover
    every kernel instantiation, with split and unsplit weight gradients of every wgmma variant"""
    if ATTEMPTED != {r.name for r in ROWS}:
        pytest.skip("needs every row of test_conv_path in the same session")
    assert WITNESSED == DECLARED, ("witnessed, not declared", WITNESSED - DECLARED, "declared, not witnessed",
                                   DECLARED - WITNESSED)
    assert {k[:4] for k in DECLARED} == INSTANTIATIONS, INSTANTIATIONS ^ {k[:4] for k in DECLARED}
    for bn in (64, 128):
        for fmt in ("tf32", "f16"):
            assert {("wgrad_tc", 128, bn, fmt, s) for s in ("split", "unsplit")} <= DECLARED
    assert {k[4] for k in DECLARED if k[0] == "wgrad_simt"} == {"split", "unsplit"}
