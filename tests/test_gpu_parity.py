"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on seeded inputs.
Bar (BASELINE.json north_star): normwise relative error <= 1e-4 per tensor, fp32."""
import numpy as np
import pytest

import parity_utils as PU
from oracle import oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def fg():
    import face_generator_b200 as fg
    return fg


def nhwc_to_nchw(flat, B, H, W, C):
    return flat.reshape(B, H, W, C).transpose(0, 3, 1, 2)


def gcheck(cond, msg=""):
    assert cond, msg


# Gradient parity is STRICT (1e-4) for every case and seed: PReLU kinks are handled by parity_utils.kink_overrides
# (the oracle's backward takes the CUDA path's branch for the few pre-activations within KINK_MARGIN of 0, decided
# from oracle data only), not by retrying seeds.
def g_preact_getters(ctx, PG, C):
    """CUDA-path pre-activations of G's three PReLU layers (flat NHWC index -> value)."""
    lay = O.G_layout(C)
    sl = lambda k: PG[lay[k][0]:lay[k][0] + int(np.prod(lay[k][1]))]
    z0, z1, z2 = (ctx.debug_tensor("G.z%d" % i) for i in range(3))
    m1, s1, m2, s2 = (ctx.debug_tensor("G.bn_" + k) for k in ("mean1", "istd1", "mean2", "istd2"))
    g1, be1, g2, be2 = sl("g1"), sl("be1"), sl("g2"), sl("be2")
    return [lambda i: z0[i],
            lambda i: PU.bn_preact_gpu(z1[i], m1[i % 256], s1[i % 256], g1[i % 256], be1[i % 256]),
            lambda i: PU.bn_preact_gpu(z2[i], m2[i % 128], s2[i % 128], g2[i % 128], be2[i % 128])]


G_KINK_SHAPES = [(128, 8, 8), (256, 16, 16), (128, 32, 32)]
D_KINK_SHAPES = [(64, 32, 32), (128, 16, 16), (256, 8, 8), (512, 4, 4), (512, 1, 1), (512, 1, 1)]


def d_preact_getters(ctx, prefix="D."):
    zs = [ctx.debug_tensor(prefix + n) for n in ("z1", "z2", "z3", "z4", "zl1", "zl2")]
    return [(lambda i, z=z: z[i]) for z in zs]


def check_grads(layout, got, ref, skip=(), tol=TOL):
    scale = np.abs(ref).max()
    worst = 0.0
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        a, b = got[o:o + n].astype(np.float64), ref[o:o + n]
        if k in skip:  # analytically-zero gradients (conv bias feeding BatchNorm): only rounding noise
            assert np.abs(a).max() <= 1e-3 * scale + 1e-6, k
            continue
        e = np.abs(a - b).max() / (np.abs(b).max() + 1e-30)
        worst = max(worst, e)
        # the ONE shared PReLU slope per layer has a gradient that is a sum of ~1e6 terms with heavy cancellation:
        # its conditioning amplifies rounding by ~100x, so it gets a 3e-4 bar (everything else: 1e-4)
        t = 3 * tol if (k[0] == "a" and k[1:].isdigit()) else tol
        gcheck(e < t, "%s: relerr %.3e" % (k, e))
    return worst


@pytest.mark.parametrize("C,B,impl", [(3, 4, 0), (1, 6, 0), (3, 4, 2), (3, 6, 1), (1, 8, 2)])
@pytest.mark.parametrize("seed_off", [0, 100])
def test_G_forward_backward(fg, C, B, impl, seed_off):
    """real PReLU slopes, every seed strict (kink overrides)"""
    _G_forward_backward(fg, C, B, impl, 31 + C + seed_off)


@pytest.mark.parametrize("C,B,impl", [(3, 4, 2), (1, 4, 0)])
def test_G_forward_backward_reference_init(fg, C, B, impl):
    """the reference's own init (nn_utils.lua:17-29): slopes ~N(0, 0.005^2), i.e. possibly negative"""
    _G_forward_backward(fg, C, B, impl, 35 + C, init="reference")


@pytest.mark.parametrize("C,B,impl", [(3, 4, 0), (3, 4, 2), (3, 6, 1), (1, 8, 2)])
def test_G_forward_backward_smooth_strict(fg, C, B, impl):
    """PReLU slopes = 1: no kinks, every gradient at 1e-4, no retries."""
    _G_forward_backward(fg, C, B, impl, 431 + C, init="smooth")


def _G_forward_backward(fg, C, B, impl, seed, init="trained"):
    from face_generator_b200.lib import NET_G
    case = PU.make_case(2 * B, C, seed=seed, init=init)
    rng = np.random.default_rng(7)
    noise = case["noise_G"][:B]
    dout = rng.standard_normal((B, C, 32, 32)).astype(np.float32)
    g = O.f64.G()
    with O.kink.record(PU.KINK_MARGIN):
        ref_out = g.forward(case["PG"], noise, C)
    calls = O.kink.calls(3)
    ctx = fg.Context(0, max_batch=8, channels=C)
    ctx.set_option("conv_impl", impl)
    ctx.set_params(NET_G, case["PG"])
    out = ctx.G_forward(noise)
    assert PU.relerr(out, ref_out) < TOL
    PU.kink_overrides(calls, 0, g_preact_getters(ctx, case["PG"], C), G_KINK_SHAPES, label="G")
    with O.kink.override():
        g.forward(case["PG"], noise, C)
        ref_dP, ref_dn = g.backward(dout, want_dnoise=True)
    O.kink.clear()
    for name, (H, W, Cc) in {"z0": (8, 8, 128), "h0": (8, 8, 128), "z1": (16, 16, 256), "h1": (16, 16, 256),
                             "z2": (32, 32, 128), "h2": (32, 32, 128), "z3": (32, 32, C)}.items():
        got = nhwc_to_nchw(ctx.debug_tensor("G." + name), B, H, W, Cc)
        assert PU.relerr(got, g.tap(name)) < TOL, name
    ctx.zero_grads(NET_G)
    dn = ctx.G_backward(dout, want_dnoise=True)
    gG = ctx.get_grads(NET_G)
    bn = ctx.get_bn_state()
    ctx.close()
    check_grads(O.G_layout(C), gG, ref_dP, skip=("C1b", "C2b"))
    gcheck(PU.relerr(dn, ref_dn) < TOL, "dnoise")
    # BN running statistics after one training forward
    st = PU.fresh_state(case)["bnG"]
    O.f64.G().forward(case["PG"], noise, C, True, st)
    assert PU.relerr(bn, st) < TOL


@pytest.mark.parametrize("C,B,impl", [(3, 6, 0), (1, 4, 0), (3, 6, 2), (3, 8, 2)])
@pytest.mark.parametrize("seed_off", [0, 100])
def test_D_forward_backward(fg, C, B, impl, seed_off):
    _D_forward_backward(fg, C, B, impl, 41 + C + seed_off)


def test_D_forward_backward_reference_init(fg):
    _D_forward_backward(fg, 3, 6, 2, 47, init="reference")


@pytest.mark.parametrize("C,B,impl", [(3, 6, 0), (3, 6, 2), (1, 8, 2)])
def test_D_forward_backward_smooth_strict(fg, C, B, impl):
    _D_forward_backward(fg, C, B, impl, 441 + C, init="smooth")


def _D_forward_backward(fg, C, B, impl, seed, init="trained"):
    from face_generator_b200.lib import NET_D
    case = PU.make_case(B, C, seed=seed, init=init)
    rng = np.random.default_rng(8)
    img = rng.random((B, C, 32, 32)).astype(np.float32)
    dout = rng.standard_normal(B).astype(np.float32)
    d = O.f64.D()
    with O.kink.record(PU.KINK_MARGIN):
        ref_out = d.forward(case["PD"], img, case["masks_D"])
    calls = O.kink.calls(6)
    ctx = fg.Context(0, max_batch=8, channels=C)
    ctx.set_option("conv_impl", impl)
    ctx.set_params(NET_D, case["PD"])
    out = ctx.D_forward(img, masks=case["masks_D"])
    assert PU.relerr(out, ref_out) < TOL
    PU.kink_overrides(calls, 0, d_preact_getters(ctx), D_KINK_SHAPES, label="D")
    with O.kink.override():
        d.forward(case["PD"], img, case["masks_D"])
        ref_dP, ref_dimg = d.backward(dout)
    O.kink.clear()
    ctx.zero_grads(NET_D)
    dimg = ctx.D_backward(dout)
    gD = ctx.get_grads(NET_D)
    # evaluate(): dropout off (SpatialDropout scales by 1-p, Dropout is the identity)
    ref_eval = d.forward(case["PD"], img, None, training=False)
    assert PU.relerr(ctx.D_forward(img, training=False), ref_eval) < TOL
    ctx.close()
    # the shared PReLU slopes' gradients are sums with heavy cancellation: 3e-4 bar
    check_grads(O.D_layout(C), gD, ref_dP)
    gcheck(PU.relerr(dimg, ref_dimg) < TOL, "dimg")


@pytest.mark.parametrize("C,B,init,impl", [(1, 16, "trained", 0), (3, 8, "trained", 0), (3, 8, "reference", 0),
                                           (1, 16, "trained", 2), (3, 8, "trained", 2), (3, 8, "reference", 2),
                                           (3, 8, "trained", 1), (3, 8, "smooth", 0), (1, 16, "smooth", 2),
                                           (3, 8, "smooth", 2), (3, 8, "smooth", 1), (3, 64, "trained", 2)])
def test_train_step_matches_oracle(fg, C, B, init, impl):
    """BASELINE config 1 (gray, B=16: 8 real + 8 fake for D, 16 for G), colour cases and a B=64 step; gradients
    strict at 1e-4 for every case (kink overrides, no seed retries)."""
    _train_step_matches_oracle(fg, C, B, init, impl, 51 + C)


def _train_step_matches_oracle(fg, C, B, init, impl, seed, max_batch=None):
    from face_generator_b200.lib import NET_D, NET_G
    case = PU.make_case(B, C, seed=seed, init=init)
    ctx = fg.Context(0, max_batch=max_batch or max(16, B), channels=C)
    ctx.set_option("conv_impl", impl)
    ctx.set_option("debug_keep", 1)
    ctx.set_params(NET_G, case["PG"])
    ctx.set_params(NET_D, case["PD"])
    hyper = fg.hyper_default()
    st = ctx.train_step(hyper, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
    # ---- the whole iteration in the oracle (adversarial.lua:240-288).  With real PReLU slopes this pass also lists
    # the ambiguous PReLU elements; prelu_fwd call order inside train_iteration: 0-2 G (D step, forward only),
    # 3-8 D (D step), 9-11 G, 12-17 D (G step)
    kinks = init != "smooth"  # slopes 1: differentiable everywhere, nothing to override
    with O.kink.record(PU.KINK_MARGIN if kinks else 0.0):
        ref = PU.oracle_iteration(case, B, C)
    calls = O.kink.calls(18)
    # Losses.  nn.BCECriterion (train.lua:148) sees D's sigmoid outputs as FLOAT32 (the reference's nn.Copy hands it
    # a FloatTensor): near saturation log(1 - x + eps) amplifies the fp32 rounding of x by 1/(1-x), so the loss of two
    # correct fp32 pipelines agrees only to ~1e-4..1e-3 at batch 256, while the fp64 oracle never rounds x.  The
    # well-conditioned statement is therefore split in two: (i) the logits match the oracle at 1e-4; (ii) the loss
    # equals the oracle's criterion (+ penalty) evaluated ON the CUDA path's own float32 outputs at 1e-5.
    tD = np.concatenate([np.ones(B // 2), np.zeros(B // 2)])
    def logits_match(got, x_ref):
        """logit(x_ref) is finite in fp64 up to ~36; beyond ~25 the sigmoid output carries no digits of the logit
        any more: compare where it does, require agreement in saturation elsewhere"""
        with np.errstate(divide="ignore"):
            ref = np.log(x_ref) - np.log1p(-x_ref)
        ok = np.isfinite(ref) & (np.abs(ref) < 25)
        got = np.asarray(got, np.float64)
        assert np.all(np.abs(got[~ok]) > 20) and np.all(np.sign(got[~ok]) == np.sign(x_ref[~ok] - 0.5))
        return not ok.any() or np.abs(got[ok] - ref[ok]).max() < TOL * max(1.0, np.abs(ref[ok]).max())

    out_D, out_G = ctx.debug_tensor("Dstep.out").astype(np.float64), ctx.debug_tensor("D.out").astype(np.float64)
    assert logits_match(ctx.debug_tensor("Dstep.logit"), ref["outD"])
    pen_D = ref["lossD"] - O.f64.bce_fwd(ref["outD"], tD)  # the L1/L2 term of fevalD (adversarial.lua:103-106)
    assert abs(st["loss_D"] - (O.f64.bce_fwd(out_D, tD) + pen_D)) < 1e-5 * max(1.0, abs(ref["lossD"]))
    assert abs(st["loss_D"] - ref["lossD"]) < 2e-3 * max(1.0, abs(ref["lossD"]))
    assert abs(st["loss_G"] - O.f64.bce_fwd(out_G, np.ones(B))) < 1e-5 * max(1.0, abs(ref["lossG"]))  # G_L1 = G_L2 = 0
    assert abs(st["loss_G"] - ref["lossG"]) < 2e-3 * max(1.0, abs(ref["lossG"]))
    assert st["conf"] == [int(v) for v in ref["conf"]]
    assert st["t_D"] == 1 and st["t_G"] == 1 and st["trained_D"] == 1
    gD, gG = ctx.get_grads(NET_D), ctx.get_grads(NET_G)
    mD, vD, tD = ctx.get_adam_state(NET_D)
    PDn = ctx.get_params(NET_D)
    # ---- D step, strict: the oracle's backward takes the CUDA path's branch at the D step's ambiguous elements
    rd = dict(gradD=ref["gradD"], mD=ref["state"]["mD"], PD=ref["state"]["PD"])
    if kinks:
        O.kink.clear()
        PU.kink_overrides(calls[3:9], 0, d_preact_getters(ctx, "Dstep."), D_KINK_SHAPES, label="D step")
        with O.kink.override():
            rd = PU.oracle_dstep(case["PD"], case["real"], ref["fake"], case["masks_D"], B, C)
        O.kink.clear()
        assert abs(rd["lossD"] - ref["lossD"]) < 1e-9  # the composition == the monolithic iteration
    gcheck(PU.relerr(gD, rd["gradD"]) < TOL, "gradD %.3e" % PU.relerr(gD, rd["gradD"]))  # post penalty + clamp
    gcheck(PU.relerr(mD, rd["mD"]) < TOL and tD == 1, "adam m")  # linear in the gradient
    # parameters: |update| = lr at t=1 whatever |g| is, so compare only where the gradient is not noise
    big = np.abs(rd["gradD"]) > 1e-3 * np.abs(rd["gradD"]).max()
    gcheck(np.abs(PDn[big] - rd["PD"][big]).max() < 2e-5, "params after Adam")
    # ---- G step, strict, on the CUDA path's own post-Adam D parameters (see parity_utils.oracle_gstep)
    if kinks:
        with O.kink.record(PU.KINK_MARGIN):
            PU.oracle_gstep(case["PG"], PDn, case["noise_G"], case["masks_G"], B, C, forward_only=True)
        calls = O.kink.calls(9)
        PU.kink_overrides(calls, 0, g_preact_getters(ctx, case["PG"], C), G_KINK_SHAPES, label="G step / G")
        PU.kink_overrides(calls, 3, d_preact_getters(ctx, "D."), D_KINK_SHAPES, label="G step / D")
    with O.kink.override():
        rg = PU.oracle_gstep(case["PG"], PDn, case["noise_G"], case["masks_G"], B, C)
    O.kink.clear()
    ctx_logit_G = ctx.debug_tensor("D.logit")
    ctx.close()
    assert logits_match(ctx_logit_G, rg["outD"])  # the G step's D logits on identical D parameters
    if init in ("trained", "smooth"):
        check_grads(O.G_layout(C), gG, rg["gradG"], skip=("C1b", "C2b"))
    else:
        gcheck(PU.relerr(gG, rg["gradG"]) < TOL, "gradG %.3e" % PU.relerr(gG, rg["gradG"]))


def test_modules_equal_fused_step(fg):
    """The nn.Module-level composition (fevalD / fevalG_on_D) and the fused fg_train_step are the same math."""
    from face_generator_b200.lib import NET_D, NET_G
    from face_generator_b200 import adversarial as A
    B, C = 8, 3
    case = PU.make_case(B, C, seed=61, init="smooth")  # no PReLU kinks: the two paths may only differ by atomics order
    hyper = fg.hyper_default()
    res = {}
    for mode in ("fused", "modules"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        if mode == "fused":
            ctx.train_step(hyper, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        else:
            A.train_batch_modules(ctx, hyper, case["real"], case["noise_D"], case["noise_G"], case["masks_D"],
                                  case["masks_G"])
        res[mode] = (ctx.get_params(NET_D), ctx.get_params(NET_G), ctx.get_grads(NET_D), ctx.get_grads(NET_G))
        ctx.close()
    for a, b in zip(res["fused"][2:], res["modules"][2:]):
        assert PU.relerr(a, b) < 2e-5
    for a, b in zip(res["fused"][:2], res["modules"][:2]):
        assert np.abs(a - b).max() < 2.1e-3  # sign flips of noise-level gradients move a parameter by 2*lr


@pytest.mark.parametrize("N,Cin,H,Cout,k", [(8, 64, 16, 128, 3), (3, 128, 8, 256, 3), (5, 256, 4, 512, 3),
                                            (2, 32, 32, 64, 5), (3, 64, 16, 128, 7), (1, 128, 32, 128, 1)])
def test_tc_conv_lop(fg, N, Cin, H, Cout, k):
    """wgmma 3xTF32 implicit-GEMM kernels (fwd, dgrad, wgrad) in isolation through the L-op ABI; includes batch
    tails that do not fill a 128-pixel tile (TMA zero fill + predicated epilogue)."""
    from face_generator_b200.lib import _ptr
    rng = np.random.default_rng(100 + N + Cin)
    ctx = fg.Context(0, max_batch=8, channels=3)
    ctx.set_option("conv_impl", 2)
    lib, h = ctx.lib, ctx.h
    f = lambda a: np.ascontiguousarray(a, np.float32)
    x, w, b = f(rng.standard_normal((N, Cin, H, H))), f(rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)), f(rng.standard_normal(Cout))
    dy = f(rng.standard_normal((N, Cout, H, H)))
    y = np.empty((N, Cout, H, H), np.float32)
    assert lib.fg_conv2d_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, H, H, Cout, k) == 0, lib.fg_last_error()
    ref = O.f64.conv_fwd(x, w, b)
    assert PU.relerr(y, ref) < 1e-5, PU.relerr(y, ref)  # 3xTF32 + chunked promotion: ~fp32 accurate (measured 1-3e-6)
    rdx, rdw, rdb = O.f64.conv_bwd(x, w, dy)
    dx = np.empty_like(x)
    assert lib.fg_conv2d_backward_data(h, _ptr(dy), _ptr(w), _ptr(dx), N, Cin, H, H, Cout, k) == 0, lib.fg_last_error()
    assert PU.relerr(dx, rdx) < 1e-5, PU.relerr(dx, rdx)
    dw, db = np.zeros_like(w), np.zeros_like(b)
    assert lib.fg_conv2d_backward_filter(h, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), N, Cin, H, H, Cout, k) == 0, lib.fg_last_error()
    assert PU.relerr(dw, rdw) < 1e-5 and PU.relerr(db, rdb) < TOL, PU.relerr(dw, rdw)
    ctx.close()


def test_lop_layers(fg):
    """L-op ABI (what the Lua b200.* nn.Modules call) against the oracle ops, NCHW in/out."""
    import ctypes as Cc
    from face_generator_b200.lib import _ptr
    rng = np.random.default_rng(71)
    ctx = fg.Context(0, max_batch=8, channels=3)
    lib, h = ctx.lib, ctx.h
    f = lambda a: np.ascontiguousarray(a, np.float32)
    for (N, Cin, H, Cout, k) in [(3, 5, 8, 7, 3), (2, 16, 16, 32, 5), (2, 4, 32, 6, 7)]:
        x, w, b = f(rng.standard_normal((N, Cin, H, H))), f(rng.standard_normal((Cout, Cin, k, k)) * 0.1), f(rng.standard_normal(Cout))
        dy = f(rng.standard_normal((N, Cout, H, H)))
        y = np.empty((N, Cout, H, H), np.float32)
        assert lib.fg_conv2d_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, H, H, Cout, k) == 0
        assert PU.relerr(y, O.f64.conv_fwd(x, w, b)) < TOL
        rdx, rdw, rdb = O.f64.conv_bwd(x, w, dy)
        dx = np.empty_like(x)
        assert lib.fg_conv2d_backward_data(h, _ptr(dy), _ptr(w), _ptr(dx), N, Cin, H, H, Cout, k) == 0
        assert PU.relerr(dx, rdx) < TOL
        dw, db = np.zeros_like(w), np.zeros_like(b)
        assert lib.fg_conv2d_backward_filter(h, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), N, Cin, H, H, Cout, k) == 0
        assert PU.relerr(dw, rdw) < TOL and PU.relerr(db, rdb) < TOL
    # Linear
    N, fi, fo = 5, 100, 37
    x, w, b, dy = f(rng.standard_normal((N, fi))), f(rng.standard_normal((fo, fi))), f(rng.standard_normal(fo)), f(rng.standard_normal((N, fo)))
    y = np.empty((N, fo), np.float32)
    assert lib.fg_linear_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, fi, fo) == 0
    assert PU.relerr(y, O.f64.linear_fwd(x, w, b)) < TOL
    dx, dw, db = np.empty_like(x), np.zeros_like(w), np.zeros_like(b)
    assert lib.fg_linear_backward(h, _ptr(x), _ptr(w), _ptr(dy), _ptr(dx), _ptr(dw), _ptr(db), N, fi, fo) == 0
    rdx, rdw, rdb = O.f64.linear_bwd(x, w, dy)
    assert PU.relerr(dx, rdx) < TOL and PU.relerr(dw, rdw) < TOL and PU.relerr(db, rdb) < TOL
    # BatchNorm (training) + backward
    N, Cn, H = 4, 24, 6
    x, g, be, dy = f(rng.standard_normal((N, Cn, H, H)) * 2 + 1), f(rng.uniform(0.5, 1.5, Cn)), f(rng.standard_normal(Cn)), f(rng.standard_normal((N, Cn, H, H)))
    y, sm, si = np.empty_like(x), np.empty(Cn, np.float32), np.empty(Cn, np.float32)
    rm, rv = np.zeros(Cn, np.float32), np.ones(Cn, np.float32)
    assert lib.fg_bn_forward_train(h, _ptr(x), _ptr(g), _ptr(be), _ptr(y), _ptr(sm), _ptr(si), _ptr(rm), _ptr(rv), N, Cn, H * H) == 0
    rrm, rrv = np.zeros(Cn), np.ones(Cn)
    ry, rmean, ristd = O.f64.bn_fwd_train(x, g, be, rrm, rrv)
    assert PU.relerr(y, ry) < TOL and PU.relerr(sm, rmean) < TOL and PU.relerr(si, ristd) < TOL
    assert PU.relerr(rm, rrm) < TOL and PU.relerr(rv, rrv) < TOL
    dx, dg, db = np.empty_like(x), np.zeros(Cn, np.float32), np.zeros(Cn, np.float32)
    assert lib.fg_bn_backward(h, _ptr(x), _ptr(g), _ptr(sm), _ptr(si), _ptr(dy), _ptr(dx), _ptr(dg), _ptr(db), N, Cn, H * H) == 0
    rdx, rdg, rdb = O.f64.bn_bwd(x, g, rmean, ristd, dy)
    assert PU.relerr(dx, rdx) < TOL and PU.relerr(dg, rdg) < TOL and PU.relerr(db, rdb) < TOL
    # PReLU
    x, dy, a = f(rng.standard_normal(1000)), f(rng.standard_normal(1000)), np.array([0.25], np.float32)
    y = np.empty_like(x)
    assert lib.fg_prelu_forward(h, _ptr(x), _ptr(a), _ptr(y), 1000) == 0
    assert PU.relerr(y, O.f64.prelu_fwd(x, 0.25)) < 1e-6
    dx, da = np.empty_like(x), np.zeros(1, np.float32)
    assert lib.fg_prelu_backward(h, _ptr(x), _ptr(a), _ptr(dy), _ptr(dx), _ptr(da), 1000) == 0
    rdx, rda = O.f64.prelu_bwd(x, 0.25, dy)
    assert PU.relerr(dx, rdx) < 1e-6 and abs(da[0] - rda) < TOL * abs(rda)
    # BCE incl. saturation: composed gradient through a saturated sigmoid is exactly 0 (SURVEY X1)
    xs, ts = f([1.0, 0.0, 0.3, 0.9]), f([0.0, 1.0, 1.0, 0.0])
    assert abs(ctx.bce_forward(xs, ts) - O.f64.bce_fwd(xs, ts)) < 1e-4 * O.f64.bce_fwd(xs, ts)
    gb = ctx.bce_backward(xs, ts)
    assert PU.relerr(gb[2:], O.f64.bce_bwd(xs, ts)[2:]) < 1e-5
    assert np.all(gb[:2] * xs[:2] * (1 - xs[:2]) == 0)
    ctx.close()


def test_adam_op_and_error_paths(fg):
    from face_generator_b200.lib import _ptr, FGError
    rng = np.random.default_rng(81)
    ctx = fg.Context(0, max_batch=8, channels=3)
    n = 100003
    p, g = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    m, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
    dp, dg, dm, dv = (ctx.dev_array(a) for a in (p, g, m, v))
    p64, m64, v64 = p.astype(np.float64), m.astype(np.float64), v.astype(np.float64)
    for t in (1, 2, 3):
        assert ctx.lib.fg_adam_step(ctx.h, dp, dg, dm, dv, n, 1e-3, 0.9, 0.999, 1e-8, t, 0.0, 1e-4, 1.0, 1.0) == 0
        g64 = g.astype(np.float64)
        O.f64.penalty_clamp(p64, g64, 0.0, 0.0, 1e-4, 1.0)
        O.f64.adam(p64, g64, m64, v64, t)
        # fg_adam_step rewrites g with the penalised/clamped gradient: restore the raw one
        ctx.lib.fg_memcpy(ctx.h, dg, _ptr(g), g.nbytes)
    out = np.empty(n, np.float32)
    ctx.lib.fg_memcpy(ctx.h, _ptr(out), dp, out.nbytes)
    assert np.abs(out - p64).max() < 1e-6
    for d in (dp, dg, dm, dv):
        ctx.dev_free(d)
    # error behaviour: odd / too-large batches are rejected with a message, nothing crashes
    case = PU.make_case(8, 3, seed=1)
    hyper = fg.hyper_default()
    with pytest.raises(FGError):
        ctx.train_step(hyper, 6 + 1, case["real"], case["noise_D"], case["noise_G"])
    with pytest.raises(FGError):
        ctx.train_step(hyper, 16, case["real"], case["noise_D"], case["noise_G"])
    with pytest.raises(FGError):
        ctx.G_backward(np.zeros((4, 3, 32, 32), np.float32))  # backward before forward
    with pytest.raises(FGError):
        fg.Context(0, max_batch=8, channels=2)
    ctx.close()


def test_sample_chunked(fg):
    """sample.lua:80: G forward in chunks with train-mode BN (per-chunk statistics)."""
    from face_generator_b200.lib import NET_G
    C, N, chunk = 3, 10, 4
    case = PU.make_case(8, C, seed=91)
    noise = np.random.default_rng(9).uniform(-1, 1, (N, 100)).astype(np.float32)
    ctx = fg.Context(0, max_batch=8, channels=C)
    ctx.set_params(NET_G, case["PG"])
    out = ctx.sample(noise, chunk)
    ref = np.concatenate([O.f64.G().forward(case["PG"], noise[s:s + chunk], C) for s in range(0, N, chunk)])
    assert PU.relerr(out, ref) < TOL
    ctx.close()


def test_accuracy_gate_closes_and_reopens(fg):
    """adversarial.lua:156-178 + interruptable_optimizers.lua:64-66: when the mean of D's last `accsInterval` batch
    accuracies is >= maxAccuracyD, fevalD returns false and interruptableAdam returns without touching x, m, v or
    its step counter.  The per-step thresholds make the gate close, stay closed and reopen; the expected decision
    is a literal transcription of the Lua fed with the batch accuracies the step reports (which are themselves
    checked against the confusion counts)."""
    from face_generator_b200.lib import NET_D, NET_G
    B, C, interval = 8, 3, 3
    case = PU.make_case(B, C, seed=77)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_params(NET_G, case["PG"])
    ctx.set_params(NET_D, case["PD"])
    accs, tD, n_closed, n_open = [], 0, 0, 0
    # 1.01 (the default) never closes, 0.0 always closes; 0.5625 = 13.5/24 lies strictly between the possible means of
    # three batch accuracies (multiples of 1/24), so the decision depends on the data but never on rounding
    thresholds = [1.01, 0.0, 0.0, 1.01, 0.5625, 0.5625, 0.5625, 1.01]
    for it, thr in enumerate(thresholds):
        rng = np.random.default_rng(100 + it)
        real = rng.random((B // 2, C, 32, 32)).astype(np.float32)
        nD, nG = rng.uniform(-1, 1, (B // 2, 100)).astype(np.float32), rng.uniform(-1, 1, (B, 100)).astype(np.float32)
        mk_D, mk_G = PU.make_masks(B, rng).astype(np.float32), PU.make_masks(B, rng).astype(np.float32)
        before = (ctx.get_params(NET_D),) + ctx.get_adam_state(NET_D)
        PG0 = ctx.get_params(NET_G)
        hyper = fg.hyper_default()
        hyper.D_maxAcc, hyper.accs_interval = thr, interval
        st = ctx.train_step(hyper, B, real, nD, nG, mk_D, mk_G)
        # ---- transcription of adversarial.lua:112-117, :156-178
        tV = (st["conf"][0] + st["conf"][3]) / float(B)
        assert abs(st["acc_D"] - tV) < 1e-6
        accs.append(tV)
        if len(accs) > interval:
            accs.pop(0)
        do_train = (sum(accs) / len(accs)) < thr
        assert st["trained_D"] == int(do_train), (it, accs, thr, st)
        after = (ctx.get_params(NET_D),) + ctx.get_adam_state(NET_D)
        if do_train:
            tD += 1
            n_open += 1
            assert np.abs(after[0] - before[0]).max() > 1e-4  # Adam moved D
        else:  # interruptable_optimizers.lua:64-66: nothing is touched
            n_closed += 1
            for a, b in zip(after[:3], before[:3]):
                np.testing.assert_array_equal(a, b)
        assert st["t_D"] == tD == after[3] and st["t_G"] == it + 1
        assert np.abs(ctx.get_params(NET_G) - PG0).max() > 1e-4  # G trains on every iteration (adversarial.lua:275-288)
    assert n_closed >= 2 and n_open >= 3
    ctx.close()
