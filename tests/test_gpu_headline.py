"""Parity at the HEADLINE size (BASELINE.json configs[1]: colour, batch 256 per GPU) and at a ragged batch (130).

At B=256 the persistent wgmma kernels run many tiles per CTA (stage-ring wrap-around, cross-block phase waits,
split-K sized to a wave, the BN=64/128 tile heuristic) -- code paths the small-batch parity tests never reach.
The fp64 C++ oracle needs ~1 min per iteration at this size, so two checkers are used:

 * a float64 PyTorch restatement on the same GPU (tests/torch_ref.py), which tests/test_oracle_vs_torch.py pins to
   the C++ oracle at 1e-8 on CPU (same functions, small batch).  It checks every tensor-core launch in ISOLATION
   (the kernel's input is the CUDA path's own tensor, so errors do not accumulate) at 1e-5, and whole-net
   gradients at 1e-4 with the PReLU-kink override of parity_utils (branches of pre-activations within 2e-5 of 0
   are taken from the CUDA path, everything else from the checker);
 * the C++ oracle itself (O.f64.train_iteration) for one full fg_train_step at B=256.
"""
import numpy as np
import pytest

import parity_utils as PU
from oracle import oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
TOL = 1e-4
KTOL = 1e-5  # one tensor-core launch against fp64 on identical inputs (3xTF32 + chunked promotion: measured 1-5e-6)


@pytest.fixture(scope="module")
def fg():
    import face_generator_b200 as fg
    return fg


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def nchw(flat, B, H, W, C):
    """NHWC debug tensor -> float64 NCHW torch tensor on the GPU"""
    return dev(flat.reshape(B, H, W, C)).permute(0, 3, 1, 2).contiguous()


def rel(a, b):
    a = a if torch.is_tensor(a) else dev(a)
    b = b if torch.is_tensor(b) else dev(b)
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


def test_torch_f64_gpu_equals_oracle_small():
    """the fast checker used below == the C++ oracle (small batch, same code path as at B=256)"""
    import torch_ref as R
    rng = np.random.default_rng(3)
    x, w, b = rng.standard_normal((3, 16, 8, 8)), rng.standard_normal((24, 16, 5, 5)) * 0.1, rng.standard_normal(24)
    y = torch.nn.functional.conv2d(dev(x), dev(w), dev(b), padding=2)
    assert rel(y, O.f64.conv_fwd(x, w, b)) < 1e-12
    case = PU.make_case(8, 3, seed=77)
    out, _ = R.G_forward(dev(case["PG"]), dev(case["noise_G"][:4]), 3)
    assert rel(out, O.f64.G().forward(case["PG"], case["noise_G"][:4], 3)) < 1e-10
    od = R.D_forward(dev(case["PD"]), dev(case["real"]), dev(case["masks_D"][:4]), 3)
    assert rel(od, O.f64.D().forward(case["PD"], case["real"], case["masks_D"][:4])) < 1e-10


def kink_branch(gpu_pos, counts, margin=PU.KINK_MARGIN):
    """branch hook for torch_ref.prelu: own decision except where |x| < margin*max|x| (then the CUDA path's)"""
    def branch(name, x):
        amb = x.abs() < margin * x.abs().max()
        counts[name] = (int(amb.sum()), x.numel())
        assert counts[name][0] <= max(8, PU.KINK_MAX_FRAC * x.numel()), (name, counts[name])
        return torch.where(amb, gpu_pos[name], x > 0)
    return branch


@pytest.mark.parametrize("B", [256, 130])
def test_G_at_headline_batch(fg, B):
    _G_at_headline_batch(fg, B, 2)


@pytest.mark.parametrize("B", [256, 130])
def test_G_dense_forward_at_headline_batch(fg, B):
    """conv_impl = 1: C1 / C2 forward on the dense 25-tap pack of the upsampled 5x5 layers (same checks)"""
    _G_at_headline_batch(fg, B, 1)


def _G_at_headline_batch(fg, B, impl):
    import torch_ref as R
    F = torch.nn.functional
    from face_generator_b200.lib import NET_G
    C = 3
    case = PU.make_case(2 * B, C, seed=2000 + B)
    noise = case["noise_G"][:B]
    dout = np.random.default_rng(B).standard_normal((B, C, 32, 32)).astype(np.float32)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_option("conv_impl", impl)
    ctx.set_params(NET_G, case["PG"])
    out = ctx.G_forward(noise)
    p = R._split(dev(case["PG"]), O.G_layout(C))
    T = {n: nchw(ctx.debug_tensor("G." + n), B, H, H, Cc) for n, H, Cc in
         (("z0", 8, 128), ("h0", 8, 128), ("z1", 16, 256), ("h1", 16, 256), ("z2", 32, 128), ("h2", 32, 128), ("z3", 32, C))}
    # ---- every forward launch on the CUDA path's own input ----
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")
    assert rel(T["z0"], F.linear(dev(noise), p["L1W"], p["L1b"]).view(B, 128, 8, 8)) < KTOL
    assert rel(T["z1"], F.conv2d(up(T["h0"]), p["C1W"], p["C1b"], padding=2)) < KTOL  # tensor cores, collapsed phases
    assert rel(T["z2"], F.conv2d(up(T["h1"]), p["C2W"], p["C2b"], padding=2)) < KTOL  # tensor cores, collapsed phases
    assert rel(T["z3"], F.conv2d(T["h2"], p["C3W"], p["C3b"], padding=1)) < KTOL
    for zn, hn, g, be, a in (("z1", "h1", "g1", "be1", "a2"), ("z2", "h2", "g2", "be2", "a3")):
        y = F.batch_norm(T[zn], None, None, p[g], p[be], training=True, eps=1e-5)
        assert rel(T[hn], torch.where(y > 0, y, p[a] * y)) < KTOL
    # ---- whole net, forward + backward, against the fp64 restatement (kink override) ----
    g_pos = {}
    m1, s1, m2, s2 = (dev(ctx.debug_tensor("G.bn_" + k)).view(1, -1, 1, 1) for k in ("mean1", "istd1", "mean2", "istd2"))
    f32 = lambda t: t.to(torch.float32)
    g_pos["z0"] = T["z0"] > 0
    for zn, m, s, g, be, key in (("z1", m1, s1, "g1", "be1", "y1"), ("z2", m2, s2, "g2", "be2", "y2")):
        t = f32(f32(f32(T[zn]) - f32(m)) * f32(s))  # the kernels' u = fma(gamma, fl((z-mean)*istd), beta), k_elem.cu
        g_pos[key] = (f32(p[g]).view(1, -1, 1, 1).double() * t.double() + f32(p[be]).view(1, -1, 1, 1).double()) > 0
    counts = {}
    P = dev(case["PG"]).requires_grad_(True)
    nz = dev(noise).requires_grad_(True)
    ref_out, _ = R.G_forward(P, nz, C, branch=kink_branch(g_pos, counts))
    assert rel(out, ref_out.detach()) < TOL
    ref_out.backward(dev(dout))
    ctx.zero_grads(NET_G)
    dn = ctx.G_backward(dout, want_dnoise=True)
    gG = ctx.get_grads(NET_G)
    assert rel(dn, nz.grad) < TOL
    ref = P.grad.cpu().numpy()
    for k, (o, s) in O.G_layout(C).items():
        n = int(np.prod(s))
        if k in ("C1b", "C2b"):  # analytically zero (bias feeding BatchNorm): rounding noise only
            continue
        tol = 3 * TOL if k in ("a1", "a2", "a3") else TOL  # one shared slope: a heavily cancelling sum
        assert PU.relerr(gG[o:o + n], ref[o:o + n]) < tol, (k, PU.relerr(gG[o:o + n], ref[o:o + n]), counts)
    # ---- the backward tensor-core launches in isolation, on the CUDA path's own dz tensors ----
    dz2, dz1, dz0 = (nchw(ctx.debug_tensor("G.dz%d" % i), B, H, H, Cc) for i, H, Cc in ((2, 32, 128), (1, 16, 256), (0, 8, 128)))
    lay = O.G_layout(C)
    blk = lambda k: gG[lay[k][0]:lay[k][0] + int(np.prod(lay[k][1]))].reshape(lay[k][1])
    wg = torch.nn.grad.conv2d_weight
    assert rel(blk("C2W"), wg(up(T["h1"]), p["C2W"].shape, dz2, padding=2)) < KTOL  # wgrad_tc (36 collapsed taps, split-K)
    assert rel(blk("C1W"), wg(up(T["h0"]), p["C1W"].shape, dz1, padding=2)) < KTOL
    pool = lambda t: F.avg_pool2d(t, 2, 2) * 4  # backward of the nearest upsample: 2x2 sum
    dh0 = pool(torch.nn.grad.conv2d_input(up(T["h0"]).shape, p["C1W"], dz1, padding=2))  # tapconv dgrad, 4 phases summed
    assert rel(dz0, dh0 * torch.where(T["z0"] > 0, 1.0, float(p["a1"]))) < KTOL
    dh1 = pool(torch.nn.grad.conv2d_input(up(T["h1"]).shape, p["C2W"], dz2, padding=2))
    z1 = T["z1"].clone().requires_grad_(True)
    y1 = F.batch_norm(z1, None, None, p["g1"], p["be1"], training=True, eps=1e-5)
    torch.where(g_pos["y1"], y1, p["a2"] * y1).backward(dh1)
    assert rel(dz1, z1.grad) < 5 * KTOL  # BN backward subtracts two batch means: a few ulps more
    ctx.close()


@pytest.mark.parametrize("B", [256, 130])
def test_D_at_headline_batch(fg, B):
    import torch_ref as R
    from face_generator_b200.lib import NET_D
    C = 3
    case = PU.make_case(B, C, seed=3000 + B)
    rng = np.random.default_rng(B + 1)
    img = rng.random((B, C, 32, 32)).astype(np.float32)
    dout = rng.standard_normal(B).astype(np.float32)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_params(NET_D, case["PD"])
    out = ctx.D_forward(img, masks=case["masks_D"])
    d_pos = {}
    for i, (H, Cc) in enumerate(((32, 64), (16, 128), (8, 256), (4, 512))):
        d_pos["z%d" % (i + 1)] = nchw(ctx.debug_tensor("D.z%d" % (i + 1)), B, H, H, Cc) > 0
    for n in ("zl1", "zl2"):
        d_pos[n] = dev(ctx.debug_tensor("D." + n).reshape(B, 512)) > 0
    counts = {}
    P = dev(case["PD"]).requires_grad_(True)
    x = dev(img).requires_grad_(True)
    ref_out = R.D_forward(P, x, dev(case["masks_D"]), C, branch=kink_branch(d_pos, counts))
    assert rel(out, ref_out.detach()) < TOL
    ref_out.backward(dev(dout))
    ctx.zero_grads(NET_D)
    dimg = ctx.D_backward(dout)
    gD = ctx.get_grads(NET_D)
    ctx.close()
    assert rel(dimg, x.grad) < TOL
    ref = P.grad.cpu().numpy()
    for k, (o, s) in O.D_layout(C).items():
        n = int(np.prod(s))
        tol = 3 * TOL if (k[0] == "a" and k[1:].isdigit()) else TOL
        assert PU.relerr(gD[o:o + n], ref[o:o + n]) < tol, (k, PU.relerr(gD[o:o + n], ref[o:o + n]), counts)


@pytest.mark.parametrize("N,Cin,H,Cout", [(256, 64, 16, 128), (256, 128, 8, 256), (256, 256, 4, 512),
                                          (130, 64, 16, 128), (130, 256, 4, 512)])
def test_D_conv_launches_at_headline_batch(fg, N, Cin, H, Cout):
    """D.C2-C4 (models.lua:390,395,400) forward / dgrad / wgrad launches at batch 256 and 130 through the L-op ABI
    (same kernels and tile heuristics as inside the net) against fp64."""
    from face_generator_b200.lib import _ptr
    F = torch.nn.functional
    rng = np.random.default_rng(N + Cin)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    x, w, b = f(rng.standard_normal((N, Cin, H, H))), f(rng.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cin * 9)), f(rng.standard_normal(Cout))
    dy = f(rng.standard_normal((N, Cout, H, H)))
    ctx = fg.Context(0, max_batch=8, channels=3)
    lib, h = ctx.lib, ctx.h
    y, dx, dw, db = np.empty((N, Cout, H, H), np.float32), np.empty_like(x), np.zeros_like(w), np.zeros_like(b)
    assert lib.fg_conv2d_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, H, H, Cout, 3) == 0, lib.fg_last_error()
    assert lib.fg_conv2d_backward_data(h, _ptr(dy), _ptr(w), _ptr(dx), N, Cin, H, H, Cout, 3) == 0, lib.fg_last_error()
    assert lib.fg_conv2d_backward_filter(h, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), N, Cin, H, H, Cout, 3) == 0, lib.fg_last_error()
    ctx.close()
    xt, wt, dyt = dev(x), dev(w), dev(dy)
    assert rel(y, F.conv2d(xt, wt, dev(b), padding=1)) < KTOL
    assert rel(dx, torch.nn.grad.conv2d_input(xt.shape, wt, dyt, padding=1)) < KTOL
    assert rel(dw, torch.nn.grad.conv2d_weight(xt, wt.shape, dyt, padding=1)) < KTOL
    assert rel(db, dyt.sum((0, 2, 3))) < TOL


@pytest.mark.parametrize("init", ["smooth", "trained"])
def test_full_train_step_at_headline_batch_vs_oracle(fg, init):
    """One fg_train_step at batch 256 (configs[1]) against O.f64.train_iteration: losses, confusion counts,
    post-clamp gradients, Adam moments at 1e-4 ("trained": real PReLU slopes with the kink override)."""
    import test_gpu_parity as TP
    TP._train_step_matches_oracle(fg, 3, 256, init, 2, 4000, max_batch=256)


@pytest.mark.parametrize("N,Cin,Cout", [(256, 128, 3), (130, 128, 3), (5, 128, 1), (256, 3, 64), (130, 3, 128), (6, 1, 64),
                                        (256, 64, 3), (7, 64, 1), (256, 3, 128), (3, 4, 64)])
def test_edge_conv_launches(fg, N, Cin, Cout):
    """the 3-channel-side 3x3 convolutions (G.C3: models.lua:73, D.C1: models.lua:385) in isolation through the L-op
    ABI: forward of shape Cin -> Cout and its dgrad (a Cout -> Cin convolution) = the "reduce" and "expand" kernels
    of k_conv_edge.cu, incl. the headline batch (TMA double buffering over ~7 strips per SM) and odd batches."""
    from face_generator_b200.lib import _ptr
    F = torch.nn.functional
    rng = np.random.default_rng(N + Cin + Cout)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    x, w, b = f(rng.standard_normal((N, Cin, 32, 32))), f(rng.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cin * 9)), f(rng.standard_normal(Cout))
    dy = f(rng.standard_normal((N, Cout, 32, 32)))
    ctx = fg.Context(0, max_batch=8, channels=3)
    lib, h = ctx.lib, ctx.h
    y, dx = np.empty((N, Cout, 32, 32), np.float32), np.empty_like(x)
    assert lib.fg_conv2d_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, 32, 32, Cout, 3) == 0, lib.fg_last_error()
    assert lib.fg_conv2d_backward_data(h, _ptr(dy), _ptr(w), _ptr(dx), N, Cin, 32, 32, Cout, 3) == 0, lib.fg_last_error()
    # the round-1 kernels as a second opinion on the same inputs
    ctx.set_option("edge_impl", 0)
    y0 = np.empty_like(y)
    assert lib.fg_conv2d_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y0), N, Cin, 32, 32, Cout, 3) == 0, lib.fg_last_error()
    ctx.close()
    xt, wt, dyt = dev(x), dev(w), dev(dy)
    assert rel(y, F.conv2d(xt, wt, dev(b), padding=1)) < KTOL
    assert rel(dx, torch.nn.grad.conv2d_input(xt.shape, wt, dyt, padding=1)) < KTOL
    assert rel(y0, y) < KTOL
