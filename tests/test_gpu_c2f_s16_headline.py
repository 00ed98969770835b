"""The coarse-to-fine (fg_c2f_*) and --scale 16 (fg_s16_*) nets at the batch size bench.py measures them at (256) and
at a ragged batch (130), against float64 PyTorch on the same GPU -- the counterpart of tests/test_gpu_headline.py.

These nets put shapes on the tensor cores that the 32x32 nets do not have: c2f G.c5 (256 -> C, 7x7: padded forward +
bias compaction, weight gradient with swapped roles), c2f G.c2 / D.c2 (64 -> 64: weight gradient on a zero-padded dY),
c2f D.L1 (16384 -> 512 with permuted columns; at B = 130 its second 128-row tile holds 2 samples), s16 G.C1 (8 samples
per box at a 4x4 low-res side; at B = 130 the last box is 2/8 full and the BatchNorm partials come from the conv
epilogue), s16 D.c3 / D.c4 (stride 2 as stride 1 + subsampling), the permuted-column Linears of s16 D.  At B = 256 the
persistent kernels run several tiles per CTA and split-K runs long: paths batch 4-16 never reach.

The checkers are tests/torch_ref_c2f.py and tests/torch_ref_s16.py, pinned to the C++ oracle on the CPU by
tests/test_oracle_{c2f,s16}_vs_torch.py.  Three kinds of checks, each for mma_f16 = 1 (3xFP16 operands) and 0 (3xTF32):
 * every forward launch in ISOLATION at 1e-5: the layer's output against F.conv2d / F.linear applied to the CUDA
   path's own input (read through fg_*_debug_tensor), so errors do not accumulate; s16 G's BatchNorm statistics
   against the float64 statistics of the CUDA G.z1 / G.z2;
 * the whole net, forward and backward, at 1e-4 per parameter tensor plus the input gradients.  Where a decision is
   ambiguous at fp32 rounding -- a PReLU pre-activation within KINK_MARGIN*max of 0, a max-pool window whose top two
   candidates lie within KINK_MARGIN*max of each other -- the checker takes the CUDA path's decision (first max wins,
   like the kernel), everywhere else its own; the ambiguous sets are asserted to stay tiny;
 * one full train step per net at B = 256 against a float64 composition of the iteration (losses, confusion counts,
   both clamped gradients = Adam's m / (1 - beta1) at t = 1, s16's BatchNorm running state), the D step's decisions
   taken from the "Dstep.*" tensors (option "debug_keep"), the G step's from the final ones.
s16 G also runs with conv_impl = 1 (the dense 25-tap forward of its upsampled 5x5 layers).
"""
import numpy as np
import pytest

import c2f_utils as CU
import parity_utils as PU
import s16_utils as SU
from oracle import oracle_c2f as OC
from oracle import oracle_s16 as OS
from test_gpu_headline import dev, kink_branch, nchw, rel

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = torch.nn.functional
TOL = 1e-4   # whole net (BASELINE.json north_star)
KTOL = 1e-5  # one launch against fp64 on identical inputs
C = 3


def f32(t):
    return t.to(torch.float32)


def prelu32(z, a):
    """the CUDA path's PReLU output (prelu_fwd_kernel: v > 0 ? v : a * v in fp32) of its own pre-activation"""
    return torch.where(z > 0, z, (f32(a) * f32(z)).double())


def bn_prelu32(z, mean, istd, g, be, a):
    """bn_prelu_apply_kernel (k_elem.cu): u = fma(gamma, fl((z - mean) * istd), beta), then PReLU, in fp32"""
    v = lambda t: t.view(1, -1, 1, 1)
    t = f32(f32(f32(z) - f32(v(mean))) * f32(v(istd))).double()
    u = f32(v(g) * t + v(be)).double()
    return u, prelu32(u, a)


def first_max(win):
    """index of the first maximum of every 2x2 window (row-major), as the max-pool kernel picks it"""
    return (win == win.max(-1, keepdim=True).values).to(torch.float32).argmax(-1)


def windows(x):
    B, Cc, H, W = x.shape
    return x.reshape(B, Cc, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, Cc, H // 2, W // 2, 4)


def pool_route(gpu_idx, counts, margin=PU.KINK_MARGIN):
    """route hook of torch_ref_c2f.maxpool2: own argmax except where the top two candidates of a window lie within
    margin * max|x| of each other (then the CUDA path's first-max-wins pick)"""
    def route(name, win):
        top = win.topk(2, dim=-1).values
        amb = (top[..., 0] - top[..., 1]) < margin * win.abs().max()
        counts[name] = (int(amb.sum()), amb.numel())
        assert counts[name][0] <= max(8, PU.KINK_MAX_FRAC * amb.numel()), (name, counts[name])
        return torch.where(amb, gpu_idx[name], win.argmax(-1))
    return route


def within(errs, name, e, bar):
    errs[name] = e
    assert e < bar, (name, e, errs)


def check_tensors(got, ref, layout, errs, prefix, zero=()):
    """per parameter tensor at TOL; a shared PReLU slope is one heavily cancelling sum (3 TOL, as for the 32x32
    nets); `zero`: biases feeding a training-mode BatchNorm, analytically zero, compared with the scale of all
    gradients"""
    scale = np.abs(ref).max()
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        a, b = got[o:o + n], ref[o:o + n]
        if k in zero:
            e, bar = max(np.abs(a).max(), np.abs(b).max()) / scale, TOL
        else:
            e, bar = PU.relerr(a, b), (3 * TOL if k[0] == "a" else TOL)
        errs[prefix + k] = e
        assert e < bar, (prefix + k, e, errs)


def _ctx(B, f16, impl=2):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_option("conv_impl", impl)
    ctx.set_option("mma_f16", f16)
    return ctx


def _close(net, ctx):
    net.close()
    ctx.close()


PARAMS = [(256, 1), (256, 0), (130, 1), (130, 0)]
IDS = ["B%d-f16_%d" % p for p in PARAMS]


# ================================================================================================ coarse-to-fine
@pytest.fixture(scope="module", params=PARAMS, ids=IDS)
def c2f_G(request):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_G
    B, f16 = request.param
    case = CU.make_case(2 * B, C, seed=4100 + B + f16)
    noise, cond = case["noise_G"][:B], case["cond_G"][:B]
    dout = np.random.default_rng(B).standard_normal((B, C, 32, 32)).astype(np.float32)
    ctx = _ctx(B, f16)
    net = fg.C2f(ctx)
    net.set_params(NET_G, case["PG"])
    out = net.G_forward(noise, cond)
    T = {n: net.debug_tensor("G." + n) for n in ("x", "z1", "z2", "z3", "z4", "z5")}
    net.zero_grads(NET_G)
    net.G_backward(dout)
    r = dict(B=B, PG=case["PG"], noise=noise, cond=cond, dout=dout, out=out, T=T, grad=net.get_grads(NET_G))
    _close(net, ctx)
    return r


def test_c2f_G_forward_launches(c2f_G):
    import torch_ref as R
    B = c2f_G["B"]
    p = R._split(dev(c2f_G["PG"]), OC.G_layout(C))
    cout = (64, 64, 128, 256, C)
    x = nchw(c2f_G["T"]["x"], B, 32, 32, C + 1)
    assert torch.equal(x, torch.cat([dev(c2f_G["noise"]), dev(c2f_G["cond"])], 1))  # JoinTable
    errs = {}
    for i in range(5):
        z = nchw(c2f_G["T"]["z%d" % (i + 1)], B, 32, 32, cout[i])
        ref = F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=(1, 1, 2, 2, 3)[i])
        within(errs, "G.c%d" % (i + 1), rel(z, ref), KTOL)  # c5: padded forward + k_compact_bias
        if i < 4:
            x = prelu32(z, p["a%d" % (i + 1)])
    print("c2f G launches", errs)


def test_c2f_G_whole_net(c2f_G):
    import torch_ref_c2f as RC
    B = c2f_G["B"]
    cout = (64, 64, 128, 256)
    g_pos = {"z%d" % (i + 1): nchw(c2f_G["T"]["z%d" % (i + 1)], B, 32, 32, cout[i]) > 0 for i in range(4)}
    counts = {}
    P = dev(c2f_G["PG"]).requires_grad_(True)
    ref_out = RC.G_forward(P, dev(c2f_G["noise"]), dev(c2f_G["cond"]), C, branch=kink_branch(g_pos, counts))
    errs = {}
    within(errs, "out", rel(c2f_G["out"], ref_out.detach()), TOL)
    ref_out.backward(dev(c2f_G["dout"]))
    # G.c5's weight gradient runs with swapped roles, G.c2's on a zero-padded dY
    check_tensors(c2f_G["grad"], P.grad.cpu().numpy(), OC.G_layout(C), errs, "G.")
    print("c2f G whole net", errs, counts)


def _c2f_route_inputs(get, P, B):
    """the CUDA path's branch decisions and max-pool picks from its D pre-activations (get(name) -> flat NHWC)"""
    import torch_ref as R
    p = R._split(dev(P), OC.D_layout(C))
    shapes = ((32, 64), (32, 64), (16, 128), (16, 256))
    z = [nchw(get("z%d" % (i + 1)), B, H, H, Cc) for i, (H, Cc) in enumerate(shapes)]
    pos = {"z%d" % (i + 1): z[i] > 0 for i in range(4)}
    pos["zl1"] = dev(get("zl1").reshape(B, 512)) > 0
    idx = {"p2": first_max(windows(prelu32(z[1], p["a2"]))), "p4": first_max(windows(prelu32(z[3], p["a4"])))}
    return pos, idx


@pytest.fixture(scope="module", params=PARAMS, ids=IDS)
def c2f_D(request):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D
    B, f16 = request.param
    case = CU.make_case(2 * B, C, seed=4200 + B + f16)
    rng = np.random.default_rng(B + 7)
    diff, cond, masks = case["real_diff"], case["cond_D"][:B], case["masks_D"][:B]
    dout = rng.standard_normal(B).astype(np.float32)
    ctx = _ctx(B, f16)
    net = fg.C2f(ctx)
    net.set_params(NET_D, case["PD"])
    out = net.D_forward(diff, cond, masks=masks)
    T = {n: net.debug_tensor("D." + n) for n in ("x", "z1", "z2", "z3", "z4", "p2", "p4", "zl1", "logit")}
    net.zero_grads(NET_D)
    ddiff = net.D_backward(dout)
    r = dict(B=B, PD=case["PD"], diff=diff, cond=cond, masks=masks, dout=dout, out=out, T=T, ddiff=ddiff,
             grad=net.get_grads(NET_D))
    _close(net, ctx)
    return r


def test_c2f_D_forward_launches(c2f_D):
    import torch_ref as R
    B, T = c2f_D["B"], c2f_D["T"]
    p = R._split(dev(c2f_D["PD"]), OC.D_layout(C))
    m = dev(c2f_D["masks"])
    x = nchw(T["x"], B, 32, 32, C)
    assert torch.equal(x, f32(dev(c2f_D["diff"]) + dev(c2f_D["cond"])).double())  # CAddTable
    shapes = ((32, 64), (32, 64), (16, 128), (16, 256))
    errs = {}
    for i, (H, Cc) in enumerate(shapes):
        z = nchw(T["z%d" % (i + 1)], B, H, H, Cc)
        ref = F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=1)
        within(errs, "D.c%d" % (i + 1), rel(z, ref), KTOL)  # c2: 64 -> 64
        x = prelu32(z, p["a%d" % (i + 1)])
        if i in (1, 3):
            pooled = nchw(T["p%d" % (i + 1)], B, H // 2, H // 2, Cc)
            assert torch.equal(pooled, F.max_pool2d(x, 2, 2))
            x = pooled
    zl1 = dev(T["zl1"].reshape(B, 512))
    ref = F.linear(x.reshape(B, 16384) * m[:, :16384] * 2.0, p["L1W"], p["L1b"])  # View(16384) of [256][8][8]
    within(errs, "D.L1", rel(zl1, ref), KTOL)
    ref = F.linear(prelu32(zl1, p["a5"]) * m[:, 16384:] * 2.0, p["L2W"], p["L2b"]).reshape(B)
    within(errs, "D.L2", rel(dev(T["logit"]), ref), KTOL)
    print("c2f D launches", errs)


def test_c2f_D_whole_net(c2f_D):
    import torch_ref_c2f as RC
    B = c2f_D["B"]
    pos, idx = _c2f_route_inputs(lambda n: c2f_D["T"][n], c2f_D["PD"], B)
    counts = {}
    P = dev(c2f_D["PD"]).requires_grad_(True)
    x = dev(c2f_D["diff"]).requires_grad_(True)
    ref_out = RC.D_forward(P, x, dev(c2f_D["cond"]), dev(c2f_D["masks"]), C, branch=kink_branch(pos, counts),
                           route=pool_route(idx, counts))
    errs = {}
    within(errs, "out", rel(c2f_D["out"], ref_out.detach()), TOL)
    ref_out.backward(dev(c2f_D["dout"]))
    within(errs, "d(diff)", rel(c2f_D["ddiff"], x.grad), TOL)
    check_tensors(c2f_D["grad"], P.grad.cpu().numpy(), OC.D_layout(C), errs, "D.")
    print("c2f D whole net", errs, counts)


def bce(x, t):
    eps = 1e-12
    return -(t * torch.log(x + eps) + (1 - t) * torch.log(1 - x + eps)).mean()


def conf_of(out, Bh):
    conf = [0, 0, 0, 0]
    for i, o in enumerate(out.tolist()):
        conf[(0 if o > 0.5 else 1) + (0 if i < Bh else 2)] += 1
    return conf


def adam_t1(P, g, hp, lr):
    """interruptableAdam / optim.adam at t = 1 (m = (1-b1) g, v = (1-b2) g^2)"""
    b1, b2 = hp["beta1"], hp["beta2"]
    return P - lr * np.sqrt(1 - b2) / (1 - b1) * ((1 - b1) * g) / (np.sqrt((1 - b2) * g * g) + hp["eps"])


def check_losses_and_update(errs, st, out_D_gpu, out_D_ref, pen_D, out_G_gpu, out_G_ref, Bh, gD, PD, PDn, hp):
    B = 2 * Bh
    tD = torch.cat([torch.ones(Bh), torch.zeros(Bh)]).double().cuda()
    # D's outputs against the checker; the losses are the criterion on the CUDA path's own fp32 outputs
    # (near saturation the fp32 rounding of x is amplified by 1/(1-x): see test_gpu_parity)
    within(errs, "D step out", rel(out_D_gpu, out_D_ref), TOL)
    within(errs, "G step out", rel(out_G_gpu, out_G_ref), TOL)
    lossD = float(bce(dev(out_D_gpu), tD)) + pen_D
    lossG = float(bce(dev(out_G_gpu), torch.ones(B).double().cuda()))  # G_L1 = G_L2 = 0
    within(errs, "loss_D", abs(st["loss_D"] - lossD) / max(1.0, abs(lossD)), 1e-5)
    within(errs, "loss_G", abs(st["loss_G"] - lossG) / max(1.0, abs(lossG)), 1e-5)
    assert st["conf"] == conf_of(out_D_ref, Bh)
    assert st["t_D"] == 1 and st["t_G"] == 1 and st["trained_D"] == 1
    # Adam moved D by its own gradient (compared where the gradient is not rounding noise: |step| = lr at t = 1)
    big = np.abs(gD) > 1e-3 * np.abs(gD).max()
    within(errs, "PD after Adam", np.abs(PDn.astype(np.float64)[big] - adam_t1(PD.astype(np.float64), gD, hp, hp["lr_D"])[big]).max(),
           2e-5)


def test_c2f_train_step_at_256():
    """one fg_c2f_train_step (adversarial_c2f.lua:121-187, train_c2f.lua defaults: D_L1 = 1e-7) against its float64
    composition; the G step runs on the CUDA path's own post-Adam D parameters"""
    import face_generator_b200 as fg
    import torch_ref as R
    import torch_ref_c2f as RC
    from face_generator_b200.lib import NET_D, NET_G
    B, Bh, hp = 256, 128, CU.HYPER
    case = CU.make_case(B, C, seed=4300)
    ctx = _ctx(B, 1)
    ctx.set_option("debug_keep", 1)
    net = fg.C2f(ctx)
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    st = net.train_step(fg.hyper_default(**hp), B, case["real_diff"], case["cond_D"], case["noise_D"], case["cond_G"],
                        case["noise_G"], case["masks_D"], case["masks_G"])
    Dk = {n: net.debug_tensor("Dstep." + n) for n in ("z1", "z2", "z3", "z4", "zl1", "out")}
    Dg = {n: net.debug_tensor("D." + n) for n in ("z1", "z2", "z3", "z4", "zl1", "out")}
    Gg = {n: net.debug_tensor("G." + n) for n in ("z1", "z2", "z3", "z4")}
    mD, _, tD = net.get_adam_state(NET_D)
    mG, _, tG = net.get_adam_state(NET_G)
    PDn = net.get_params(NET_D)
    _close(net, ctx)
    assert tD == 1 and tG == 1
    # ---- D step ----
    PG = dev(case["PG"]).requires_grad_(True)
    PD = dev(case["PD"]).requires_grad_(True)
    with torch.no_grad():
        fake = RC.G_forward(PG, dev(case["noise_D"]), dev(case["cond_D"][Bh:]), C)
    counts = {}
    pos, idx = _c2f_route_inputs(lambda n: Dk[n], case["PD"], B)
    out = RC.D_forward(PD, torch.cat([dev(case["real_diff"]), fake]), dev(case["cond_D"]), dev(case["masks_D"]), C,
                       branch=kink_branch(pos, counts), route=pool_route(idx, counts))
    tgt = torch.cat([torch.ones(Bh), torch.zeros(Bh)]).double().cuda()
    out.backward(R.bce_grad(out.detach(), tgt))
    P0 = case["PD"].astype(np.float64)
    gD = np.clip(PD.grad.cpu().numpy() + hp["D_L1"] * np.sign(P0), -hp["D_clamp"], hp["D_clamp"])
    errs = {}
    check_tensors(mD / (1 - hp["beta1"]), gD, OC.D_layout(C), errs, "gradD.")
    # ---- G step, on the CUDA path's D parameters after its Adam step ----
    cout = (64, 64, 128, 256)
    g_pos = {"z%d" % (i + 1): nchw(Gg["z%d" % (i + 1)], B, 32, 32, cout[i]) > 0 for i in range(4)}
    pos, idx = _c2f_route_inputs(lambda n: Dg[n], PDn, B)
    gcounts, dcounts = {}, {}
    diff = RC.G_forward(PG, dev(case["noise_G"]), dev(case["cond_G"]), C, branch=kink_branch(g_pos, gcounts))
    outG = RC.D_forward(dev(PDn), diff, dev(case["cond_G"]), dev(case["masks_G"]), C, branch=kink_branch(pos, dcounts),
                        route=pool_route(idx, dcounts))
    outG.backward(R.bce_grad(outG.detach(), torch.ones(B).double().cuda()))
    gG = np.clip(PG.grad.cpu().numpy(), -hp["G_clamp"], hp["G_clamp"])
    check_tensors(mG / (1 - hp["beta1"]), gG, OC.G_layout(C), errs, "gradG.")
    check_losses_and_update(errs, st, Dk["out"], out.detach(), hp["D_L1"] * float(np.abs(P0).sum()), Dg["out"],
                            outG.detach(), Bh, gD, case["PD"], PDn, hp)
    print("c2f train step", errs, counts, gcounts, dcounts)


# ================================================================================================ --scale 16
S16_G_PARAMS = [(B, f16, 2) for B, f16 in PARAMS] + [(256, 1, 1), (130, 1, 1)]


def _bn_ref(z):
    """float64 batch statistics of the CUDA path's own conv output"""
    mean = z.mean((0, 2, 3))
    return mean, 1.0 / torch.sqrt(z.var((0, 2, 3), unbiased=False) + 1e-5)


@pytest.fixture(scope="module", params=S16_G_PARAMS, ids=["B%d-f16_%d-impl%d" % p for p in S16_G_PARAMS])
def s16_G(request):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_G
    B, f16, impl = request.param
    case = SU.make_case(2 * B, C, seed=4400 + B + f16 + 10 * impl, init="trained")
    noise = case["noise_G"][:B]
    dout = np.random.default_rng(B + 3).standard_normal((B, C, 16, 16)).astype(np.float32)
    ctx = _ctx(B, f16, impl)
    net = fg.S16(ctx)
    net.set_params(NET_G, case["PG"])
    img = net.G_forward(noise, training=True)
    T = {n: net.debug_tensor("G." + n) for n in ("z0", "z1", "z2", "z3", "bn_mean1", "bn_istd1", "bn_mean2", "bn_istd2")}
    net.zero_grads(NET_G)
    dn = net.G_backward(dout, want_dnoise=True)
    r = dict(B=B, PG=case["PG"], noise=noise, dout=dout, img=img, T=T, dnoise=dn, grad=net.get_grads(NET_G))
    _close(net, ctx)
    return r


def _s16_G_tensors(T, B):
    z = dict(z0=nchw(T["z0"], B, 4, 4, 128), z1=nchw(T["z1"], B, 8, 8, 256), z2=nchw(T["z2"], B, 16, 16, 128),
             z3=nchw(T["z3"], B, 16, 16, C))
    for k in ("bn_mean1", "bn_istd1", "bn_mean2", "bn_istd2"):
        z[k] = dev(T[k])
    return z


def test_s16_G_forward_launches(s16_G):
    import torch_ref as R
    B = s16_G["B"]
    p = R._split(dev(s16_G["PG"]), OS.G_layout(C))
    z = _s16_G_tensors(s16_G["T"], B)
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")
    ref = F.linear(dev(s16_G["noise"]), p["L1W"], p["L1b"]).view(B, 128, 4, 4)  # View(128,4,4): permuted rows
    errs = {}
    within(errs, "G.L1", rel(z["z0"], ref), KTOL)
    h = prelu32(z["z0"], p["a1"])
    for i, (zn, W, b, g, be, a) in enumerate((("z1", "C1W", "C1b", "g1", "be1", "a2"), ("z2", "C2W", "C2b", "g2", "be2", "a3"))):
        ref = F.conv2d(up(h), p[W], p[b], padding=2)  # upsampled 5x5: collapsed phases (impl 2) / dense 25 taps (impl 1)
        within(errs, "G.C%d" % (i + 1), rel(z[zn], ref), KTOL)
        # BatchNorm statistics (from the conv epilogue's per-box partials) against the CUDA output's own statistics;
        # the mean error in units of the standard deviation
        mean, istd = _bn_ref(z[zn])
        gm, gs = z["bn_mean%d" % (i + 1)], z["bn_istd%d" % (i + 1)]
        within(errs, "bn_mean%d" % (i + 1), float(((gm - mean).abs() * istd).max()), KTOL)
        within(errs, "bn_istd%d" % (i + 1), rel(gs, istd), KTOL)
        _, h = bn_prelu32(z[zn], gm, gs, p[g], p[be], p[a])
    within(errs, "G.C3", rel(z["z3"], F.conv2d(h, p["C3W"], p["C3b"], padding=1)), KTOL)
    print("s16 G launches", errs)


def _s16_g_pos(z, p):
    pos = {"z0": z["z0"] > 0}
    for i, (zn, g, be, a) in enumerate((("z1", "g1", "be1", "a2"), ("z2", "g2", "be2", "a3"))):
        u, _ = bn_prelu32(z[zn], z["bn_mean%d" % (i + 1)], z["bn_istd%d" % (i + 1)], p[g], p[be], p[a])
        pos["y%d" % (i + 1)] = u > 0
    return pos


def test_s16_G_whole_net(s16_G):
    import torch_ref as R
    import torch_ref_s16 as RS
    B = s16_G["B"]
    z = _s16_G_tensors(s16_G["T"], B)
    pos = _s16_g_pos(z, R._split(dev(s16_G["PG"]), OS.G_layout(C)))
    counts = {}
    P = dev(s16_G["PG"]).requires_grad_(True)
    nz = dev(s16_G["noise"]).requires_grad_(True)
    ref = RS.torch_G16(P, nz, C, branch=kink_branch(pos, counts))
    errs = {}
    within(errs, "img", rel(s16_G["img"], ref.detach()), TOL)
    ref.backward(dev(s16_G["dout"]))
    within(errs, "d(noise)", rel(s16_G["dnoise"], nz.grad), TOL)
    check_tensors(s16_G["grad"], P.grad.cpu().numpy(), OS.G_layout(C), errs, "G.", zero=("C1b", "C2b"))
    print("s16 G whole net", errs, counts)


def _s16_d_pos(get, B):
    shapes = dict(z1=(16, 128), z2=(16, 128), z3=(4, 512), z4=(2, 1024))
    pos = {k: nchw(get(k), B, H, H, Cc) > 0 for k, (H, Cc) in shapes.items()}
    for k, n in (("zf", 1024), ("ze1", 128), ("ze2", 128)):
        pos[k] = dev(get(k).reshape(B, n)) > 0
    return pos


@pytest.fixture(scope="module", params=PARAMS, ids=IDS)
def s16_D(request):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D
    B, f16 = request.param
    case = SU.make_case(2 * B, C, seed=4500 + B + f16, init="trained")
    rng = np.random.default_rng(B + 11)
    img = rng.random((B, C, 16, 16)).astype(np.float32)
    masks = case["masks_D"][:B]
    dout = rng.standard_normal(B).astype(np.float32)
    ctx = _ctx(B, f16)
    net = fg.S16(ctx)
    net.set_params(NET_D, case["PD"])
    out = net.D_forward(img, masks, training=True)
    T = {n: net.debug_tensor("D." + n) for n in ("z1", "z2", "z3", "z4", "p1", "zf", "ze1", "ze2", "logit")}
    net.zero_grads(NET_D)
    dimg = net.D_backward(dout, want_wgrad=True, want_dimg=True)
    r = dict(B=B, PD=case["PD"], img=img, masks=masks, dout=dout, out=out, T=T, dimg=dimg, grad=net.get_grads(NET_D))
    _close(net, ctx)
    return r


def test_s16_D_forward_launches(s16_D):
    import torch_ref as R
    B, T = s16_D["B"], s16_D["T"]
    p = R._split(dev(s16_D["PD"]), OS.D_layout(C))
    m, img = dev(s16_D["masks"]), dev(s16_D["img"])
    z1, z2 = nchw(T["z1"], B, 16, 16, 128), nchw(T["z2"], B, 16, 16, 128)
    errs = {}
    within(errs, "D.c1", rel(z1, F.conv2d(img, p["c1W"], p["c1b"], padding=1)), KTOL)
    within(errs, "D.c2", rel(z2, F.conv2d(prelu32(z1, p["a1"]), p["c2W"], p["c2b"], padding=1)), KTOL)
    p1 = nchw(T["p1"], B, 8, 8, 128)
    within(errs, "D.pool", rel(p1, F.avg_pool2d(prelu32(z2, p["a2"]), 2, 2)), KTOL)
    z3, z4 = nchw(T["z3"], B, 4, 4, 512), nchw(T["z4"], B, 2, 2, 1024)
    ref = F.conv2d(p1, p["c3W"], p["c3b"], stride=2, padding=1)  # stride 1 + subsample2 on the CUDA path
    within(errs, "D.c3", rel(z3, ref), KTOL)
    ref = F.conv2d(prelu32(z3, p["a3"]), p["c4W"], p["c4b"], stride=2, padding=1)  # 512 -> 1024 at 4x4
    within(errs, "D.c4", rel(z4, ref), KTOL)
    zf, ze1, ze2 = (dev(T[k].reshape(B, -1)) for k in ("zf", "ze1", "ze2"))
    ref = F.linear((prelu32(z4, p["a4"]) * m[:, :1024].reshape(B, 1024, 1, 1)).reshape(B, 4096), p["F1W"], p["F1b"])
    within(errs, "D.F1", rel(zf, ref), KTOL)  # View(4096) of [1024][2][2]: permuted columns
    ref = F.linear(img.reshape(B, -1), p["E1W"], p["E1b"])  # View(C*256) of the NCHW image, K = 256 C
    within(errs, "D.E1", rel(ze1, ref), KTOL)
    ref = F.linear(prelu32(ze1, p["ae1"]) * m[:, 1024:] * 2.0, p["E2W"], p["E2b"])
    within(errs, "D.E2", rel(ze2, ref), KTOL)
    ref = F.linear(torch.cat([prelu32(zf, p["af"]), prelu32(ze2, p["ae2"])], 1), p["JW"], p["Jb"]).reshape(B)
    within(errs, "D.J", rel(dev(T["logit"]), ref), KTOL)
    print("s16 D launches", errs)


def test_s16_D_whole_net(s16_D):
    import torch_ref_s16 as RS
    B = s16_D["B"]
    pos = _s16_d_pos(lambda k: s16_D["T"][k], B)
    counts = {}
    P = dev(s16_D["PD"]).requires_grad_(True)
    x = dev(s16_D["img"]).requires_grad_(True)
    ref = RS.torch_D16(P, x, dev(s16_D["masks"]), C, branch=kink_branch(pos, counts))
    errs = {}
    within(errs, "out", rel(s16_D["out"], ref.detach()), TOL)
    ref.backward(dev(s16_D["dout"]))
    within(errs, "d(img)", rel(s16_D["dimg"], x.grad), TOL)  # conv branch + dense branch
    check_tensors(s16_D["grad"], P.grad.cpu().numpy(), OS.D_layout(C), errs, "D.")
    print("s16 D whole net", errs, counts)


def test_s16_train_step_at_256():
    """one fg_s16_train_step (adversarial.lua:240-288 on the 16x16 nets, train.lua defaults: D_L2 = 1e-4) against its
    float64 composition (test_s16_iteration_composition_matches_torch), incl. the BatchNorm running state"""
    import face_generator_b200 as fg
    import torch_ref as R
    import torch_ref_s16 as RS
    from face_generator_b200.lib import NET_D, NET_G
    B, Bh, hp = 256, 128, SU.HYPER
    case = SU.make_case(B, C, seed=4600, init="trained")
    ctx = _ctx(B, 1)
    ctx.set_option("debug_keep", 1)
    net = fg.S16(ctx)
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    st = net.train_step(fg.hyper_default(**hp), B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"],
                        case["masks_G"])
    names = ("z1", "z2", "z3", "z4", "zf", "ze1", "ze2", "out")
    Dk = {n: net.debug_tensor("Dstep." + n) for n in names}
    Dg = {n: net.debug_tensor("D." + n) for n in names}
    Gg = _s16_G_tensors({n: net.debug_tensor("G." + n) for n in
                         ("z0", "z1", "z2", "z3", "bn_mean1", "bn_istd1", "bn_mean2", "bn_istd2")}, B)
    mD, _, tD = net.get_adam_state(NET_D)
    mG, _, tG = net.get_adam_state(NET_G)
    PDn, bn = net.get_params(NET_D), net.get_bn_state()
    _close(net, ctx)
    assert tD == 1 and tG == 1
    running = dev(SU.bn_init())
    # ---- D step ----
    PG = dev(case["PG"]).requires_grad_(True)
    PD = dev(case["PD"]).requires_grad_(True)
    with torch.no_grad():
        fake = RS.torch_G16(PG, dev(case["noise_D"]), C, running=running)
    counts = {}
    out = RS.torch_D16(PD, torch.cat([dev(case["real"]), fake]), dev(case["masks_D"]), C,
                       branch=kink_branch(_s16_d_pos(lambda k: Dk[k], B), counts))
    tgt = torch.cat([torch.ones(Bh), torch.zeros(Bh)]).double().cuda()
    out.backward(R.bce_grad(out.detach(), tgt))
    P0 = case["PD"].astype(np.float64)
    gD = np.clip(PD.grad.cpu().numpy() + hp["D_L1"] * np.sign(P0) + hp["D_L2"] * P0, -hp["D_clamp"], hp["D_clamp"])
    pen_D = hp["D_L1"] * float(np.abs(P0).sum()) + 0.5 * hp["D_L2"] * float((P0 * P0).sum())
    errs = {}
    check_tensors(mD / (1 - hp["beta1"]), gD, OS.D_layout(C), errs, "gradD.")
    # ---- G step, on the CUDA path's D parameters after its Adam step ----
    gcounts, dcounts = {}, {}
    img = RS.torch_G16(PG, dev(case["noise_G"]), C, branch=kink_branch(_s16_g_pos(Gg, R._split(dev(case["PG"]), OS.G_layout(C))),
                                                                       gcounts), running=running)
    outG = RS.torch_D16(dev(PDn), img, dev(case["masks_G"]), C, branch=kink_branch(_s16_d_pos(lambda k: Dg[k], B), dcounts))
    outG.backward(R.bce_grad(outG.detach(), torch.ones(B).double().cuda()))
    gG = np.clip(PG.grad.cpu().numpy(), -hp["G_clamp"], hp["G_clamp"])  # G_L1 = G_L2 = 0
    check_tensors(mG / (1 - hp["beta1"]), gG, OS.G_layout(C), errs, "gradG.", zero=("C1b", "C2b"))
    check_losses_and_update(errs, st, Dk["out"], out.detach(), pen_D, Dg["out"], outG.detach(), Bh, gD, case["PD"], PDn, hp)
    within(errs, "bn_state", rel(bn, running), TOL)  # two training-mode G forwards: B/2 (D step), then B
    print("s16 train step", errs, counts, gcounts, dcounts)
