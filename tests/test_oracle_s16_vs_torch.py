"""CPU: the --scale 16 nets of the oracle (models.lua:26-51 create_G_decoder_upsampling16, :279-316 create_D16_d with
its stride-2 convolutions and ConcatTable/JoinTable) against PyTorch-CPU autograd in fp64 (tests/torch_ref_s16.py,
the checker tests/test_gpu_c2f_s16_headline.py holds the CUDA path to at batch 256)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle_s16 as OS
from torch_ref_c2f import trained_like
from torch_ref_s16 import torch_D16, torch_G16

torch.set_num_threads(8)


def rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.abs(a - b).max() / (np.abs(b).max() + 1e-300)


@pytest.mark.parametrize("stride,pad,H,k", [(2, 1, 8, 3), (2, 1, 5, 3), (1, 1, 6, 3), (2, 2, 9, 5), (3, 0, 10, 3)])
def test_strided_conv_matches_torch(stride, pad, H, k):
    rng = np.random.default_rng(50 + stride + H)
    x, w, b = rng.standard_normal((2, 3, H, H + 1)), rng.standard_normal((4, 3, k, k)), rng.standard_normal(4)
    y = OS.f64.convs_fwd(x, w, b, stride, pad)
    xt, wt, bt = (torch.tensor(v, requires_grad=True) for v in (x, w, b))
    yt = F.conv2d(xt, wt, bt, stride=stride, padding=pad)
    assert y.shape == tuple(yt.shape) and rel(y, yt.detach().numpy()) < 1e-12
    dy = rng.standard_normal(y.shape)
    yt.backward(torch.tensor(dy))
    dx, dw, db = OS.f64.convs_bwd(x, w, dy, stride, pad)
    assert rel(dx, xt.grad.numpy()) < 1e-12 and rel(dw, wt.grad.numpy()) < 1e-12 and rel(db, bt.grad.numpy()) < 1e-12


def test_param_counts():
    # G16: the 32px generator minus 3/4 of its first Linear; D16_d from the layer list of models.lua:279-316
    assert OS.G_param_count(3) == 2470406 - 6144 * 101
    assert OS.D_param_count(3) == sum(int(np.prod(s)) for _, s in OS.D_layout(3).values())


@pytest.mark.parametrize("C", [3, 1])
def test_G16_fwd_bwd_matches_torch(C):
    rng = np.random.default_rng(60 + C)
    B = 4
    P = trained_like(OS.G_layout(C), OS.G_param_count(C), rng, gain=1.0)
    for k in ("g1", "g2"):
        o, s = OS.G_layout(C)[k]
        P[o:o + s[0]] = rng.uniform(0.5, 1.5, s[0])
    noise = rng.uniform(-1, 1, (B, 100))
    dout = rng.standard_normal((B, C, 16, 16))
    g = OS.f64.G()
    out = g.forward(P, noise, C)
    dP = g.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    out_t = torch_G16(Pt, torch.tensor(noise), C)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-11
    gt = Pt.grad.numpy()
    for k, (o, s) in OS.G_layout(C).items():
        n = int(np.prod(s))
        if k in ("C1b", "C2b"):  # bias in front of BatchNorm: analytically zero, rounding noise only
            assert np.abs(dP[o:o + n]).max() < 1e-9 * np.abs(gt).max()
            continue
        assert rel(dP[o:o + n], gt[o:o + n]) < 1e-8, k


def test_G16_running_statistics_match_torch():
    """the BatchNorm running statistics of two training-mode forwards (the D and the G step of one iteration)"""
    import s16_utils as SU
    rng = np.random.default_rng(64)
    C = 3
    P = trained_like(OS.G_layout(C), OS.G_param_count(C), rng, gain=1.0)
    bn = SU.bn_init()
    running = torch.tensor(bn)
    for B in (3, 5):
        noise = rng.uniform(-1, 1, (B, 100))
        OS.f64.G().forward(P, noise, C, bn)
        torch_G16(torch.tensor(P), torch.tensor(noise), C, running=running)
    assert rel(bn, running.numpy()) < 1e-12


@pytest.mark.parametrize("C", [3, 1])
def test_D16_fwd_bwd_matches_torch(C):
    rng = np.random.default_rng(70 + C)
    B = 3
    P = trained_like(OS.D_layout(C), OS.D_param_count(C), rng, gain=1.0)
    img = rng.random((B, C, 16, 16))
    masks = (rng.random((B, OS.MASK_PER_SAMPLE)) < 0.5).astype(np.float64)
    dout = rng.standard_normal(B)
    d = OS.f64.D()
    out = d.forward(P, img, masks)
    dP, dimg = d.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    it = torch.tensor(img, requires_grad=True)
    out_t = torch_D16(Pt, it, torch.tensor(masks), C)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-12
    gt = Pt.grad.numpy()
    for k, (o, s) in OS.D_layout(C).items():
        n = int(np.prod(s))
        assert rel(dP[o:o + n], gt[o:o + n]) < 1e-9, k
    assert rel(dimg, it.grad.numpy()) < 1e-9  # ConcatTable: both branches contribute to the input gradient


def test_s16_iteration_composition_matches_torch():
    """tests/s16_utils.oracle_iteration (the checker of fg_s16_train_step) against the same adversarial.lua:240-288
    iteration written with PyTorch autograd in fp64: BCE (2015 Lua eps form), L2 penalty -> clamp, the D step's Adam
    update feeding the G step, D's weight gradients discarded in the G step."""
    import s16_utils as SU
    B, C = 8, 3
    case = SU.make_case(B, C, seed=77, init="near")
    hp = SU.HYPER
    ref = SU.oracle_iteration(case, B, C)
    t64 = lambda a: torch.tensor(np.asarray(a, np.float64))

    def bce(out, target):  # nn.BCECriterion of the 2015 Torch: -(t log(x+eps) + (1-t) log(1-x+eps)), eps = 1e-12, mean
        eps = 1e-12
        return -(target * torch.log(out + eps) + (1 - target) * torch.log(1 - out + eps)).mean()

    def clamp_pen(P, g, l1_loss, l1_grad, l2, c):
        g = g + l1_grad * torch.sign(P) + l2 * P
        return g.clamp(-c, c), l1_loss * P.abs().sum() + 0.5 * l2 * (P * P).sum()

    PG, PD = t64(case["PG"]).requires_grad_(True), t64(case["PD"]).requires_grad_(True)
    # ---- D step ----
    with torch.no_grad():
        fake = torch_G16(PG, t64(case["noise_D"]), C)
    assert rel(ref["fake"], fake.numpy()) < 1e-10
    x = torch.cat([t64(case["real"]), fake])
    tg = torch.cat([torch.ones(B // 2, dtype=torch.float64), torch.zeros(B // 2, dtype=torch.float64)])
    out = torch_D16(PD, x, t64(case["masks_D"]), C)
    lossD = bce(out, tg)
    gD, = torch.autograd.grad(lossD, PD)
    gD, pen = clamp_pen(PD.detach(), gD, hp["D_L1"], hp["D_L1"], hp["D_L2"], hp["D_clamp"])
    assert abs(float((lossD + pen).detach()) - ref["lossD"]) < 1e-9 * max(1.0, abs(ref["lossD"]))
    assert rel(ref["gradD"], gD.numpy()) < 1e-8
    # interruptableAdam at t = 1 (interruptable_optimizers.lua:49-94): m = (1-b1) g, v = (1-b2) g^2
    b1, b2, eps, lr = hp["beta1"], hp["beta2"], hp["eps"], hp["lr_D"]
    m, v = (1 - b1) * gD, (1 - b2) * gD * gD
    step = lr * np.sqrt(1 - b2) / (1 - b1)
    PD1 = (PD.detach() - step * m / (v.sqrt() + eps)).requires_grad_(True)
    assert rel(ref["PD"], PD1.detach().numpy()) < 1e-10
    # ---- G step ----
    img = torch_G16(PG, t64(case["noise_G"]), C)
    outG = torch_D16(PD1, img, t64(case["masks_G"]), C)
    lossG = bce(outG, torch.ones(B, dtype=torch.float64))
    gG, = torch.autograd.grad(lossG, PG)
    gG, penG = clamp_pen(PG.detach(), gG, hp["G_L1"], hp["G_L2"], hp["G_L2"], hp["G_clamp"])  # the :223 quirk
    assert abs(float((lossG + penG).detach()) - ref["lossG"]) < 1e-9 * max(1.0, abs(ref["lossG"]))
    LG = OS.G_layout(C)
    scale = np.abs(ref["gradG"]).max()
    for k, (o, s) in LG.items():
        n = int(np.prod(s))
        if k in ("C1b", "C2b"):
            assert np.abs(ref["gradG"][o:o + n]).max() < 1e-9 * scale
            continue
        assert rel(ref["gradG"][o:o + n], gG.numpy()[o:o + n]) < 1e-7, k


@pytest.mark.parametrize("factor", [1, 2, 3])
def test_scu_is_the_wide_convolution_under_a_view(factor):
    """layers/cudnnSpatialConvolutionUpsample.lua:14-58 restated with torch: parent conv to nOut*f*f planes, output
    .view(N, nOut, h*f, w*f), gradOutput viewed back.  The oracle's convolution + numpy reshape (what
    tests/test_gpu_s16.py holds fg_scu_* to) gives the same forward values and gradients."""
    from oracle import oracle as O
    rng = np.random.default_rng(90 + factor)
    N, Cin, nOut, k, H = 2, 5, 3, 3, 4
    planes = nOut * factor * factor
    x, w, b = rng.standard_normal((N, Cin, H, H)), rng.standard_normal((planes, Cin, k, k)), rng.standard_normal(planes)
    xt, wt, bt = (torch.tensor(v, requires_grad=True) for v in (x, w, b))
    yt = F.conv2d(xt, wt, bt, padding=k // 2).view(N, nOut, H * factor, H * factor)   # updateOutput :18-30
    y = O.f64.conv_fwd(x, w, b).reshape(N, nOut, H * factor, H * factor)
    assert rel(y, yt.detach().numpy()) < 1e-12
    dy = rng.standard_normal(y.shape)
    yt.backward(torch.tensor(dy))                                                    # autograd views gradOutput back (:32-58)
    dx, dw, db = O.f64.conv_bwd(x, w, dy.reshape(N, planes, H, H))
    assert rel(dx, xt.grad.numpy()) < 1e-12 and rel(dw, wt.grad.numpy()) < 1e-12 and rel(db, bt.grad.numpy()) < 1e-12
