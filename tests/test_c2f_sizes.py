"""CPU: the coarse-to-fine nets at fine sizes 16 and 64 (train_c2f.lua --fineSize), the oracle against an independent
PyTorch-CPU autograd restatement in float64, and the sized C entry points against the oracle's layouts.

At fine size S, G is unchanged in parameters and runs at S x S; D's convolutions run at S and S/2 and its Linear
reads View(256*(S/4)^2), so D's parameter count moves by 512 * (256*(S/4)^2 - 16384) from the 32x32 nets."""
import numpy as np
import pytest
import torch

import c2f_sized_utils as SU
from oracle import oracle_c2f as OC
from oracle import oracle_c2f_sized as OS
import torch_ref as R
import torch_ref_c2f as RC

torch.set_num_threads(8)

SIZES = [16, 64]
HYPER = dict(lr_D=1e-3, lr_G=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, D_L1=1e-7, D_L2=0.0, G_L1=0.0, G_L2=0.0,
             D_clamp=1.0, G_clamp=5.0)


def rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.abs(a - b).max() / (np.abs(b).max() + 1e-300)


def normwise(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-300)


def test_oracle_layouts_at_each_size():
    for S, nD, mask in ((16, 2505926, 4608), (32, 8797382, 16896), (64, 33963206, 66048)):
        assert OC.G_param_count(3) == 1101319
        assert OS.D_param_count(3, S) == nD == 8797382 + 512 * (256 * (S // 4) ** 2 - 16384)
        assert OS.mask_per_sample(S) == mask == 256 * (S // 4) ** 2 + 512
        lay = OS.D_layout(3, S)
        assert lay["L1W"][1] == (512, 256 * (S // 4) ** 2)
        assert sum(int(np.prod(s)) for _, s in lay.values()) == nD


def test_library_sized_counts_match_oracle():
    from face_generator_b200.lib import NET_D, NET_G, c2f_mask_per_sample, load_library
    from face_generator_b200 import layouts as LY
    lib = load_library()
    for S in (16, 32, 64):
        for C in (1, 3):
            assert lib.fg_c2f_param_count_sized(NET_G, C, S) == OC.G_param_count(C)
            assert lib.fg_c2f_param_count_sized(NET_D, C, S) == OS.D_param_count(C, S) == LY.c2f_D_layout(C, S)[1]
        assert lib.fg_c2f_mask_per_sample_sized(S) == OS.mask_per_sample(S) == c2f_mask_per_sample(S)
    assert lib.fg_c2f_param_count_sized(NET_D, 3, 16) == 2505926
    assert lib.fg_c2f_param_count_sized(NET_D, 3, 64) == 33963206
    # the unsized entry points are the 32x32 case
    assert lib.fg_c2f_param_count_sized(NET_D, 3, 32) == lib.fg_c2f_param_count(NET_D, 3)
    assert lib.fg_c2f_mask_per_sample_sized(32) == lib.fg_c2f_mask_per_sample()
    for S in (0, 8, 24, 48, 128, -32):
        assert lib.fg_c2f_param_count_sized(NET_G, 3, S) == -1
        assert lib.fg_c2f_param_count_sized(NET_D, 3, S) == -1
        assert lib.fg_c2f_mask_per_sample_sized(S) == -1


@pytest.mark.parametrize("S", SIZES)
def test_G_fwd_bwd_matches_torch(S):
    rng = np.random.default_rng(300 + S)
    B, C = 2, 3
    P = RC.trained_like_G(C, rng)
    noise = rng.uniform(-1, 1, (B, 1, S, S))
    _, cond = SU.make_pairs(B, C, rng, S)
    dout = rng.standard_normal((B, C, S, S))
    g = OS.f64.G(S)
    out = g.forward(P, noise, cond)
    dP = g.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    out_t = RC.G_forward(Pt, torch.tensor(noise), torch.tensor(cond), C)
    out_t.backward(torch.tensor(dout))
    assert out.shape == (B, C, S, S)
    assert normwise(out, out_t.detach().numpy()) < 1e-10
    gt = Pt.grad.numpy()
    for k, (o, s) in OC.G_layout(C).items():
        n = int(np.prod(s))
        assert normwise(dP[o:o + n], gt[o:o + n]) < 1e-10, k


@pytest.mark.parametrize("S", SIZES)
def test_D_fwd_bwd_matches_torch(S):
    rng = np.random.default_rng(400 + S)
    B, C = 4, 3
    P = SU.trained_like_D(C, rng, S)
    diff, cond = SU.make_pairs(B, C, rng, S)
    masks = SU.make_masks(B, rng, S)
    dout = rng.standard_normal(B)
    d = OS.f64.D(S)
    out = d.forward(P, diff, cond, masks)
    dP, dd = d.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    dt = torch.tensor(diff, requires_grad=True)
    out_t = SU.D_forward(Pt, dt, torch.tensor(cond), torch.tensor(masks), C, fine_size=S)
    out_t.backward(torch.tensor(dout))
    assert normwise(out, out_t.detach().numpy()) < 1e-10
    gt = Pt.grad.numpy()
    for k, (o, s) in OS.D_layout(C, S).items():
        n = int(np.prod(s))
        assert normwise(dP[o:o + n], gt[o:o + n]) < 1e-10, k
    assert dd.shape == (B, C, S, S)
    assert normwise(dd, dt.grad.numpy()) < 1e-10


@pytest.mark.parametrize("S", SIZES)
def test_train_iteration_matches_torch(S):
    """one adversarial_c2f.lua loop body at batch 4 with the script's defaults (D_L1 = 1e-7 active)"""
    rng = np.random.default_rng(90 + S)
    B, C = 4, 3
    PD, PG = SU.trained_like_D(C, rng, S), RC.trained_like_G(C, rng)
    real_diff, cond_real = SU.make_pairs(B // 2, C, rng, S)
    _, cond_fake = SU.make_pairs(B // 2, C, rng, S)
    condD = np.concatenate([cond_real, cond_fake])
    _, condG = SU.make_pairs(B, C, rng, S)
    nD, nG = rng.uniform(-1, 1, (B // 2, 1, S, S)), rng.uniform(-1, 1, (B, 1, S, S))
    mD, mG = SU.make_masks(B, rng, S), SU.make_masks(B, rng, S)
    st = dict(PD=PD.copy(), PG=PG.copy(), mD=np.zeros_like(PD), vD=np.zeros_like(PD), mG=np.zeros_like(PG),
              vG=np.zeros_like(PG), tD=0, tG=0)
    res = OS.f64.train_iteration(S, B, C, HYPER, real_diff, condD, nD, condG, nG, mD, mG, st)
    PDt = torch.tensor(PD, requires_grad=True)
    PGt = torch.tensor(PG, requires_grad=True)
    with torch.no_grad():
        fake = RC.G_forward(PGt, torch.tensor(nD), torch.tensor(cond_fake), C)
    inputs = torch.cat([torch.tensor(real_diff), fake])
    targets = torch.tensor([1.0] * (B // 2) + [0.0] * (B // 2))
    out = SU.D_forward(PDt, inputs, torch.tensor(condD), torch.tensor(mD), C, fine_size=S)
    out.backward(R.bce_grad(out.detach(), targets))
    lossD = float(R.bce(out.detach(), targets)) + 1e-7 * float(PDt.detach().abs().sum())
    gD = np.clip(PDt.grad.numpy() + 1e-7 * np.sign(PD), -1, 1)
    assert abs(res["lossD"] - lossD) < 1e-10
    assert normwise(res["gradD"], gD) < 1e-10
    assert normwise(res["fake"], fake.numpy()) < 1e-10
    PD1 = PD - 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9) * (0.1 * gD) / (np.sqrt(0.001 * gD * gD) + 1e-8)
    assert normwise(st["PD"], PD1) < 1e-10
    PD1t = torch.tensor(st["PD"], requires_grad=True)
    diff = RC.G_forward(PGt, torch.tensor(nG), torch.tensor(condG), C)
    out = SU.D_forward(PD1t, diff, torch.tensor(condG), torch.tensor(mG), C, fine_size=S)
    ones = torch.ones(B, dtype=torch.float64)
    out.backward(R.bce_grad(out.detach(), ones))
    gG = np.clip(PGt.grad.numpy(), -5, 5)
    assert abs(res["lossG"] - float(R.bce(out.detach(), ones))) < 1e-10
    assert normwise(res["gradG"], gG) < 1e-10
    assert st["tD"] == 1 and st["tG"] == 1 and res["conf"].sum() == B


def test_sized_oracle_at_32_is_the_fixed_size_oracle():
    """the restatement with a runtime fine size, at 32, is the 32x32 restatement: one iteration agrees to float64
    rounding (the fixed-size loops have compile-time bounds, so the compiler may order a few sums differently)"""
    import c2f_utils as CU
    case = CU.make_case(4, 3, seed=12)
    a = CU.oracle_iteration(case, 4, 3)
    b = SU.oracle_iteration(case, 4, 3, 32)
    for k in ("gradD", "gradG", "fake", "outD"):
        assert rel(b[k], a[k]) < 1e-13, k
    np.testing.assert_array_equal(a["conf"], b["conf"])
    assert abs(a["lossD"] - b["lossD"]) < 1e-13 and abs(a["lossG"] - b["lossG"]) < 1e-13
    for k in ("PD", "PG", "mD", "vD", "mG", "vG"):
        assert rel(b["state"][k], a["state"][k]) < 1e-13, k
    assert OS.D_layout(3, 32) == OC.D_layout(3) and OS.mask_per_sample(32) == OC.MASK_PER_SAMPLE


def test_python_surfaces_default_to_32():
    from face_generator_b200 import adversarial_c2f as A
    from face_generator_b200 import layouts as LY
    rng = np.random.default_rng(0)
    assert A.create_noise_inputs(2, rng).shape == (2, 1, 32, 32)
    assert A.create_noise_inputs(2, rng, 64).shape == (2, 1, 64, 64)
    assert LY.c2f_D_layout(3) == LY.c2f_D_layout(3, 32)
    diff, coarse = LY.c2f_pairs(2, 3, rng, 16)
    assert diff.shape == coarse.shape == (2, 3, 16, 16)
