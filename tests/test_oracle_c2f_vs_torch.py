"""CPU: the coarse-to-fine part of the oracle against an independent PyTorch-CPU autograd restatement (fp64).
BASELINE.json configs[3] (train_c2f.lua).  "Parity unpinned": the reference holds no vectors for this path."""
import numpy as np
import pytest
import torch

from oracle import oracle_c2f as OC
import torch_ref as R
import torch_ref_c2f as RC

torch.set_num_threads(8)


def rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.abs(a - b).max() / (np.abs(b).max() + 1e-300)


def test_param_counts():
    # SURVEY.md section 8a: 1 101 319 (G_d) and 8 797 382 (D_c) for colour
    assert OC.G_param_count(3) == 1101319
    assert OC.D_param_count(3) == 8797382
    assert OC.G_param_count(1) == 1101319 - 2 * 64 * 9 - 2 * (256 * 49 + 1)


def test_maxpool_first_max_wins():
    x = np.zeros((1, 1, 2, 4))
    x[0, 0] = [[1, 5, 2, 2], [5, 0, 2, 2]]  # ties: (0,1) vs (1,0) -> row-major first; all-equal -> (0,0)
    y, arg = OC.f64.maxpool2_fwd(x)
    assert y.ravel().tolist() == [5, 2] and arg.ravel().tolist() == [1, 0]
    dx = OC.f64.maxpool2_bwd(np.array([[[[7.0, 3.0]]]]), arg)
    assert dx[0, 0].tolist() == [[0, 7, 3, 0], [0, 0, 0, 0]]


def test_routed_restatement_matches_oracle():
    """D_forward with the branch / max-pool routing hooks making their own decisions (the hooks of the batch-256 GPU
    checks) is the same function as the oracle, values and gradients; forcing another window element moves the value"""
    rng = np.random.default_rng(45)
    B, C = 3, 3
    P = RC.trained_like_D(C, rng)
    diff, cond = RC.make_pairs(B, C, rng)
    masks = RC.make_masks(B, rng)
    dout = rng.standard_normal(B)
    d = OC.f64.D()
    out = d.forward(P, diff, cond, masks)
    dP, dd = d.backward(dout)
    own = lambda name, x: x > 0
    route = lambda name, win: win.argmax(-1)
    Pt = torch.tensor(P, requires_grad=True)
    dt = torch.tensor(diff, requires_grad=True)
    out_t = RC.D_forward(Pt, dt, torch.tensor(cond), torch.tensor(masks), C, branch=own, route=route)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-12
    assert rel(dP, Pt.grad.numpy()) < 1e-9 and rel(dd, dt.grad.numpy()) < 1e-9
    x = torch.tensor(rng.standard_normal((2, 4, 6, 8)))
    assert torch.equal(RC.maxpool2(x, route, "p"), torch.nn.functional.max_pool2d(x, 2, 2))
    assert (RC.maxpool2(x, lambda n, w: w.argmin(-1), "p") < RC.maxpool2(x)).all()


@pytest.mark.parametrize("C", [3, 1])
def test_G_fwd_bwd_matches_torch(C):
    rng = np.random.default_rng(30 + C)
    B = 3
    P = RC.trained_like_G(C, rng)
    noise = rng.uniform(-1, 1, (B, 1, 32, 32))
    _, cond = RC.make_pairs(B, C, rng)
    dout = rng.standard_normal((B, C, 32, 32))
    g = OC.f64.G()
    out = g.forward(P, noise, cond)
    dP = g.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    out_t = RC.G_forward(Pt, torch.tensor(noise), torch.tensor(cond), C)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-11
    gt = Pt.grad.numpy()
    for k, (o, s) in OC.G_layout(C).items():
        n = int(np.prod(s))
        assert rel(dP[o:o + n], gt[o:o + n]) < 1e-9, k


@pytest.mark.parametrize("C", [3, 1])
def test_D_fwd_bwd_matches_torch(C):
    rng = np.random.default_rng(40 + C)
    B = 4
    P = RC.trained_like_D(C, rng)
    diff, cond = RC.make_pairs(B, C, rng)
    masks = RC.make_masks(B, rng)
    dout = rng.standard_normal(B)
    d = OC.f64.D()
    out = d.forward(P, diff, cond, masks)
    dP, dd = d.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    dt = torch.tensor(diff, requires_grad=True)
    out_t = RC.D_forward(Pt, dt, torch.tensor(cond), torch.tensor(masks), C)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-12
    gt = Pt.grad.numpy()
    for k, (o, s) in OC.D_layout(C).items():
        n = int(np.prod(s))
        assert rel(dP[o:o + n], gt[o:o + n]) < 1e-9, k
    assert rel(dd, dt.grad.numpy()) < 1e-9
    # weight gradients are optional (G step): the input gradient must not depend on them
    d.forward(P, diff, cond, masks)
    _, dd2 = d.backward(dout, want_dP=False)
    assert np.array_equal(dd, dd2)


def test_train_iteration_matches_torch():
    """One adversarial_c2f.lua loop body with the script's defaults (D_L1 = 1e-7 active, train_c2f.lua:29)."""
    rng = np.random.default_rng(9)
    B, C = 4, 3
    hyper = dict(lr_D=1e-3, lr_G=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, D_L1=1e-7, D_L2=0.0, G_L1=0.0, G_L2=0.0,
                 D_clamp=1.0, G_clamp=5.0)
    PD, PG = RC.trained_like_D(C, rng), RC.trained_like_G(C, rng)
    real_diff, cond_real = RC.make_pairs(B // 2, C, rng)
    _, cond_fake = RC.make_pairs(B // 2, C, rng)
    condD = np.concatenate([cond_real, cond_fake])
    _, condG = RC.make_pairs(B, C, rng)
    nD, nG = rng.uniform(-1, 1, (B // 2, 1, 32, 32)), rng.uniform(-1, 1, (B, 1, 32, 32))
    mD, mG = RC.make_masks(B, rng), RC.make_masks(B, rng)
    st = dict(PD=PD.copy(), PG=PG.copy(), mD=np.zeros_like(PD), vD=np.zeros_like(PD), mG=np.zeros_like(PG),
              vG=np.zeros_like(PG), tD=0, tG=0)
    res = OC.f64.train_iteration(B, C, hyper, real_diff, condD, nD, condG, nG, mD, mG, st)
    PDt = torch.tensor(PD, requires_grad=True)
    PGt = torch.tensor(PG, requires_grad=True)
    with torch.no_grad():
        fake = RC.G_forward(PGt, torch.tensor(nD), torch.tensor(cond_fake), C)
    inputs = torch.cat([torch.tensor(real_diff), fake])
    targets = torch.tensor([1.0] * (B // 2) + [0.0] * (B // 2))
    out = RC.D_forward(PDt, inputs, torch.tensor(condD), torch.tensor(mD), C)
    out.backward(R.bce_grad(out.detach(), targets))
    lossD = float(R.bce(out.detach(), targets)) + 1e-7 * float(PDt.detach().abs().sum())
    gD = np.clip(PDt.grad.numpy() + 1e-7 * np.sign(PD), -1, 1)
    assert abs(res["lossD"] - lossD) < 1e-10
    assert rel(res["gradD"], gD) < 1e-8
    assert rel(res["fake"], fake.numpy()) < 1e-11
    PD1 = PD - 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9) * (0.1 * gD) / (np.sqrt(0.001 * gD * gD) + 1e-8)
    assert rel(st["PD"], PD1) < 1e-9
    PD1t = torch.tensor(st["PD"], requires_grad=True)
    diff = RC.G_forward(PGt, torch.tensor(nG), torch.tensor(condG), C)
    out = RC.D_forward(PD1t, diff, torch.tensor(condG), torch.tensor(mG), C)
    ones = torch.ones(B, dtype=torch.float64)
    out.backward(R.bce_grad(out.detach(), ones))
    gG = np.clip(PGt.grad.numpy(), -5, 5)
    assert abs(res["lossG"] - float(R.bce(out.detach(), ones))) < 1e-10
    assert rel(res["gradG"], gG) < 1e-8
    assert st["tD"] == 1 and st["tG"] == 1 and res["conf"].sum() == B
