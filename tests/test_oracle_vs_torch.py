"""Cross-check of the CPU oracle against an independent PyTorch-CPU (autograd, fp64) restatement.

The reference has no golden vectors (SURVEY.md section 4) and cannot run here, so this is the strongest pin
available for the oracle ("parity unpinned" per the task rules; see oracle/fg_oracle.cpp header).
"""
import numpy as np
import pytest
import torch

from oracle import oracle as O
import torch_ref as R

torch.set_num_threads(8)


def rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.abs(a - b).max() / (np.abs(b).max() + 1e-300)


@pytest.mark.parametrize("C", [3, 1])
def test_G_fwd_bwd_matches_torch(C):
    rng = np.random.default_rng(10 + C)
    B = 4
    P = R.trained_like_G(C, rng)
    noise = rng.uniform(-1, 1, (B, 100))
    dout = rng.standard_normal((B, C, 32, 32))
    g = O.f64.G()
    out = g.forward(P, noise, C)
    dP, dn = g.backward(dout, want_dnoise=True)
    Pt = torch.tensor(P, requires_grad=True)
    nt = torch.tensor(noise, requires_grad=True)
    out_t, taps = R.G_forward(Pt, nt, C)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-11
    for k in ("z0", "h0", "z1", "h1", "z2", "h2", "z3"):
        assert rel(g.tap(k), taps[k].detach().numpy()) < 1e-10, k
    gt = Pt.grad.numpy()
    for k, (o, s) in O.G_layout(C).items():
        n = int(np.prod(s))
        if k in ("C1b", "C2b"):  # conv bias before BN: analytically zero gradient, pure rounding noise
            assert np.abs(dP[o:o + n]).max() < 1e-9 * np.abs(gt).max()
            continue
        assert rel(dP[o:o + n], gt[o:o + n]) < 1e-8, k
    assert rel(dn, nt.grad.numpy()) < 1e-8


@pytest.mark.parametrize("C", [3, 1])
def test_D_fwd_bwd_matches_torch(C):
    rng = np.random.default_rng(20 + C)
    B = 6
    P = R.trained_like_D(C, rng)
    img = rng.random((B, C, 32, 32))
    masks = R.make_masks(B, rng)
    dout = rng.standard_normal(B)
    d = O.f64.D()
    out = d.forward(P, img, masks)
    dP, dimg = d.backward(dout)
    Pt = torch.tensor(P, requires_grad=True)
    it = torch.tensor(img, requires_grad=True)
    out_t = R.D_forward(Pt, it, torch.tensor(masks), C)
    out_t.backward(torch.tensor(dout))
    assert rel(out, out_t.detach().numpy()) < 1e-12
    gt = Pt.grad.numpy()
    for k, (o, s) in O.D_layout(C).items():
        n = int(np.prod(s))
        assert rel(dP[o:o + n], gt[o:o + n]) < 1e-9, k
    assert rel(dimg, it.grad.numpy()) < 1e-9


def test_bce_forms():
    rng = np.random.default_rng(3)
    x = rng.uniform(0.01, 0.99, 16)
    t = (rng.random(16) < 0.5).astype(np.float64)
    assert abs(O.f64.bce_fwd(x, t) - float(R.bce(torch.tensor(x), torch.tensor(t)))) < 1e-14
    assert rel(O.f64.bce_bwd(x, t), R.bce_grad(torch.tensor(x), torch.tensor(t)).numpy()) < 1e-14
    # saturated sigmoid: reference's composed chain BCE.grad * y(1-y) gives exactly 0 (SURVEY.md X1)
    xs = np.array([1.0, 0.0])
    ts = np.array([0.0, 1.0])
    g = O.f64.bce_bwd(xs, ts) * xs * (1 - xs)
    assert np.all(g == 0)


def test_adam_closed_form():
    # interruptable_optimizers.lua:49-94: at t=1 the step is lr*sign(g) (up to eps)
    rng = np.random.default_rng(4)
    n = 1000
    x = rng.standard_normal(n)
    x0 = x.copy()
    g = rng.standard_normal(n)
    g = np.sign(g) * (np.abs(g) + 0.1)  # keep eps/(sqrt(1-b2)|g|) negligible
    m, v = np.zeros(n), np.zeros(n)
    O.f64.adam(x, g, m, v, 1)
    np.testing.assert_allclose(x0 - x, 1e-3 * np.sign(g), rtol=1e-5)
    # t=2 against a literal numpy transcription
    g2 = rng.standard_normal(n)
    m_ref = 0.9 * m + 0.1 * g2
    v_ref = 0.999 * v + 0.001 * g2 * g2
    step = 1e-3 * np.sqrt(1 - 0.999 ** 2) / (1 - 0.9 ** 2)
    x_ref = x - step * m_ref / (np.sqrt(v_ref) + 1e-8)
    O.f64.adam(x, g2, m, v, 2)
    np.testing.assert_allclose(x, x_ref, rtol=1e-13)
    np.testing.assert_allclose(m, m_ref, rtol=1e-12)


def test_penalty_clamp_order_and_G_quirk():
    p = np.array([0.5, -2.0, 0.0, 3.0])
    g = np.array([0.9, -0.2, 0.1, 10.0])
    # D: penalty then clamp (adversarial.lua:103-123)
    gd = g.copy()
    add = O.f64.penalty_clamp(p, gd, 0.01, 0.01, 0.1, 1.0)
    np.testing.assert_allclose(add, 0.01 * 5.5 + 0.1 * (0.25 + 4 + 9) / 2)
    np.testing.assert_allclose(gd, np.clip(g + 0.01 * np.sign(p) + 0.1 * p, -1, 1))
    # G quirk: L1 gradient term scaled by G_L2 (adversarial.lua:223)
    gg = g.copy()
    O.f64.penalty_clamp(p, gg, 0.01, 0.1, 0.1, 5.0)
    np.testing.assert_allclose(gg, np.clip(g + 0.1 * np.sign(p) + 0.1 * p, -5, 5))


def test_upsample_conv_phase_identity():
    """up2 -> 5x5/pad2 conv == four 3x3/pad1 phase convs with row/col pre-summed weights (SURVEY.md 7.3).
    This identity is what the tensor-core 'collapsed' conv path relies on."""
    rng = np.random.default_rng(5)
    B, Cin, Cout, H = 2, 5, 4, 6
    x = rng.standard_normal((B, Cin, H, H))
    W = rng.standard_normal((Cout, Cin, 5, 5))
    b = rng.standard_normal(Cout)
    ref = O.f64.conv_fwd(O.f64.up2_fwd(x), W, b)
    groups = {0: [(0, 1), (2, 3), (4,)], 1: [(0,), (1, 2), (3, 4)]}  # tap groups per phase parity
    out = np.zeros_like(ref)
    for py in (0, 1):
        for px in (0, 1):
            W3 = np.zeros((Cout, Cin, 3, 3))
            for i, gi in enumerate(groups[py]):
                for j, gj in enumerate(groups[px]):
                    W3[:, :, i, j] = sum(W[:, :, a, c] for a in gi for c in gj)
            out[:, :, py::2, px::2] = O.f64.conv_fwd(x, W3, b)
    assert rel(out, ref) < 1e-13


def test_train_iteration_matches_torch():
    """One full adversarial.lua loop body (config 1: gray, B=16 is exercised in test_golden; here B=4 color)."""
    rng = np.random.default_rng(6)
    B, C = 4, 3
    hyper = dict(lr_D=1e-3, lr_G=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, D_L1=0.0, D_L2=1e-4, G_L1=0.0, G_L2=0.0,
                 D_clamp=1.0, G_clamp=5.0)
    PD, PG = R.trained_like_D(C, rng), R.trained_like_G(C, rng)
    real = rng.random((B // 2, C, 32, 32))
    nD, nG = rng.uniform(-1, 1, (B // 2, 100)), rng.uniform(-1, 1, (B, 100))
    mD, mG = R.make_masks(B, rng), R.make_masks(B, rng)
    st = dict(PD=PD.copy(), PG=PG.copy(), mD=np.zeros_like(PD), vD=np.zeros_like(PD), mG=np.zeros_like(PG),
              vG=np.zeros_like(PG), tD=0, tG=0, bnG=np.concatenate([np.zeros(256), np.ones(256), np.zeros(128),
                                                                    np.ones(128)]))
    res = O.f64.train_iteration(B, C, hyper, real, nD, nG, mD, mG, st)
    # --- torch restatement ---
    PDt = torch.tensor(PD, requires_grad=True)
    PGt = torch.tensor(PG, requires_grad=True)
    with torch.no_grad():
        fake, _ = R.G_forward(PGt, torch.tensor(nD), C)
    inputs = torch.cat([torch.tensor(real), fake])
    targets = torch.tensor([1.0] * (B // 2) + [0.0] * (B // 2))
    out = R.D_forward(PDt, inputs, torch.tensor(mD), C)
    out.backward(R.bce_grad(out.detach(), targets))
    lossD = float(R.bce(out.detach(), targets)) + 1e-4 * float((PDt.detach() ** 2).sum()) / 2
    gD = np.clip(PDt.grad.numpy() + 1e-4 * PD, -1, 1)
    assert abs(res["lossD"] - lossD) < 1e-10
    assert rel(res["gradD"], gD) < 1e-8
    assert rel(res["fake"], fake.numpy()) < 1e-11
    PD1 = PD - 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9) * (0.1 * gD) / (np.sqrt(0.001 * gD * gD) + 1e-8)
    assert rel(st["PD"], PD1) < 1e-9
    PD1t = torch.tensor(st["PD"], requires_grad=True)
    img, _ = R.G_forward(PGt, torch.tensor(nG), C)
    out = R.D_forward(PD1t, img, torch.tensor(mG), C)
    ones = torch.ones(B, dtype=torch.float64)
    out.backward(R.bce_grad(out.detach(), ones))
    gG = np.clip(PGt.grad.numpy(), -5, 5)
    assert abs(res["lossG"] - float(R.bce(out.detach(), ones))) < 1e-10
    big = np.abs(gG) > 1e-6 * np.abs(gG).max()
    assert rel(res["gradG"][big], gG[big]) < 1e-7
    assert st["tD"] == 1 and st["tG"] == 1
    assert res["conf"].sum() == B


def test_f32_port_blas_path_matches_loop_path():
    """The optional OpenBLAS route of the fp32 port (oracle.use_blas, opt-in for the CPU baseline) computes the same
    convolution / Linear results as the blocked loops; the fp64 oracle is unaffected."""
    rng = np.random.default_rng(12)
    x = rng.standard_normal((3, 16, 12, 12)).astype(np.float32)
    w = (rng.standard_normal((8, 16, 5, 5)) * 0.05).astype(np.float32)
    b = rng.standard_normal(8).astype(np.float32)
    dy = rng.standard_normal((3, 8, 12, 12)).astype(np.float32)
    y0 = O.f32.conv_fwd(x, w, b)
    g0 = O.f32.conv_bwd(x, w, dy)
    ref64 = O.f64.conv_fwd(x, w, b)
    path = O.use_blas(2)
    try:
        if path is None:
            pytest.skip("no OpenBLAS shared object next to scipy")
        assert O.blas_active()
        y1 = O.f32.conv_fwd(x, w, b)
        g1 = O.f32.conv_bwd(x, w, dy)
        assert rel(y1, y0) < 1e-5 and all(rel(a, c) < 1e-5 for a, c in zip(g1, g0))
        np.testing.assert_array_equal(O.f64.conv_fwd(x, w, b), ref64)
        xl, wl, bl = rng.standard_normal((5, 70)).astype(np.float32), rng.standard_normal((9, 70)).astype(np.float32), rng.standard_normal(9).astype(np.float32)
        assert rel(O.f32.linear_fwd(xl, wl, bl), O.f64.linear_fwd(xl, wl, bl)) < 1e-5
    finally:
        O.lib().fgo_use_blas(None, 0)
    assert not O.blas_active()
