"""tests/bn_ref.py (the float64 BatchNorm + PReLU yardstick of tests/test_gpu_batchnorm.py) pinned on the CPU to
PyTorch float64 autograd (F.batch_norm + torch.where) and to the C++ oracle's bn_fwd_train / bn_bwd, on ordinary
channels, on channels whose mean is 1e4 times their spread and on exactly constant channels."""
import numpy as np
import pytest

import bn_ref as R
from oracle import oracle as O

torch = pytest.importorskip("torch")
F = torch.nn.functional
TOL = 1e-10


def chan_err(a, b):
    """max over channels of max|a - b| / max|b| within the channel for NC... tensors; normwise over the channels for
    [C] vectors (the gamma gradient of a constant channel is 0)"""
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    if a.dim() == 1:
        return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))
    d = (a - b).abs().transpose(0, 1).reshape(a.shape[1], -1).max(1).values
    s = b.abs().transpose(0, 1).reshape(b.shape[1], -1).max(1).values
    return float((d / s.clamp_min(1e-300)).max())


def make(kind, seed, N=4, C=6, H=5):
    """float64 NCHW data, gamma, beta: "plain" channels, channels offset by 1e4 of their spread, or one channel
    exactly constant at 3.3 among plain ones"""
    g = torch.Generator().manual_seed(seed)
    sig = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    off = torch.randn(C, generator=g, dtype=torch.float64) * sig
    if kind == "offset":
        off = off + 1e4 * sig * torch.where(torch.arange(C) % 2 == 0, 1.0, -1.0)
    z = torch.randn(N, C, H, H, generator=g, dtype=torch.float64) * sig.view(1, -1, 1, 1) + off.view(1, -1, 1, 1)
    if kind == "constant":
        z[:, 1] = 3.3
    gamma = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    beta = torch.randn(C, generator=g, dtype=torch.float64) * 0.5
    dh = torch.randn(N, C, H, H, generator=g, dtype=torch.float64)
    return z, gamma, beta, dh


KINDS = ["plain", "offset", "constant"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("act", [False, True])
def test_forward_backward_match_torch_autograd(kind, act):
    z, gamma, beta, dh = make(kind, 1 + KINDS.index(kind))
    a = torch.tensor(0.25, dtype=torch.float64)
    zt, gt, bt, at = (t.clone().requires_grad_(True) for t in (z, gamma, beta, a))
    y = F.batch_norm(zt, None, None, gt, bt, training=True, eps=R.EPS)
    h = torch.where(y > 0, y, at * y) if act else y
    h.backward(dh)
    ref = R.forward_train(z, gamma, beta, a if act else None)
    assert chan_err(ref["h"], h.detach()) < TOL
    dz, dg, db, da = R.backward(z, gamma, beta, ref["mean"], ref["istd"], dh, a if act else None)
    assert chan_err(dz, zt.grad) < TOL
    assert chan_err(dg, gt.grad) < TOL and chan_err(db, bt.grad) < TOL
    if act:
        assert abs(float(da - at.grad)) < TOL * abs(float(at.grad))
    else:
        assert da is None


@pytest.mark.parametrize("kind", KINDS)
def test_running_statistics_and_evaluate_match_torch(kind):
    z, gamma, beta, _ = make(kind, 10 + KINDS.index(kind))
    C = z.shape[1]
    rm0 = torch.linspace(-2, 3, C, dtype=torch.float64)
    rv0 = torch.linspace(0.5, 4, C, dtype=torch.float64)
    rm, rv = rm0.clone(), rv0.clone()
    F.batch_norm(z, rm, rv, gamma, beta, training=True, momentum=R.MOMENTUM, eps=R.EPS)  # updates rm, rv in place
    ref = R.forward_train(z, gamma, beta)
    m, v = R.running_update(rm0, rv0, ref["mean"], ref["var"], R.count(z))
    assert chan_err(m, rm) < TOL and chan_err(v, rv) < TOL
    ev = F.batch_norm(z, rm, rv, gamma, beta, training=False, eps=R.EPS)
    assert chan_err(R.forward_eval(z, gamma, beta, rm, rv), ev) < TOL
    a = 0.25
    assert chan_err(R.forward_eval(z, gamma, beta, rm, rv, a), torch.where(ev > 0, ev, a * ev)) < TOL


@pytest.mark.parametrize("kind", KINDS)
def test_matches_oracle(kind):
    z, gamma, beta, dh = make(kind, 20 + KINDS.index(kind), N=3, C=5, H=7)
    C = z.shape[1]
    rm, rv = np.linspace(-1, 1, C), np.linspace(0.5, 2, C)
    ref = R.forward_train(z, gamma, beta)
    m, v = R.running_update(torch.as_tensor(rm), torch.as_tensor(rv), ref["mean"], ref["var"], R.count(z))
    y, mean, istd = O.f64.bn_fwd_train(z.numpy(), gamma.numpy(), beta.numpy(), rm, rv)
    assert chan_err(ref["u"], y) < TOL
    assert chan_err(ref["mean"], mean) < TOL and chan_err(ref["istd"], istd) < TOL
    assert chan_err(m, rm) < TOL and chan_err(v, rv) < TOL
    dx, dg, db = O.f64.bn_bwd(z.numpy(), gamma.numpy(), mean, istd, dh.numpy())
    dz, rdg, rdb, _ = R.backward(z, gamma, beta, ref["mean"], ref["istd"], dh)
    assert chan_err(dz, dx) < TOL and chan_err(rdg, dg) < TOL and chan_err(rdb, db) < TOL


def test_constant_channel_is_exact():
    """var 0: istd = 1/sqrt(eps), x_hat = 0, the output is beta and the input gradient g - mean(g), scaled"""
    z, gamma, beta, dh = make("constant", 30)
    ref = R.forward_train(z, gamma, beta)
    assert float(ref["var"][1]) == 0.0 and float(ref["istd"][1]) == 1.0 / np.sqrt(R.EPS)
    assert torch.equal(ref["u"][:, 1], torch.full_like(ref["u"][:, 1], float(beta[1])))
    dz, _, _, _ = R.backward(z, gamma, beta, ref["mean"], ref["istd"], dh)
    want = gamma[1] * ref["istd"][1] * (dh[:, 1] - dh[:, 1].mean())
    assert chan_err(dz[:, 1:2], want.unsqueeze(1)) < 1e-13


def test_supplied_mean_moves_only_x_hat():
    """an externally supplied mean m' shifts x_hat by (mean - m') * istd; the variance still comes from the data"""
    z, gamma, beta, _ = make("offset", 40)
    ref = R.forward_train(z, gamma, beta)
    same = R.forward_train(z, gamma, beta, mean=ref["mean"])
    assert torch.equal(same["u"], ref["u"])
    d = torch.linspace(-1e-3, 1e-3, z.shape[1], dtype=torch.float64)
    sh = R.forward_train(z, gamma, beta, mean=ref["mean"] + d)
    assert torch.equal(sh["istd"], ref["istd"]) and torch.equal(sh["mean"], ref["mean"])
    want = ref["u"] - (gamma * d * ref["istd"]).view(1, -1, 1, 1)
    assert float((sh["u"] - want).abs().max()) < 1e-9


def test_kink_pos_takes_the_given_branch_only_near_zero():
    u = torch.tensor([[-1.0, 2.0, 1e-9, -1e-9, 3.0]], dtype=torch.float64)
    gpu = torch.tensor([[True, False, False, True, False]])
    p = R.kink_pos(u, gpu, margin=2e-5)
    assert p.tolist() == [[False, True, False, True, True]]
    dz, _, _, da = R.backward(u.view(1, 5, 1, 1), torch.ones(5, dtype=torch.float64), torch.zeros(5, dtype=torch.float64),
                              torch.zeros(5, dtype=torch.float64), torch.ones(5, dtype=torch.float64),
                              torch.ones(1, 5, 1, 1, dtype=torch.float64), torch.tensor(0.25, dtype=torch.float64),
                              pos=p.view(1, 5, 1, 1))
    assert float(da) == -1.0 + 1e-9  # sum of u over the elements taken as u <= 0
