"""CPU: the float64 restatement tests/ae_ref.py of train_autoencoder.lua against PyTorch float64 autograd and the
oracle's Adam, the host-side layout helpers, the checkpoint reader on a synthetic `autoencoder.net`, and a golden step."""
import os

import numpy as np
import pytest
import torch

import ae_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(32, 256), (16, 256), (16, 64)]


def torch_forward(P, x, masks, S, d, p=0.5):
    W = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in R.unflat(np.asarray(P, np.float64), S, d).items()}
    x = torch.tensor(np.asarray(x, np.float64).reshape(-1, S * S))
    h1 = torch.relu(torch.nn.functional.linear(x, W["L1W"], W["L1b"]))
    code = torch.tanh(torch.nn.functional.linear(h1, W["L2W"], W["L2b"]))
    h2 = code if masks is None else code * torch.tensor(np.asarray(masks, np.float64).reshape(-1, d)) / (1 - p)
    h3 = torch.relu(torch.nn.functional.linear(h2, W["L3W"], W["L3b"]))
    y = torch.sigmoid(torch.nn.functional.linear(h3, W["L4W"], W["L4b"]))
    return W, x, code, y


def flat_grads(W, S, d):
    return np.concatenate([W[n].grad.numpy().ravel() for n, _ in R.shapes(S, d)])


@pytest.mark.parametrize("S,d", CASES)
@pytest.mark.parametrize("training", [True, False])
def test_forward_backward_matches_autograd(S, d, training):
    case = R.make_case(S, 6, d, seed=S + d)
    masks = case["masks"] if training else None
    c = R.forward(case["P"], case["images"], masks, S, d)
    W, x, code, y = torch_forward(case["P"], case["images"], masks, S, d)
    np.testing.assert_allclose(c["code"], code.detach().numpy(), rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(c["y"], y.detach().numpy(), rtol=1e-10, atol=1e-13)
    loss, dy = R.criterion(c["y"], c["x"])
    tl = torch.nn.L1Loss()(y, x)
    tl.backward()
    assert abs(loss - tl.item()) < 1e-12
    g, _ = R.backward(c, dy)
    assert R.relerr(g, flat_grads(W, S, d)) < 1e-10


def test_tie_counts_as_positive_and_relu_is_closed_at_zero():
    y = np.array([[0.25, 0.5, 0.75]])
    loss, dy = R.criterion(y, np.array([[0.25, 0.75, 0.5]]))
    np.testing.assert_array_equal(dy * 3, [[1.0, -1.0, 1.0]])
    assert abs(loss - 0.5 / 3) < 1e-15
    assert not R._side(np.zeros((1, 2)), "z1", None).any()
    assert R._side(np.zeros((1, 2)), "z1", {"z1": (np.array([1]), np.array([True]))}).tolist() == [[False, True]]


def test_three_steps_match_autograd_and_the_oracle_adam():
    from oracle import oracle as O
    S, d, B = 16, 64, 5
    h = dict(R.HYPER, L1=1e-5, L2=1e-4)
    case = R.make_case(S, B, d, seed=11)
    st = R.fresh_state(case["P"])
    P, m, v = st["P"].copy(), st["m"].copy(), st["v"].copy()
    rng = np.random.default_rng(3)
    for k in range(3):
        masks = (rng.uniform(size=(B, d)) >= 0.5).astype(np.float32)
        W, x, _, y = torch_forward(P, case["images"], masks, S, d)
        torch.nn.L1Loss()(y, x).backward()
        g = flat_grads(W, S, d) + h["L1"] * np.sign(P) + h["L2"] * P
        loss, g_ref, _ = R.train_step(st, case["images"], masks, S, d, h)
        assert R.relerr(g_ref, g) < 1e-10
        assert abs(loss - torch.nn.L1Loss()(y, x).item()) < 1e-12  # the reported loss carries no penalty term
        O.f64.adam(P, g, m, v, k + 1, h["lr"], h["beta1"], h["beta2"], h["eps"])
        np.testing.assert_allclose(st["P"], P, rtol=1e-10, atol=1e-14)
        np.testing.assert_allclose(st["v"], v, rtol=1e-9, atol=1e-30)
    assert st["t"] == 3


def test_param_counts_and_layout():
    from face_generator_b200 import autoencoder as A
    assert R.param_count(32, 256) == 985088 and R.param_count(16, 256) == 394496
    for S, d in CASES:
        assert A.param_count(S, d) == R.param_count(S, d)
        assert A.layout(S, d) == R.shapes(S, d)
        p = A.init_params(S, d, np.random.default_rng(0))
        assert p.size == R.param_count(S, d) and p.dtype == np.float32
        w = R.unflat(p, S, d)
        assert abs(w["L1W"].std() - 0.005) < 2e-4 and abs(w["L4b"].std() - 0.001) < 2e-4
    # the code width is a multiple of 8 in [8, 1024]; sizes are 16 and 32
    for S, d in [(32, 8), (32, 1024), (16, 40)]:
        assert A.param_count(S, d) == R.param_count(S, d)
    for S, d in [(32, 0), (32, 4), (32, 12), (32, 1032), (64, 256), (8, 256)]:
        assert A.param_count(S, d) == -1


def test_hyper_defaults_match_train_autoencoder():
    from face_generator_b200.autoencoder import ae_hyper_default
    h = ae_hyper_default()
    for k, v in R.HYPER.items():
        assert abs(getattr(h, k) - v) < 1e-7 * max(1, abs(v)) + 1e-12, k
    assert ae_hyper_default(L2=0.5).L2 == 0.5
    with pytest.raises(KeyError):
        ae_hyper_default(clamp=1)  # the script clamps nothing


def test_golden_step_is_reproduced():
    g = np.load(os.path.join(HERE, "golden", "ae_step_s16_b4.npz"))
    S, d = int(g["S"]), int(g["d"])
    case = R.make_case(S, int(g["B"]), d, seed=int(g["seed"]))
    np.testing.assert_array_equal(case["images"], g["images"])
    np.testing.assert_array_equal(case["masks"], g["masks"])
    st = R.fresh_state(case["P"])
    loss, grad, c = R.train_step(st, case["images"], case["masks"], S, d, dict(R.HYPER, L1=float(g["L1"]), L2=float(g["L2"])))
    np.testing.assert_allclose(loss, g["loss"], rtol=1e-12)
    sel = g["sel"]
    np.testing.assert_allclose(grad[sel], g["g"], rtol=1e-9, atol=1e-18)
    for k in ("P", "m", "v"):
        np.testing.assert_allclose(st[k][sel], g[k], rtol=1e-9, atol=1e-18)
    np.testing.assert_allclose(c["code"], g["code"], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(c["y"], g["y"], rtol=1e-12)
    assert st["t"] == 1


def write_autoencoder_net(path, S, d, P):
    """a train_autoencoder.lua-style `autoencoder.net` ({AE = MODEL_AE, optstate = OPTSTATE}, :234), built with the
    test_t7 helpers; the script saves the CUDA net as it is"""
    from test_t7 import W, cuda_net
    off, lay = 0, {}
    for name, shape in R.shapes(S, d):
        lay[name] = (off, list(shape))
        off += int(np.prod(shape))
    classes = [("nn.View", 0), ("nn.Linear", 2), ("nn.ReLU", 0), ("nn.Linear", 2), ("nn.Tanh", 0), ("nn.Dropout", 0),
               ("nn.Linear", 2), ("nn.ReLU", 0), ("nn.Linear", 2), ("nn.Sigmoid", 0), ("nn.View", 0)]
    root = {"AE": cuda_net(np.asarray(P, np.float32), lay, classes),
            "optstate": {"adagrad": {}, "adam": {"t": 3}, "rmsprop": {}, "sgd": {"learningRate": 0.02, "momentum": 0}}}
    w = W()
    w.obj(root)
    with open(path, "wb") as f:
        f.write(bytes(w.buf))


def test_loads_synthetic_autoencoder_checkpoint(tmp_path):
    from face_generator_b200.checkpoint import read_autoencoder_checkpoint
    from face_generator_b200.lib import FGError
    S, d = 16, 64
    want = np.random.default_rng(5).standard_normal(R.param_count(S, d)).astype(np.float32)
    p = tmp_path / "autoencoder.net"
    write_autoencoder_net(str(p), S, d, want)
    np.testing.assert_array_equal(read_autoencoder_checkpoint(str(p), S, d), want)
    with pytest.raises(FGError, match="parameters"):
        read_autoencoder_checkpoint(str(p), S, 256)
