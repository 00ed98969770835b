"""CPU: the float64 restatement of train_denoiser.lua (tests/dn_ref.py) against PyTorch float64 autograd, the parameter
counts of the C ABI, the committed golden step and the loading of a synthetic `denoiser_CxHxW.net`."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dn_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(1, 16), (3, 16), (1, 32), (3, 32)]


def torch_decoder(P, x, state, training, masks, C, S, p_drop=0.2):
    """the DECODER in torch float64; P is a leaf tensor; state (numpy) is updated like nn.BatchNormalization's"""
    off, W = 0, {}
    for name, shape in R.shapes(C, S):
        n = int(np.prod(shape))
        W[name] = P[off:off + n].view(shape)
        off += n
    B, A2, sc = x.shape[0], (S - 4) ** 2, 1.0 / (1.0 - p_drop)

    def bn_act(z, l, mask):
        sm, sv = R._bn_slices(l)
        rm, rv = torch.tensor(state[sm]), torch.tensor(state[sv])
        u = F.batch_norm(z, rm, rv, W["g%d" % (l + 1)], W["b%d" % (l + 1)], training, 0.1, R.BN_EPS)
        state[sm], state[sv] = rm.numpy(), rv.numpy()
        h = torch.where(u > 0, u, R.SLOPE * u)
        return h * mask * sc if mask is not None else h

    m2 = m3 = None
    if training:
        mk = torch.tensor(np.asarray(masks, np.float64))
        m2, m3 = mk[:, :8 * A2].reshape(B, 8, S - 4, S - 4), mk[:, 8 * A2:]
    h1 = bn_act(F.conv2d(x, W["c1W"], W["c1b"]), 0, None)
    h2 = bn_act(F.conv2d(h1, W["c2W"], W["c2b"]), 1, m2)
    h3 = bn_act(F.linear(h2.reshape(B, -1), W["L1W"], W["L1b"]), 2, m3)
    return F.linear(h3, W["L2W"], W["L2b"])


def torch_bce(z, t):
    y = torch.sigmoid(z)
    return -torch.mean(t * torch.log(y + R.BCE_EPS) + (1 - t) * torch.log(1 - y + R.BCE_EPS))


@pytest.mark.parametrize("C,S", CASES)
@pytest.mark.parametrize("training", [True, False])
def test_decoder_forward_backward_matches_autograd(C, S, training):
    case = R.make_case(C, S, 4, seed=10 + C + S)
    x = case["images"].astype(np.float64) + case["noise"][0]
    st_ref, st_t = R.bn_init(), R.bn_init()
    st_ref[:16] += 0.1  # evaluation reads the running statistics: make them non-trivial
    st_t[:16] += 0.1
    z, cache = R.decoder_forward(case["P1"], x, st_ref, training, case["masks"][0], C, S)
    t = R.to_flat_img(case["images"].astype(np.float64))
    loss, dz = R.bce(R.sigmoid(z), t)
    g = R.decoder_backward(cache, dz, C, S)
    P = torch.tensor(case["P1"].astype(np.float64), requires_grad=True)
    zt = torch_decoder(P, torch.tensor(x), st_t, training, case["masks"][0], C, S)
    lt = torch_bce(zt, torch.tensor(t))
    lt.backward()
    assert R.relerr(z, zt.detach().numpy()) < 1e-12
    assert abs(loss - lt.item()) < 1e-12
    assert R.relerr(g, P.grad.numpy()) < 1e-10
    np.testing.assert_allclose(st_ref, st_t, rtol=1e-12, atol=1e-14)
    if not training:
        np.testing.assert_allclose(R.evaluate(case["P1"], st_ref, x, C, S),
                                   torch.sigmoid(zt).detach().numpy().reshape(case["images"].shape), rtol=1e-12)


def torch_step(st, images, noise, masks, C, S, h=R.HYPER):
    """train_denoiser.lua:247-341 with autograd gradients and optim.adam written out on one shared state"""
    t = torch.tensor(R.to_flat_img(images.astype(np.float64)))
    x = torch.tensor(images.astype(np.float64))

    def adam(P, g):
        st["t"] += 1
        g = torch.clamp(g + h["L1"] * torch.sign(P) + h["L2"] * P, -h["clamp"], h["clamp"])
        st["m"] = h["beta1"] * st["m"] + (1 - h["beta1"]) * g
        st["v"] = h["beta2"] * st["v"] + (1 - h["beta2"]) * g * g
        step = h["lr"] * np.sqrt(1 - h["beta2"] ** st["t"]) / (1 - h["beta1"] ** st["t"])
        return (P - step * st["m"] / (torch.sqrt(st["v"]) + h["eps"])).detach()

    P1 = st["P1"].clone().requires_grad_(True)
    l1 = torch_bce(torch_decoder(P1, x + torch.tensor(noise[0], dtype=torch.float64), st["bn1"], True, masks[0], C, S), t)
    l1.backward()
    st["P1"] = adam(st["P1"], P1.grad)
    with torch.no_grad():
        y1 = torch.sigmoid(torch_decoder(st["P1"], x + torch.tensor(noise[1], dtype=torch.float64), st["bn1"], True, masks[1],
                                         C, S)).reshape(x.shape)
    P2 = st["P2"].clone().requires_grad_(True)
    l2 = torch_bce(torch_decoder(P2, y1, st["bn2"], True, masks[2], C, S), t)
    l2.backward()
    st["P2"] = adam(st["P2"], P2.grad)
    return l1.item(), l2.item()


@pytest.mark.parametrize("C,S", CASES)
def test_batch_step_shares_one_adam_state(C, S):
    B = 4
    case = R.make_case(C, S, B, seed=3 * C + S)
    n = R.param_count(C, S)
    ref = dict(P1=case["P1"].astype(np.float64), P2=case["P2"].astype(np.float64), m=np.zeros(n), v=np.zeros(n), t=0,
               bn1=R.bn_init(), bn2=R.bn_init())
    tt = dict(P1=torch.tensor(ref["P1"]), P2=torch.tensor(ref["P2"]), m=torch.zeros(n, dtype=torch.float64),
              v=torch.zeros(n, dtype=torch.float64), t=0, bn1=R.bn_init(), bn2=R.bn_init())
    rng = np.random.default_rng(5)
    bn1_prev = R.bn_init()
    for batch in range(2):
        images = case["images"] if batch == 0 else rng.uniform(0, 1, case["images"].shape)
        noise = case["noise"] if batch == 0 else rng.normal(0, 0.1, case["noise"].shape)
        masks = case["masks"] if batch == 0 else rng.uniform(0, 1, case["masks"].shape) >= 0.2
        (a1, a2), _ = R.train_step(ref, images, noise, masks, C, S)
        b1, b2 = torch_step(tt, images, noise, masks, C, S)
        assert abs(a1 - b1) < 1e-12 and abs(a2 - b2) < 1e-12
        assert ref["t"] == tt["t"] == 2 * (batch + 1)
        for k in ("P1", "P2", "m", "v"):
            assert R.relerr(ref[k], tt[k].numpy()) < 1e-10, k
        np.testing.assert_allclose(ref["bn1"], tt["bn1"], rtol=1e-8, atol=1e-12)
        np.testing.assert_allclose(ref["bn2"], tt["bn2"], rtol=1e-8, atol=1e-12)
        # AE's running statistics moved twice in this batch: rm <- 0.81 rm + 0.09 m_a + 0.1 m_b
        assert not np.allclose(ref["bn1"], bn1_prev)
        bn1_prev = ref["bn1"].copy()
    # m and v hold both nets' gradients: after AE2's update, m is not AE2's gradient alone
    assert np.abs(ref["m"]).max() > 0


def test_param_counts_match_the_restatement():
    from face_generator_b200.lib import load_library
    lib = load_library()
    for C, S in CASES:
        assert lib.fg_dn_param_count(C, S) == R.param_count(C, S)
        assert lib.fg_dn_mask_per_sample(S) == R.mask_per_sample(S)
    assert lib.fg_dn_param_count(3, 32) == 19146568
    assert lib.fg_dn_param_count(3, 16) == 3939912
    assert lib.fg_dn_param_count(3, 64) == -1 and lib.fg_dn_param_count(2, 16) == -1 and lib.fg_dn_mask_per_sample(8) == -1


def test_hyper_defaults_match_train_denoiser():
    from face_generator_b200.denoiser import dn_hyper_default
    h = dn_hyper_default()
    for k, v in R.HYPER.items():
        assert abs(getattr(h, k) - v) <= 1e-7 * max(1.0, abs(v)), k


def test_host_layout_and_init_match_the_restatement():
    from face_generator_b200 import denoiser as D
    for C, S in CASES:
        assert D.layout(C, S) == R.shapes(C, S)
        assert D.init_params(C, S, np.random.default_rng(0)).size == R.param_count(C, S)


def test_golden_step_is_reproduced():
    g = np.load(os.path.join(HERE, "golden", "dn_step_c1_s16_b4.npz"))
    C, S = int(g["C"]), int(g["S"])
    case = R.make_case(C, S, int(g["B"]), seed=int(g["seed"]))
    for k in ("images", "noise", "masks"):
        np.testing.assert_array_equal(case[k], g[k])
    n = R.param_count(C, S)
    st = dict(P1=case["P1"].astype(np.float64), P2=case["P2"].astype(np.float64), m=np.zeros(n), v=np.zeros(n), t=0,
              bn1=R.bn_init(), bn2=R.bn_init())
    (l1, l2), _ = R.train_step(st, case["images"], case["noise"], case["masks"], C, S)
    np.testing.assert_allclose([l1, l2], g["losses"], rtol=1e-12)
    sel = g["sel"]
    for k in ("P1", "P2", "m", "v"):
        np.testing.assert_allclose(st[k][sel], g[k], rtol=1e-9, atol=1e-15)
    np.testing.assert_allclose(st["bn1"], g["bn1"], rtol=1e-12)
    np.testing.assert_allclose(st["bn2"], g["bn2"], rtol=1e-12)
    assert st["t"] == 2


def write_denoiser_net(path, C, S, nets, bn_style="var"):
    """a train_denoiser.lua-style `denoiser_CxHxW.net` ({AE1_ENCODER, AE1_DECODER, AE2_DECODER}, :360-362) built with
    the test_t7 helpers; nets = {"AE1_DECODER": (flat params, bn state), ...} with the BatchNorm state in the
    fg_dn_get_bn_state layout, stored as running_var or (2015 nn) running_std"""
    from test_t7 import W, Obj, Tensor, cuda_net, fstore, seq
    off, lay = 0, {}
    for name, shape in R.shapes(C, S):
        lay[name] = (off, list(shape))
        off += int(np.prod(shape))
    classes = [("nn.SpatialConvolution", 2), ("nn.SpatialBatchNormalization", 2), ("nn.LeakyReLU", 0),
               ("nn.SpatialConvolution", 2), ("nn.SpatialBatchNormalization", 2), ("nn.LeakyReLU", 0), ("nn.Dropout", 0),
               ("nn.View", 0), ("nn.Linear", 2), ("nn.BatchNormalization", 2), ("nn.LeakyReLU", 0), ("nn.Dropout", 0),
               ("nn.Linear", 2), ("nn.Sigmoid", 0), ("nn.View", 0)]
    t1 = lambda a: Tensor(fstore(a), [a.size], cls="torch.FloatTensor")  # noqa: E731
    root = {"AE1_ENCODER": seq(Obj("nn.WhiteNoise", {"mean": 0, "std": 0.1, "train": True}))}
    for key, (P, st) in nets.items():
        st, bn, o = np.asarray(st, np.float32), [], 0
        for c in (8, 8, 2048):  # SpatialBN(8), SpatialBN(8), BatchNormalization(2048)
            rm, rv = st[o:o + c], st[o + c:o + 2 * c]
            o += 2 * c
            if bn_style == "var":
                bn.append({"running_mean": t1(rm), "running_var": t1(rv), "eps": 1e-5, "momentum": 0.1})
            else:
                bn.append({"running_mean": t1(rm), "running_std": t1(1 / np.sqrt(rv + 1e-5)), "eps": 1e-5})
        # deactivateCuda / prepareNetworkForSave leave float tensors; the nn.Copy wrappers are walked through
        root[key] = cuda_net(np.asarray(P, np.float32), lay, classes, tensor_cls="torch.FloatTensor",
                             storage_cls="torch.FloatStorage", bn=bn)
    w = W()
    w.obj(root)
    with open(path, "wb") as f:
        f.write(bytes(w.buf))


@pytest.mark.parametrize("bn_style", ["var", "std"])
def test_loads_synthetic_denoiser_checkpoint(tmp_path, bn_style):
    from face_generator_b200.checkpoint import read_denoiser_checkpoint
    C, S = 3, 32
    rng = np.random.default_rng(7)
    n = R.param_count(C, S)
    want, nets = {}, {}
    for key, pk, bk in (("AE1_DECODER", "P1", "bn1"), ("AE2_DECODER", "P2", "bn2")):
        st = np.concatenate([np.concatenate([rng.standard_normal(c), rng.uniform(0.5, 2, c)]) for c in (8, 8, 2048)])
        want[pk], want[bk] = rng.standard_normal(n).astype(np.float32), st.astype(np.float32)
        nets[key] = (want[pk], want[bk])
    p = tmp_path / "denoiser_3x32x32.net"
    write_denoiser_net(str(p), C, S, nets, bn_style)
    got = read_denoiser_checkpoint(str(p), C, S)
    for k in ("P1", "P2"):
        np.testing.assert_array_equal(got[k], want[k])
    for k in ("bn1", "bn2"):
        np.testing.assert_allclose(got[k], want[k], rtol=2e-6 if bn_style == "std" else 0)
        assert got[k].size == 2 * (8 + 8 + 2048)
