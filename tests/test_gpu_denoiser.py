"""GPU: the denoising autoencoders of train_denoiser.lua (fg_dn_*) against the float64 restatement tests/dn_ref.py.

Tolerances: normwise relative error <= 1e-4 per tensor.  The conv biases and Linear1's bias sit in front of a BatchNorm,
so their gradients are analytically zero and numerically rounding noise: they are held to a magnitude bound only, and
after Adam (which turns any nonzero gradient into a step of about lr) the parameters are held to a few lr elementwise.
LeakyReLU kinks: an input within rounding of 0 may take the other branch; that changes one element's gradient, which the
normwise bound absorbs."""
import numpy as np
import pytest

import dn_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=256, channels=3)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx1():
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=256, channels=1)
    yield c
    c.close()


def make_dn(c, S, case):
    from face_generator_b200.denoiser import Denoiser
    dn = Denoiser(c, S)
    dn.set_params(0, case["P1"])
    dn.set_params(1, case["P2"])
    return dn


ZERO_GRAD = ("c1b", "c2b", "L1b")  # in front of a BatchNorm: analytically zero gradient in training


def slices(C, S):
    o = 0
    for name, shape in R.shapes(C, S):
        n = int(np.prod(shape))
        yield name, slice(o, o + n)
        o += n


def bn_slices():
    o = 0
    for l, c in enumerate((8, 8, 2048)):
        yield "mean%d" % (l + 1), slice(o, o + c)
        yield "var%d" % (l + 1), slice(o + c, o + 2 * c)
        o += 2 * c


def check_grads(got, ref, C, S, training=True, tol=1e-4):
    """per parameter tensor (dn_ref.shapes): normwise relative error <= tol; the zero-gradient biases to a magnitude
    bound relative to the largest gradient of the net"""
    scale = np.abs(ref).max()
    for name, sl in slices(C, S):
        if training and name in ZERO_GRAD:
            assert np.abs(got[sl]).max() <= 1e-4 * scale + 1e-7, name
        else:
            assert R.relerr(got[sl], ref[sl]) < tol, name


def check_bn(got, ref, tol=1e-4):
    for name, sl in bn_slices():
        assert R.relerr(got[sl], ref[sl]) < tol, name


@pytest.mark.parametrize("S,B", [(32, 128), (32, 16), (32, 2), (32, 256), (16, 128)])
@pytest.mark.parametrize("mma_f16", [1, 0])
@pytest.mark.parametrize("training", [True, False])
def test_forward_backward_match_float64(ctx, S, B, mma_f16, training):
    C = 3
    ctx.set_option("mma_f16", mma_f16)
    try:
        case = R.make_case(C, S, B, seed=100 + S + B)
        dn = make_dn(ctx, S, case)
        bn0 = R.bn_init()
        bn0[:16] += 0.05
        bn0[32:32 + 2048] = 0.02
        for net in (0, 1):
            dn.set_bn_state(net, bn0.astype(np.float32))
            P = case["P1"] if net == 0 else case["P2"]
            x = case["images"].astype(np.float64) + (case["noise"][0] if net == 0 and training else 0)
            st = bn0.copy()
            z, cache = R.decoder_forward(P, x, st, training, case["masks"][0], C, S)
            y = R.sigmoid(z).reshape(x.shape)
            out = dn.forward(net, case["images"], training=training, noise=case["noise"][0] if net == 0 else None,
                             masks=case["masks"][0])
            assert R.relerr(out, y) < 1e-4, net
            check_bn(dn.get_bn_state(net), st)
            dout = np.random.default_rng(net).standard_normal(x.shape).astype(np.float32)
            dn.zero_grads(net)
            dn.backward(net, dout)
            g = R.decoder_backward(cache, R.to_flat_img(dout * y * (1 - y)), C, S)
            check_grads(dn.get_grads(net), g, C, S, training)
        dn.close()
    finally:
        ctx.set_option("mma_f16", 1)


def gpu_state(dn):
    m, v, t = dn.get_adam_state()
    return dict(P1=dn.get_params(0).astype(np.float64), P2=dn.get_params(1).astype(np.float64), m=m.astype(np.float64),
                v=v.astype(np.float64), t=t, bn1=dn.get_bn_state(0).astype(np.float64), bn2=dn.get_bn_state(1).astype(np.float64))


KINK_MARGIN, KINK_MAX_FRAC = 2e-5, 2e-3


def gpu_kinks(dn, net, P, C, S):
    """dn_ref's `kinks` for the last forward of decoder `net` on the GPU: the LeakyReLU inputs within KINK_MARGIN of 0
    (relative to the layer's largest) take the branch the GPU took, read from its pre-activations and batch statistics.
    Everywhere else the reference keeps its own branch, so a wrong branch rule or mask still fails the 1e-4 bar.  The
    set must be tiny, and the GPU's values there ~0 as well."""
    W = R.unflat(P, C, S)
    sides = {0: S - 2, 1: S - 4}

    def kinks(l, u):
        mx = np.abs(u).max()
        idx = np.flatnonzero(np.abs(u) < KINK_MARGIN * mx)
        assert idx.size <= max(8, KINK_MAX_FRAC * u.size), (net, l, idx.size)
        if idx.size == 0:
            return idx, np.zeros(0, bool)
        z = dn.debug_tensor("%s.z%d" % (net, l + 1)).astype(np.float32)
        mean, istd = dn.debug_tensor("%s.mean%d" % (net, l + 1)), dn.debug_tensor("%s.istd%d" % (net, l + 1))
        if l < 2:  # NCHW flat index -> NHWC
            H = sides[l]
            b, r = np.divmod(idx, 8 * H * H)
            ch, q = np.divmod(r, H * H)
            zi = (b * H * H + q) * 8 + ch
        else:
            ch, zi = idx % 2048, idx
        t = ((z[zi] - mean[ch]).astype(np.float32) * istd[ch]).astype(np.float32).astype(np.float64)
        ug = W["g%d" % (l + 1)][ch] * t + W["b%d" % (l + 1)][ch]
        assert np.abs(ug).max() <= 10 * KINK_MARGIN * mx, (net, l, np.abs(ug).max())
        return idx, ug >= 0

    return kinks


@pytest.mark.parametrize("C,S,B", [(3, 32, 128), (1, 16, 16)])
def test_train_step_matches_float64_over_three_batches(ctx, ctx1, C, S, B):
    """three consecutive steps; each is checked against a float64 step from the state the GPU holds before it, so the
    1e-4 bar measures one step's arithmetic and not float32 rounding compounded by Adam over the earlier steps.  AE2's
    LeakyReLU inputs within rounding of 0 take the GPU's branch (gpu_kinks); AE's first forward is not kept on the
    GPU, and its gradients are checked through m (they agree to ~1e-6 per tensor)."""
    c = ctx if C == 3 else ctx1
    from face_generator_b200.denoiser import dn_hyper_default
    case = R.make_case(C, S, B, seed=7 * S + B)
    dn = make_dn(c, S, case)
    h = dn_hyper_default()
    lr = 1e-3
    for k in range(3):
        b = R.make_case(C, S, B, seed=1000 + k)
        st = gpu_state(dn)
        assert st["t"] == 2 * k
        P2 = st["P2"].copy()
        got = dn.train_step(h, b["images"], b["noise"], b["masks"], seed=k)
        (l1, l2), _ = R.train_step(st, b["images"], b["noise"], b["masks"], C, S, ae2_kinks=gpu_kinks(dn, "AE2", P2, C, S))
        assert got["t"] == st["t"] == 2 * (k + 1)
        assert abs(got["loss_AE1"] - l1) < 1e-4 * abs(l1) and abs(got["loss_AE2"] - l2) < 1e-4 * abs(l2)
        g = gpu_state(dn)
        for key in ("P1", "P2"):
            for name, sl in slices(C, S):
                if name in ZERO_GRAD:  # rounding-noise gradients: an Adam step moves them by up to a few lr, either sign
                    assert np.abs(g[key][sl] - st[key][sl]).max() <= 10 * lr, (k, key, name)
                else:
                    assert R.relerr(g[key][sl], st[key][sl]) < 1e-4, (k, key, name)
        for key in ("bn1", "bn2"):
            check_bn(g[key], st[key])
        for name, sl in slices(C, S):
            if name in ZERO_GRAD:
                continue
            assert R.relerr(g["m"][sl], st["m"][sl]) < 1e-4, (k, name)
            assert R.relerr(g["v"][sl], st["v"][sl]) < 3e-4, (k, name)  # quadratic in the gradients: twice their error
    dn.close()


def test_seeded_steps_are_reproducible_and_graph_replay_is_exact(ctx):
    from face_generator_b200.denoiser import dn_hyper_default
    C, S, B = 3, 16, 64
    case = R.make_case(C, S, B, seed=5)
    h = dn_hyper_default()
    results = []
    for use_graph in (0, 1, 1):
        ctx.set_option("use_graph", use_graph)
        dn = make_dn(ctx, S, case)
        for k in range(4):  # with the graph: eager, capture, then replays
            st = dn.train_step(h, case["images"], seed=11 + k)
        m, v, t = dn.get_adam_state()
        results.append((dn.get_params(0), dn.get_params(1), m, v, dn.get_bn_state(0), dn.get_bn_state(1), st["loss_AE1"],
                        st["loss_AE2"], t))
        dn.close()
    ctx.set_option("use_graph", 1)
    for a, b in zip(results[0], results[1]):
        np.testing.assert_array_equal(a, b)  # replayed graph == eager run
    for a, b in zip(results[1], results[2]):
        np.testing.assert_array_equal(a, b)  # same seed twice
    assert results[0][-1] == 8


def test_seed_drawn_noise_and_masks(ctx):
    from face_generator_b200.denoiser import dn_hyper_default
    C, S, B = 3, 32, 128
    case = R.make_case(C, S, B, seed=9)
    dn = make_dn(ctx, S, case)
    dn.train_step(dn_hyper_default(), case["images"], seed=3)
    n0, n1 = dn.debug_tensor("noise0"), dn.debug_tensor("noise1")
    assert n0.size == B * C * S * S
    for nz in (n0, n1):
        assert abs(nz.mean()) < 3e-3 and abs(nz.std() - 0.1) < 2e-3
    assert np.abs(n0 - n1).max() > 0.1  # fresh noise for AE's second forward
    for k in range(3):
        mk = dn.debug_tensor("masks%d" % k)
        assert set(np.unique(mk)) <= {0.0, 1.0} and abs(mk.mean() - 0.8) < 5e-3
    assert (dn.debug_tensor("masks0") != dn.debug_tensor("masks1")).any()
    dn.close()


def test_denoise_sampled_images_matches_evaluate(ctx):
    from face_generator_b200.lib import NET_G, f32
    import face_generator_b200 as fg
    C, S, N = 3, 32, 100
    rng = np.random.default_rng(4)
    ctx.set_params(NET_G, f32(rng.normal(0, 0.02, ctx.count(NET_G))))
    images = ctx.sample(f32(rng.uniform(-1, 1, (N, fg.NOISE_DIM))), 50)
    case = R.make_case(C, S, 2, seed=21)
    dn = make_dn(ctx, S, case)
    bn = R.bn_init()
    bn[:16] = rng.uniform(0.2, 1.0, 16)
    bn[32:] = rng.uniform(0.2, 1.0, 2 * 2048)
    dn.set_bn_state(0, bn.astype(np.float32))
    got = dn.denoise(images, chunk=64)
    ref = R.evaluate(case["P1"], bn.astype(np.float32).astype(np.float64), images, C, S)
    assert R.relerr(got, ref) < 1e-4
    dn.close()


def test_unsupported_sizes_and_batches(ctx):
    from face_generator_b200.denoiser import Denoiser, dn_hyper_default
    from face_generator_b200.lib import FGError
    with pytest.raises(FGError):
        Denoiser(ctx, 64)
    dn = Denoiser(ctx, 16)
    with pytest.raises(FGError):
        dn.train_step(dn_hyper_default(), np.zeros((1, 3, 16, 16), np.float32))
    dn.close()


def nchw(a, B, H, C):
    return a.reshape(B, H, H, C).transpose(0, 3, 1, 2).astype(np.float64)


@pytest.mark.parametrize("B", [2, 16, 128, 256])
def test_isolated_launches_match_float64(ctx, B):
    """each kernel family on the GPU's own inputs (debug tensors): the valid convolutions (forward, data and weight
    gradients) at 1e-5 and the 1-D BatchNorm + LeakyReLU + Dropout at C = 2048, running statistics included"""
    C, S = 3, 32
    A2 = (S - 4) ** 2
    case = R.make_case(C, S, B, seed=300 + B)
    dn = make_dn(ctx, S, case)
    bn0 = R.bn_init()
    bn0[32:32 + 2048] = 0.02
    dn.set_bn_state(0, bn0.astype(np.float32))
    dn.forward(0, case["images"], training=True, noise=case["noise"][0], masks=case["masks"][0])
    dn.zero_grads(0)
    dn.backward(0, np.random.default_rng(1).standard_normal(case["images"].shape).astype(np.float32))
    W = R.unflat(case["P1"], C, S)
    g = R.unflat(dn.get_grads(0), C, S)
    t = dn.debug_tensor
    x, h1 = nchw(t("AE1.x"), B, S, C), nchw(t("AE1.h1"), B, S - 2, 8)
    dz1, dz2 = nchw(t("dz1"), B, S - 2, 8), nchw(t("dz2"), B, S - 4, 8)
    # convolutions
    assert R.relerr(nchw(t("AE1.z1"), B, S - 2, 8), R.conv_valid(x, W["c1W"], W["c1b"])) < 1e-5
    assert R.relerr(nchw(t("AE1.z2"), B, S - 4, 8), R.conv_valid(h1, W["c2W"], W["c2b"])) < 1e-5
    assert R.relerr(nchw(t("dh1"), B, S - 2, 8), R.conv_dgrad(dz2, W["c2W"])) < 1e-5
    for (wn, bn_), xin, dz in ((("c1W", "c1b"), x, dz1), (("c2W", "c2b"), h1, dz2)):
        dW, db = R.conv_wgrad(xin, dz)
        assert R.relerr(g[wn], dW) < 1e-5, wn
        # the bias gradient is a sum of terms that cancel: held to the size of those terms
        assert np.abs(g[bn_] - db).max() <= 1e-5 * np.abs(dz).sum(axis=(0, 2, 3)).max(), bn_
    # 1-D BatchNorm at C = 2048 over B rows, forward with its running statistics, and backward
    z3 = t("AE1.z3").reshape(B, 2048).astype(np.float64)
    st = bn0.copy()
    mask3 = case["masks"][0][:, 8 * A2:].astype(np.float64)
    h3, cache = R.bn_act_fwd(z3, W["g3"], W["b3"], st, 2, True, mask3, 1 / 0.8)
    assert R.relerr(t("AE1.h3").reshape(B, 2048), h3) < 1e-5
    got_st = dn.get_bn_state(0)
    for name, sl in list(bn_slices())[4:]:
        assert R.relerr(got_st[sl], st[sl]) < 1e-5, name
    dz3, dg3, db3 = R.bn_act_bwd(t("dh3").reshape(B, 2048).astype(np.float64), W["g3"], cache, 1 / 0.8)
    assert R.relerr(t("dz3").reshape(B, 2048), dz3) < 1e-5
    assert R.relerr(g["g3"], dg3) < 1e-5 and R.relerr(g["b3"], db3) < 1e-5
    dn.close()


def test_backward_after_a_step_needs_a_forward(ctx):
    from face_generator_b200.denoiser import dn_hyper_default
    from face_generator_b200.lib import FGError
    case = R.make_case(3, 16, 8, seed=2)
    dn = make_dn(ctx, 16, case)
    dn.train_step(dn_hyper_default(), case["images"], seed=1)
    with pytest.raises(FGError):
        dn.backward(0, np.zeros_like(case["images"]))
    dn.forward(0, case["images"], training=False)
    dn.backward(0, np.zeros_like(case["images"]))
    dn.close()


def test_trained_state_survives_a_checkpoint(ctx, tmp_path):
    """train, write parameters AND BatchNorm running statistics into a train_denoiser.lua-style .net, load it into a
    fresh Denoiser: evaluate-mode denoising is bit for bit the trained instance's"""
    from test_denoiser_cpu import write_denoiser_net
    from face_generator_b200.checkpoint import load_denoiser_checkpoint
    from face_generator_b200.denoiser import Denoiser, dn_hyper_default
    C, S, B = 3, 16, 32
    case = R.make_case(C, S, B, seed=41)
    dn = make_dn(ctx, S, case)
    h = dn_hyper_default()
    for k in range(3):
        dn.train_step(h, R.make_case(C, S, B, seed=500 + k)["images"], seed=k)
    bn = [dn.get_bn_state(0), dn.get_bn_state(1)]
    assert not np.allclose(bn[0], R.bn_init())  # training moved the running statistics
    p = tmp_path / "denoiser_3x16x16.net"
    write_denoiser_net(str(p), C, S, {"AE1_DECODER": (dn.get_params(0), bn[0]), "AE2_DECODER": (dn.get_params(1), bn[1])})
    fresh = Denoiser(ctx, S)
    load_denoiser_checkpoint(fresh, str(p))
    np.testing.assert_array_equal(fresh.get_bn_state(0), bn[0])
    images = R.make_case(C, S, 40, seed=77)["images"]
    np.testing.assert_array_equal(fresh.denoise(images), dn.denoise(images))
    fresh.close()
    dn.close()


def test_device_fed_epoch_loop(ctx):
    """denoiser.train on a DeviceDataset equals the same batches gathered to the host and stepped one by one; the
    ragged last batch runs, a last batch of one image is skipped"""
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.denoiser import dn_hyper_default, train
    C, S, bs, seed = 3, 16, 32, 9
    rng = np.random.default_rng(3)
    h = dn_hyper_default()
    for N, nsteps in ((70, 3), (65, 2)):
        ds = DeviceDataset(ctx, rng.integers(0, 256, (N, C, 64, 64), dtype=np.uint8))
        case = R.make_case(C, S, 2, seed=8)
        a, b = make_dn(ctx, S, case), make_dn(ctx, S, case)
        hist = train(a, ds, h, batch_size=bs, epochs=1, seed=seed, log=None)
        perm = np.random.default_rng(seed).permutation(N).astype(np.int32)
        step = 0
        for t0 in range(0, N, bs):
            idx = perm[t0:t0 + bs]
            if idx.size < 2:
                continue
            b.train_step(h, ds.gather(idx, S), seed=(seed << 32) + step)
            step += 1
        assert step == nsteps and a.get_adam_state()[2] == 2 * nsteps and len(hist) == 1 and np.isfinite(hist[0]).all()
        for net in (0, 1):
            np.testing.assert_array_equal(a.get_params(net), b.get_params(net))
            np.testing.assert_array_equal(a.get_bn_state(net), b.get_bn_state(net))
        a.close()
        b.close()
        ds.close()
