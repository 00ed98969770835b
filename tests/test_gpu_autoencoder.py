"""GPU: the autoencoder of train_autoencoder.lua (fg_ae_*) against the float64 restatement tests/ae_ref.py.

Tolerances: normwise relative error <= 1e-4 per tensor.  nn.ReLU and nn.AbsCriterion have kinks: for the elements
within rounding of one (gpu_kinks) the reference takes the side the GPU took, read from the GPU's own tensors, and
those elements must be few; everywhere else the reference keeps its own side, so a wrong rule still fails."""
import ctypes as C

import numpy as np
import pytest

import ae_ref as R

pytestmark = pytest.mark.gpu

ACTS = ("z1", "h1", "z2", "code", "h2", "z3", "h3", "z4", "y")
GRADS = ("dz4", "dz3", "dz2", "dz1")
KINK_MARGIN, KINK_MAX_FRAC = 2e-5, 2e-3


@pytest.fixture(scope="module")
def ctx3():
    """a 3-channel context created before everything here and stepped after it (test_other_nets_are_untouched)"""
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=64, channels=3)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx(ctx3):
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=256, channels=1)
    yield c
    c.close()


def make_ae(c, S, d, P):
    from face_generator_b200.autoencoder import Autoencoder
    ae = Autoencoder(c, S, d)
    ae.set_params(P)
    return ae


def slices(S, d):
    o = 0
    for name, shape in R.shapes(S, d):
        n = int(np.prod(shape))
        yield name, slice(o, o + n)
        o += n


def check_grads(got, ref, S, d, tol=1e-4):
    for name, sl in slices(S, d):
        assert R.relerr(got[sl], ref[sl]) < tol, name


def gpu_kinks(ae, criterion=False):
    """ae_ref's `kinks` from the GPU's last forward: ReLU inputs within KINK_MARGIN of 0 (relative to the layer's
    largest) take the side the GPU took; with `criterion`, so do outputs within KINK_MARGIN of their target (the side is
    the sign of the GPU's dz4, whose other factor y(1-y) is positive).  The sets must be tiny."""
    kinks = {}
    for key in ("z1", "z3"):
        z = ae.debug_tensor(key)
        idx = np.flatnonzero(np.abs(z) < KINK_MARGIN * np.abs(z).max())
        assert idx.size <= max(8, KINK_MAX_FRAC * z.size), (key, idx.size)
        kinks[key] = (idx, z[idx] > 0)
    if criterion:
        y, t, dz4 = ae.debug_tensor("y"), ae.debug_tensor("x"), ae.debug_tensor("dz4")
        idx = np.flatnonzero(np.abs(y - t) < KINK_MARGIN)
        assert idx.size <= max(8, KINK_MAX_FRAC * y.size), ("y", idx.size)
        kinks["y"] = (idx, dz4[idx] >= 0)
    return kinks


@pytest.mark.parametrize("S,B,d", [(32, 128, 256), (32, 16, 256), (32, 1, 256), (32, 256, 256), (16, 128, 256), (32, 128, 64),
                                   (16, 16, 64), (32, 16, 40)])
@pytest.mark.parametrize("mma_f16", [1, 0])
@pytest.mark.parametrize("training", [True, False])
def test_forward_backward_match_float64(ctx, S, B, d, mma_f16, training):
    ctx.set_option("mma_f16", mma_f16)
    try:
        case = R.make_case(S, B, d, seed=100 + S + B + d)
        ae = make_ae(ctx, S, d, case["P"])
        masks = case["masks"] if training else None
        code, out = ae.forward(case["images"], training=training, masks=masks)
        c = R.forward(case["P"], case["images"], masks, S, d, kinks=gpu_kinks(ae))
        assert R.relerr(code, c["code"]) < 1e-4 and R.relerr(out, c["y"]) < 1e-4
        for k in ACTS:
            assert R.relerr(ae.debug_tensor(k), c[k]) < 1e-4, k
        dout = np.random.default_rng(B).standard_normal(out.shape).astype(np.float32)
        ae.zero_grads()
        ae.backward(dout)
        g, dz = R.backward(c, dout.astype(np.float64).reshape(B, -1))
        for k in GRADS:
            assert R.relerr(ae.debug_tensor(k), dz[k]) < 1e-4, k
        check_grads(ae.get_grads(), g, S, d)
        ae.backward(dout)  # accumulates
        check_grads(ae.get_grads(), 2 * g, S, d)
        ae.close()
    finally:
        ctx.set_option("mma_f16", 1)


def test_fp32_ffma_path_matches_float64(ctx):
    """conv_impl = SIMT: the four Linear layers on the fp32 FFMA kernels (the cross-check of the wgmma path)"""
    S, B, d = 32, 32, 256
    ctx.set_option("conv_impl", 0)
    try:
        case = R.make_case(S, B, d, seed=5)
        ae = make_ae(ctx, S, d, case["P"])
        _, out = ae.forward(case["images"], training=True, masks=case["masks"])
        c = R.forward(case["P"], case["images"], case["masks"], S, d, kinks=gpu_kinks(ae))
        assert R.relerr(out, c["y"]) < 1e-5
        dout = np.random.default_rng(1).standard_normal(out.shape).astype(np.float32)
        ae.zero_grads()
        ae.backward(dout)
        check_grads(ae.get_grads(), R.backward(c, dout.astype(np.float64).reshape(B, -1))[0], S, d, tol=1e-5)
        ae.close()
    finally:
        ctx.set_option("conv_impl", 2)


@pytest.mark.parametrize("S,B,d,L1,L2", [(32, 128, 256, 0.0, 0.0), (16, 16, 64, 1e-5, 1e-4)])
def test_three_train_steps_match_the_reference_loop(ctx, S, B, d, L1, L2):
    """each step from the state the GPU holds before it: loss, every activation, and the gradient the optimizer saw
    (with the penalty terms), which is what the parameters are compared through; the Adam state is checked where the
    update is well conditioned"""
    from face_generator_b200.autoencoder import ae_hyper_default
    case = R.make_case(S, B, d, seed=7)
    ae = make_ae(ctx, S, d, case["P"])
    h = dict(R.HYPER, L1=L1, L2=L2)
    hyper = ae_hyper_default(L1=L1, L2=L2)
    rng = np.random.default_rng(9)
    for k in range(3):
        masks = (rng.uniform(size=(B, d)) >= 0.5).astype(np.float32)
        m, v, t = ae.get_adam_state()
        st = dict(P=ae.get_params().astype(np.float64), m=m.astype(np.float64), v=v.astype(np.float64), t=t)
        P_before = st["P"].copy()
        got = ae.train_step(hyper, case["images"], masks=masks, seed=k)
        loss, g, c = R.train_step(st, case["images"], masks, S, d, h, kinks=gpu_kinks(ae, criterion=True))
        assert got["t"] == k + 1 == st["t"]
        assert abs(got["loss"] - loss) <= 1e-4 * loss
        for name in ACTS + GRADS:
            assert R.relerr(ae.debug_tensor(name), c[name]) < 1e-4, (k, name)
        np.testing.assert_array_equal(ae.debug_tensor("masks"), masks.ravel())
        check_grads(ae.get_grads(), g, S, d)  # as GRAD_PARAMETERS_AE after fevalAE: penalty terms included
        m2, v2, _ = ae.get_adam_state()
        assert R.relerr(m2, st["m"]) < 1e-4 and R.relerr(v2, st["v"]) < 3e-4
        # every parameter moved by at most about lr, towards where the reference moved it
        P_after = ae.get_params().astype(np.float64)
        assert np.abs(P_after - P_before).max() <= 1.5 * h["lr"]
        assert R.relerr(P_after - P_before, st["P"] - P_before) < 5e-2
    with pytest.raises(Exception, match=r"\(-5\)"):  # FG_ERR_STATE: the step left no forward to differentiate
        ae.backward(np.zeros_like(case["images"]))
    ae.close()


def test_sigmoid_abs_ties_saturation_and_loss(ctx):
    """the fused Sigmoid + AbsCriterion of the step alone, driven through a net whose last layer is only its bias"""
    from face_generator_b200.autoencoder import ae_hyper_default
    S, B, d = 32, 256, 64
    n = B * S * S
    rng = np.random.default_rng(3)
    P = np.zeros(R.param_count(S, d), np.float32)
    bias = rng.uniform(-3, 3, S * S).astype(np.float32)
    bias[:8] = [40, -40, 110, -110, 40, -40, 110, -110]
    P[-S * S:] = bias
    ae = make_ae(ctx, S, d, P)
    images = rng.uniform(0, 1, (B, 1, S, S)).astype(np.float32)
    hyper = ae_hyper_default(lr=0.0)  # the parameters stay
    ae.train_step(hyper, images, seed=0)
    y = ae.debug_tensor("y").reshape(B, -1)  # zero weights: y = sigmoid(bias) whatever the input
    t = images.reshape(B, -1).copy()
    t[::2, 16:] = y[::2, 16:]  # ties: the targets are the step's own outputs
    got = ae.train_step(hyper, t.reshape(images.shape), seed=1)
    np.testing.assert_array_equal(ae.debug_tensor("y").reshape(B, -1), y)
    dz4 = ae.debug_tensor("dz4").reshape(B, -1)
    inv = np.float32(1.0) / np.float32(n)
    yy = y[::2, 16:]
    np.testing.assert_array_equal(dz4[::2, 16:], inv * (np.float32(1) - yy) * yy)  # a tie is +1/n, composed as the reference does
    assert (dz4[::2, 16:] > 0).all()
    # saturation: logits +40, +-110 round the sigmoid to exactly 1 or 0 and pass exactly 0; -40 leaves y = 4e-18 and a
    # gradient of that size, as the composed chain gives
    for col in (0, 2, 3, 4, 6, 7):
        assert (dz4[:, col] == 0).all(), col
    for col in (1, 5):
        assert (y[:, col] > 0).all() and (np.abs(dz4[:, col]) <= 1e-17 * inv).all() and (dz4[:, col] != 0).all()
    ref = np.abs(y.astype(np.float64) - t.astype(np.float64)).mean()
    assert abs(got["loss"] - ref) <= 1e-6 * ref
    ae.close()


def test_seeded_step_is_reproducible_and_the_replay_is_bit_exact(ctx):
    from face_generator_b200.autoencoder import ae_hyper_default
    S, B, d = 32, 128, 256
    case = R.make_case(S, B, d, seed=21)
    hyper = ae_hyper_default()
    ae = make_ae(ctx, S, d, case["P"])
    n = ae.n
    results = []
    for rep in range(4):  # the first call runs eagerly, the second captures, the rest replay
        ae.set_params(case["P"])
        ae.set_adam_state(np.zeros(n, np.float32), np.zeros(n, np.float32), 0)
        st = ae.train_step(hyper, case["images"], seed=77)
        results.append((st["loss"], ae.get_params(), ae.debug_tensor("masks"), ae.get_grads()))
    for r in results[1:]:
        assert r[0] == results[0][0]
        for a, b in zip(r[1:], results[0][1:]):
            np.testing.assert_array_equal(a, b)
    keep = results[0][2]
    assert set(np.unique(keep)) == {0.0, 1.0}
    assert abs(keep.mean() - 0.5) < 3 * 0.5 / np.sqrt(keep.size)
    ae.train_step(hyper, case["images"], seed=78)
    other = ae.debug_tensor("masks")
    assert 0.4 < (other != keep).mean() < 0.6
    ae.close()


@pytest.mark.parametrize("N", [70, 65])
def test_device_fed_epoch_equals_host_stepped_batches(ctx, N):
    """autoencoder.train on a DeviceDataset at batch 32 (tails of 6 and 1) against the same batches gathered to the
    host and stepped one by one"""
    from face_generator_b200 import autoencoder as A
    from face_generator_b200.dataset import DeviceDataset
    S, d, bs, seed = 16, 64, 32, 5
    u8 = np.random.default_rng(N).integers(0, 256, (N, 3, 24, 20), dtype=np.uint8)  # colour cache, grayscale context
    ds = DeviceDataset(ctx, u8)
    P = A.init_params(S, d, np.random.default_rng(1)) * 10
    hyper = A.ae_hyper_default()
    a = make_ae(ctx, S, d, P)
    hist = A.train(a, ds, hyper, batch_size=bs, epochs=2, seed=seed, log=None)
    b = make_ae(ctx, S, d, P)
    rng, step, want = np.random.default_rng(seed), 0, []
    for _ in range(2):
        losses = []
        for idx in A.epoch_batches(N, bs, rng):
            losses.append(b.train_step(hyper, ds.gather(idx, S), seed=(seed << 32) + step)["loss"])
            step += 1
        want.append(float(np.mean(np.array(losses, np.float32).astype(np.float64))))
    assert step == 2 * 3 and hist == want
    np.testing.assert_array_equal(a.get_params(), b.get_params())
    for x, y in zip(a.get_adam_state(), b.get_adam_state()):
        np.testing.assert_array_equal(x, y)
    assert a.get_adam_state()[2] == step
    a.close()
    b.close()
    ds.close()


def test_reconstruct_and_encode(ctx):
    S, d, N = 32, 256, 70
    case = R.make_case(S, N, d, seed=31)
    ae = make_ae(ctx, S, d, case["P"])
    x = case["images"]
    full = ae.reconstruct(x, chunk=256)
    np.testing.assert_array_equal(full, ae.reconstruct(x, chunk=32))
    np.testing.assert_array_equal(full, ae.reconstruct(x, chunk=7))
    for s in range(0, N, 32):
        code, out = ae.forward(x[s:s + 32], training=False)
        np.testing.assert_array_equal(out, full[s:s + 32])
        np.testing.assert_array_equal(code, ae.encode(x)[s:s + 32])
    assert R.relerr(full, R.forward(case["P"], x, None, S, d)["y"]) < 1e-4
    live = ae.reconstruct(x, chunk=256, training=True, seed=9)  # getSamples: Dropout stays live
    assert R.relerr(live, full) > 1e-3
    np.testing.assert_array_equal(live, ae.forward(x, training=True, seed=9)[1])
    np.testing.assert_array_equal(ae.reconstruct(x, chunk=35, training=True, seed=9)[35:], ae.forward(x[35:], training=True, seed=10)[1])
    ae.close()


def test_relu_tanh_abs_ops_host_and_device(ctx):
    lib, h = ctx.lib, ctx.h
    n = 5000
    rng = np.random.default_rng(4)
    x = rng.standard_normal(n).astype(np.float32)
    x[:10] = 0.0
    dy = rng.standard_normal(n).astype(np.float32)
    t = x + rng.choice([-0.5, 0.0, 0.25], n).astype(np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    x64, dy64, t64 = x.astype(np.float64), dy.astype(np.float64), t.astype(np.float64)
    want = dict(relu_f=np.maximum(x64, 0), relu_b=np.where(x64 > 0, dy64, 0), tanh_f=np.tanh(x64),
                tanh_b=dy64 * (1 - np.tanh(x64).astype(np.float32).astype(np.float64) ** 2), abs_f=np.abs(x64 - t64).mean(),
                abs_b=np.where(x64 - t64 >= 0, 1.0, -1.0) / n)
    y_tanh = np.tanh(x64).astype(np.float32)

    def run(dev):
        bufs = []

        def inp(a):
            if not dev:
                return p(a)
            q = lib.fg_dev_alloc(a.nbytes)
            bufs.append(q)
            assert lib.fg_memcpy(h, C.c_void_p(q), p(a), a.nbytes) == 0
            return C.c_void_p(q)

        def call(fn, ins, n_out, n_before_out=False):
            out = np.empty(n_out, np.float32)
            o = inp(out)
            rc = fn(h, *ins, n, o) if n_before_out else fn(h, *ins, o, n)
            assert rc == 0, lib.fg_last_error()
            if dev:
                assert lib.fg_memcpy(h, p(out), o, out.nbytes) == 0
                ctx.sync()
            return out

        got = dict(relu_f=call(lib.fg_relu_forward, [inp(x)], n), relu_b=call(lib.fg_relu_backward, [inp(x), inp(dy)], n),
                   tanh_f=call(lib.fg_tanh_forward, [inp(x)], n), tanh_b=call(lib.fg_tanh_backward, [inp(y_tanh), inp(dy)], n),
                   abs_f=call(lib.fg_abs_forward, [inp(x), inp(t)], 1, True)[0],
                   abs_b=call(lib.fg_abs_backward, [inp(x), inp(t)], n, True))
        for q in bufs:
            lib.fg_dev_free(C.c_void_p(q))
        return got

    for dev in (False, True):
        got = run(dev)
        np.testing.assert_array_equal(got["relu_f"], want["relu_f"].astype(np.float32))
        np.testing.assert_array_equal(got["relu_b"], want["relu_b"].astype(np.float32))
        np.testing.assert_allclose(got["tanh_f"], want["tanh_f"], rtol=2e-6, atol=1e-7)
        np.testing.assert_allclose(got["tanh_b"], want["tanh_b"], rtol=2e-6, atol=1e-7)
        assert abs(got["abs_f"] - want["abs_f"]) <= 1e-6 * want["abs_f"]
        np.testing.assert_array_equal(got["abs_b"], want["abs_b"].astype(np.float32))


def test_refusals_leave_the_context_usable(ctx, ctx3):
    import face_generator_b200 as fg
    from face_generator_b200.autoencoder import Autoencoder, ae_hyper_default
    lib = ctx.lib

    def refused(code, fn):
        with pytest.raises(fg.FGError, match=r"\(%d\)" % code) as e:
            fn()
        assert len(str(e.value).split(": ", 1)[1]) > 10  # fg_last_error says why
        return str(e.value)

    assert "grayscale" in refused(-4, lambda: Autoencoder(ctx3, 32, 256))
    for size in (8, 24, 64):
        refused(-4, lambda: Autoencoder(ctx, size, 256))
    for d in (0, 4, 12, 260, 1032):
        assert "multiple of 8" in refused(-4, lambda: Autoencoder(ctx, 32, d))
    Autoencoder(ctx, 32, 8).close()
    Autoencoder(ctx, 16, 1024).close()
    S, d = 16, 64
    case = R.make_case(S, 4, d, seed=1)
    ae = make_ae(ctx, S, d, case["P"])
    hyper = ae_hyper_default()
    big = np.zeros((257, 1, S, S), np.float32)
    refused(-1, lambda: ae.train_step(hyper, big))
    refused(-1, lambda: ae.forward(big))
    refused(-1, lambda: ae.train_step(hyper, C.c_void_p(1).value, B=0))
    refused(-1, lambda: ae.reconstruct(case["images"], chunk=257))
    refused(-1, lambda: ae.train_step(ae_hyper_default(p_drop=1.0), case["images"]))
    before = lib.fg_kernel_launches(ctx.h)
    refused(-5, lambda: ae.backward(np.zeros_like(case["images"])))  # nothing to differentiate yet
    assert lib.fg_kernel_launches(ctx.h) == before
    st = ae.train_step(hyper, case["images"], masks=case["masks"])
    assert st["t"] == 1 and np.isfinite(st["loss"])
    ae.close()


def test_export_and_reload_give_identical_reconstructions(ctx, tmp_path):
    from face_generator_b200.autoencoder import ae_hyper_default
    from face_generator_b200.checkpoint import load_autoencoder_flat, save_autoencoder_flat
    S, B, d = 16, 32, 64
    case = R.make_case(S, B, d, seed=41)
    hyper = ae_hyper_default()
    a = make_ae(ctx, S, d, case["P"])
    for k in range(3):
        a.train_step(hyper, case["images"], seed=k)
    path = str(tmp_path / "autoencoder_flat.t7")
    save_autoencoder_flat(a, path, epoch=4)
    b = make_ae(ctx, S, d, np.zeros_like(case["P"]))
    assert load_autoencoder_flat(b, path) == 4
    np.testing.assert_array_equal(a.reconstruct(case["images"]), b.reconstruct(case["images"]))
    sa, sb = a.train_step(hyper, case["images"], seed=3), b.train_step(hyper, case["images"], seed=3)
    assert sa == sb and sa["t"] == 4
    np.testing.assert_array_equal(a.get_params(), b.get_params())
    a.close()
    b.close()


def test_other_nets_are_untouched(ctx, ctx3):
    """runs last: fg_train_step on the 3-channel context created before every autoencoder above is bit for bit the
    step of a fresh context with the same state"""
    import face_generator_b200 as fg
    B = 16
    rng = np.random.default_rng(0)
    real = rng.uniform(0, 1, (B // 2, 3, 32, 32)).astype(np.float32)
    nD = rng.uniform(-1, 1, (B // 2, 100)).astype(np.float32)
    nG = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
    PG = (rng.standard_normal(ctx3.count(fg.lib.NET_G)) * 0.02).astype(np.float32)
    PD = (rng.standard_normal(ctx3.count(fg.lib.NET_D)) * 0.02).astype(np.float32)
    hyper = fg.hyper_default()
    fresh = fg.Context(0, max_batch=64, channels=3)
    outs = []
    for c in (ctx3, fresh):
        c.set_params(fg.lib.NET_G, PG)
        c.set_params(fg.lib.NET_D, PD)
        st = [c.train_step(hyper, B, real, nD, nG, seed=5) for _ in range(2)]
        outs.append((st, c.get_params(fg.lib.NET_G), c.get_params(fg.lib.NET_D)))
    fresh.close()
    assert outs[0][0] == outs[1][0]
    np.testing.assert_array_equal(outs[0][1], outs[1][1])
    np.testing.assert_array_equal(outs[0][2], outs[1][2])
