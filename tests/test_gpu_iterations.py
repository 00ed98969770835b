"""Several D and G iterations per call (train.lua / train_c2f.lua --D_iterations, --G_iterations) on the GPU.

  identity     *_iters(1, 1) is bitwise the single-iteration entry, host- and device-fed, for every trainer
  composition  fused (d, g) == the same sequence composed from the L-net calls (test_modules_equal_fused_step's bars)
  gate         the accuracy gate decides per D iteration inside one call; conf / trained_D add up
  device feed  *_dataset_iters == *_iters on the inputs rebuilt on the host from the documented streams, bitwise
  replay       a replayed graph == an eager call, bitwise; the device-fed graph holds the draws (kernel counts)
  recreate     a destroyed and recreated dataset is never read through a graph captured on the old one
  s16 / c2f    fused (d, g) == the composition from the fg_s16_* / fg_c2f_* L-net calls, s16 also at batch 256
  oracle       every iteration of the composition against the fp64 oracle at 1e-4
  DP           two GPUs, (2, 1), dp_overlap on and off: bit-identical replicas (skipped on one GPU)
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import parity_utils as PU  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fg():
    import face_generator_b200 as fg
    return fg


def _state(net, bn=True):
    from face_generator_b200.lib import NET_D, NET_G
    out = []
    for k in (NET_G, NET_D):
        m, v, t = net.get_adam_state(k)
        out += [net.get_params(k), net.get_grads(k), m, v, np.array([t])]
    if bn:
        out.append(net.get_bn_state())
    return out


def _assert_same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def _init(net, seed):
    from face_generator_b200.lib import NET_D, NET_G
    rng = np.random.default_rng(seed)
    net.set_params(NET_G, (rng.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32))
    net.set_params(NET_D, (rng.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32))


def _trainer(fg, kind, ctx):
    """(net, side, uses BatchNorm) of one trainer: "32" = the ctx's own 32x32 nets, "s16", "c2f32" / "c2f64"."""
    if kind == "32":
        return ctx, 32, True
    if kind == "s16":
        return fg.S16(ctx), 16, True
    S = int(kind[3:])
    return fg.C2f(ctx, S), S, False


def _host_inputs(rng, kind, net, B, d, g, C):
    """stacked random inputs of one call (masks drawn from the seed)"""
    f = lambda a: np.ascontiguousarray(a, np.float32)
    Bh = B // 2
    if kind in ("32", "s16"):
        S = 32 if kind == "32" else 16
        return [f(rng.random((d, Bh, C, S, S))), f(rng.uniform(-1, 1, (d, Bh, 100))), f(rng.uniform(-1, 1, (g, B, 100)))]
    S = net.S
    return [f(rng.uniform(-0.3, 0.3, (d, Bh, C, S, S))), f(rng.random((d, B, C, S, S))),
            f(rng.uniform(-1, 1, (d, Bh, 1, S, S))), f(rng.random((g, B, C, S, S))), f(rng.uniform(-1, 1, (g, B, 1, S, S)))]


def _call_iters(net, kind, hyper, B, d, g, inp, seed):
    return net.train_step_iters(hyper, B, d, g, *inp, None, None, seed)


def _call_single(net, kind, hyper, B, inp, seed):
    one = [a[0] for a in inp]
    return net.train_step(hyper, B, *one, None, None, seed)


TRAINERS = [("32", 3), ("32", 1), ("s16", 3), ("c2f32", 3), ("c2f64", 3)]


# ---- (1) identity at 1 + 1 ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,C", TRAINERS)
def test_iters_1x1_is_the_single_iteration_step(fg, kind, C):
    """Three calls (eager, captured, replayed) of *_iters(1, 1) == three single-iteration calls, bitwise: parameters,
    gradients, moments, step counters, BN running statistics and every statistics field."""
    B = 32
    res = []
    for mode in ("iters", "single"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net, _, bn = _trainer(fg, kind, ctx)
        _init(net, 7)
        hyper = fg.hyper_default()
        rng = np.random.default_rng(8)
        stats = []
        for seed in (11, 12, 13):
            inp = _host_inputs(rng, kind, net, B, 1, 1, C)
            if mode == "iters":
                stats.append(_call_iters(net, kind, hyper, B, 1, 1, inp, seed))
            else:
                stats.append(_call_single(net, kind, hyper, B, inp, seed))
        res.append((stats, _state(net, bn)))
        if net is not ctx:
            net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])


def _dataset_call(fg, kind, net, ds, hyper, B, d, g, seed, cs=8, iters=True):
    if kind == "32":
        return ds.train_step_iters(hyper, B, d, g, seed) if iters else ds.train_step(hyper, B, seed)
    if kind == "s16":
        return net.train_step_dataset_iters(ds, hyper, B, d, g, seed) if iters else net.train_step_dataset(ds, hyper, B, seed)
    return net.train_step_dataset_iters(ds, hyper, B, d, g, cs, seed) if iters else net.train_step_dataset(ds, hyper, B, cs, seed)


@pytest.mark.parametrize("kind,C", TRAINERS)
def test_dataset_iters_1x1_is_the_single_iteration_dataset_step(fg, kind, C):
    from face_generator_b200.dataset import DeviceDataset
    B = 32
    imgs = np.random.default_rng(20).integers(0, 256, (200, 3, 64, 64), dtype=np.uint8)
    res = []
    for iters in (True, False):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net, _, bn = _trainer(fg, kind, ctx)
        _init(net, 21)
        ds = DeviceDataset(ctx, imgs)
        hyper = fg.hyper_default()
        stats = [_dataset_call(fg, kind, net, ds, hyper, B, 1, 1, seed, iters=iters) for seed in (3, 4, 5)]
        res.append((stats, _state(net, bn)))
        ds.close()
        if net is not ctx:
            net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])


# ---- (4) device feed == host feed on the documented streams ----------------------------------------------------------
def _rebuilt_inputs(ctx, ds, kind, net, B, d, g, seed, cs=8):
    """the inputs of *_dataset_iters(d, g, seed), rebuilt with fg_dataset_draw / fg_dataset_gather* / fg_noise_uniform
    from the stream roots of fg_b200.h"""
    from face_generator_b200.dataset import noise_uniform
    from face_generator_b200.lib import iteration_root
    Bh = B // 2
    r = [iteration_root(seed, j) for j in range(max(d, g))]
    m = 2 ** 64
    if kind in ("32", "s16"):
        S = 32 if kind == "32" else 16
        real = np.stack([ds.gather(ds.draw((4 * r[j]) % m, Bh), S) for j in range(d)])
        nD = np.stack([noise_uniform(ctx, (4 * r[j] + 1) % m, (Bh, 100)) for j in range(d)])
        nG = np.stack([noise_uniform(ctx, (4 * r[j] + 2) % m, (B, 100)) for j in range(g)])
        return [real, nD, nG]
    S = net.S
    rd, cD, nD, cG, nG = [], [], [], [], []
    for j in range(d):
        _, cr, dr = ds.gather_c2f(ds.draw((8 * r[j]) % m, Bh), cs, S)
        _, cf, _ = ds.gather_c2f(ds.draw((8 * r[j] + 1) % m, Bh), cs, S)
        rd.append(dr)
        cD.append(np.concatenate([cr, cf]))
        nD.append(noise_uniform(ctx, (8 * r[j] + 3) % m, (Bh, 1, S, S)))
    for j in range(g):
        _, cg, _ = ds.gather_c2f(ds.draw((8 * r[j] + 2) % m, B), cs, S)
        cG.append(cg)
        nG.append(noise_uniform(ctx, (8 * r[j] + 4) % m, (B, 1, S, S)))
    return [np.ascontiguousarray(np.stack(a), np.float32) for a in (rd, cD, nD, cG, nG)]


@pytest.mark.parametrize("kind,C", [("32", 3), ("s16", 1), ("c2f32", 3), ("c2f64", 1)])
@pytest.mark.parametrize("d,g", [(2, 2), (3, 1)])
def test_dataset_iters_equal_host_iters_on_the_documented_streams(fg, kind, C, d, g):
    from face_generator_b200.dataset import DeviceDataset
    B = 32
    imgs = np.random.default_rng(30).integers(0, 256, (300, 3, 64, 64), dtype=np.uint8)
    res = []
    for mode in ("device", "host"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net, _, bn = _trainer(fg, kind, ctx)
        _init(net, 31)
        ds = DeviceDataset(ctx, imgs)
        hyper = fg.hyper_default()
        stats = []
        for seed in (6, 7, 8):  # eager, captured, replayed
            if mode == "device":
                stats.append(_dataset_call(fg, kind, net, ds, hyper, B, d, g, seed))
            else:
                stats.append(_call_iters(net, kind, hyper, B, d, g, _rebuilt_inputs(ctx, ds, kind, net, B, d, g, seed), seed))
        res.append((stats, _state(net, bn)))
        ds.close()
        if net is not ctx:
            net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])


def test_iteration_roots_do_not_collide():
    from face_generator_b200.lib import iteration_root
    roots = {iteration_root(s, j) for s in range(200) for j in range(16)}
    assert len(roots) == 200 * 16
    assert iteration_root(12345, 0) == 12345


# ---- (5) replay == eager; the device-fed call is one graph --------------------------------------------------------
@pytest.mark.parametrize("kind", ["32", "s16", "c2f32"])
def test_replayed_iters_equal_eager_iters(fg, kind):
    from face_generator_b200.dataset import DeviceDataset
    B, C, d, g = 32, 3, 2, 2
    imgs = np.random.default_rng(40).integers(0, 256, (200, 3, 64, 64), dtype=np.uint8)
    res = []
    for use_graph in (1, 0):
        ctx = fg.Context(0, max_batch=B, channels=C)
        ctx.set_option("use_graph", use_graph)
        net, _, bn = _trainer(fg, kind, ctx)
        _init(net, 41)
        ds = DeviceDataset(ctx, imgs)
        hyper = fg.hyper_default()
        rng = np.random.default_rng(42)
        stats, launches, host_launches = [], [], []
        for seed in (1, 2, 3):
            l0 = ctx.launches()
            stats.append(_call_iters(net, kind, hyper, B, d, g, _host_inputs(rng, kind, net, B, d, g, C), seed))
            host_launches.append(ctx.launches() - l0)
        for seed in (4, 5, 6):
            l0 = ctx.launches()
            stats.append(_dataset_call(fg, kind, net, ds, hyper, B, d, g, seed))
            launches.append(ctx.launches() - l0)
        res.append((stats, _state(net, bn), launches, host_launches))
        ds.close()
        if net is not ctx:
            net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])
    # A replayed call counts its graph's kernels plus the seed upload.  The replayed device-fed call must count exactly
    # the replayed host-fed call's kernels plus its draws -- draw + gather + noise per D iteration and a noise per G
    # iteration (c2f: two draw + gather pairs and a noise per D iteration, draw + gather + noise per G iteration).  Draws
    # launched eagerly before an unchanged graph would be missing from the graph and the totals would not add up.
    draws = 5 * d + 3 * g if kind.startswith("c2f") else 3 * d + g
    assert res[0][2][2] == res[0][3][2] + draws, (res[0][2], res[0][3], draws)


# ---- (2) / (6) composition from the L-net calls ------------------------------------------------------------------------
def _iters_case(B, C, d, g, seed):
    case = PU.make_case(B, C, seed=seed, init="smooth")
    rng = np.random.default_rng(seed + 1000)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    case["reals"] = f(np.stack([case["real"]] + [rng.random(case["real"].shape) for _ in range(d - 1)]))
    case["noises_D"] = f(np.stack([case["noise_D"]] + [rng.uniform(-1, 1, case["noise_D"].shape) for _ in range(d - 1)]))
    case["noises_G"] = f(np.stack([case["noise_G"]] + [rng.uniform(-1, 1, case["noise_G"].shape) for _ in range(g - 1)]))
    case["masks_Ds"] = f(np.stack([PU.make_masks(B, rng) for _ in range(d)]))
    case["masks_Gs"] = f(np.stack([PU.make_masks(B, rng) for _ in range(g)]))
    return case


def _fused_vs_modules(fg, B, C, d, g, seed, hyper):
    from face_generator_b200 import adversarial as A
    from face_generator_b200.lib import NET_D, NET_G
    case = _iters_case(B, C, d, g, seed)
    res = {}
    for mode in ("fused", "modules"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        if mode == "fused":
            st = ctx.train_step_iters(hyper, B, d, g, case["reals"], case["noises_D"], case["noises_G"], case["masks_Ds"],
                                      case["masks_Gs"])
        else:
            st = A.train_batch_iters_modules(ctx, hyper, case["reals"], case["noises_D"], case["noises_G"],
                                             case["masks_Ds"], case["masks_Gs"])
        res[mode] = (st, [ctx.get_params(NET_D), ctx.get_params(NET_G)], [ctx.get_grads(NET_D), ctx.get_grads(NET_G)],
                     ctx.get_bn_state(), [ctx.get_adam_state(NET_D)[2], ctx.get_adam_state(NET_G)[2]])
        ctx.close()
    return res


def _assert_close(res, lr_allowance=2.1e-3, check_grad_D=True):
    """check_grad_D = False when the last D iteration's gate was closed: the fused step leaves the penalised, clamped
    gradient behind (fevalD penalises and clamps before it decides), the composition skips the optimizer call"""
    f, m = res["fused"], res["modules"]
    for a, b in list(zip(f[2], m[2]))[0 if check_grad_D else 1:]:
        assert PU.relerr(a, b) < 2e-5, PU.relerr(a, b)
    for a, b in zip(f[1], m[1]):
        assert np.abs(a - b).max() < lr_allowance  # sign flips of noise-level gradients move a parameter by 2*lr
    # BN running statistics after d + g training-mode G forwards
    assert PU.relerr(f[3], m[3]) < 1e-5, PU.relerr(f[3], m[3])


@pytest.mark.parametrize("d,g", [(2, 1), (1, 2), (3, 2)])
def test_fused_iters_equal_lnet_composition(fg, d, g):
    hyper = fg.hyper_default()
    res = _fused_vs_modules(fg, 8, 3, d, g, 61 + 10 * d + g, hyper)
    _assert_close(res)
    st, mod = res["fused"][0], res["modules"][0]
    assert st["trained_D"] == d and st["t_D"] == d and st["t_G"] == g
    assert res["fused"][4] == res["modules"][4] == [d, g]
    assert sum(st["conf"]) == d * 8
    assert abs(st["loss_G"] - mod["loss_G"][-1]) < 1e-4 * max(1.0, abs(mod["loss_G"][-1]))


def test_fused_iters_equal_lnet_composition_at_batch_256(fg):
    """the headline size: (2, 1) at batch 256"""
    res = _fused_vs_modules(fg, 256, 3, 2, 1, 77, fg.hyper_default())
    _assert_close(res)


# ---- (3) the gate inside one call --------------------------------------------------------------------------------
def test_gate_closed_leaves_D_untouched(fg):
    from face_generator_b200.lib import NET_D
    B, C, d = 16, 3, 3
    ctx = fg.Context(0, max_batch=B, channels=C)
    _init(ctx, 50)
    rng = np.random.default_rng(51)
    inp = _host_inputs(rng, "32", ctx, B, d, 1, C)
    before = [ctx.get_params(NET_D), *ctx.get_adam_state(NET_D)[:2]]
    st = ctx.train_step_iters(fg.hyper_default(D_maxAcc=0.0), B, d, 1, *inp, None, None, 9)
    assert st["trained_D"] == 0 and st["t_D"] == 0 and st["t_G"] == 1
    assert sum(st["conf"]) == d * B
    _assert_same(before, [ctx.get_params(NET_D), *ctx.get_adam_state(NET_D)[:2]])
    st = ctx.train_step_iters(fg.hyper_default(D_maxAcc=1.01), B, d, 1, *inp, None, None, 10)
    assert st["trained_D"] == d and st["t_D"] == d and sum(st["conf"]) == d * B
    ctx.close()


def test_gate_decides_per_iteration(fg):
    """a data-dependent threshold whose decision changes inside one call: the fused call's per-iteration decisions
    (trained_D, t_D and the resulting parameters) match the L-net composition gated by the transcription of
    adversarial.lua:154-178 (interval 1: the gate sees each iteration's own accuracy)"""
    from face_generator_b200 import adversarial as A
    d, g, B, C = 4, 1, 8, 3
    found = None
    for thr in np.arange(1, 16) / 16.0:
        hyper = fg.hyper_default(D_maxAcc=float(thr), accs_interval=1)
        res = _fused_vs_modules(fg, B, C, d, g, 91, hyper)
        trained = res["modules"][0]["trained"]
        if any(trained) and not all(trained):
            found = (thr, res)
            break
    assert found is not None, "no threshold straddles a gate change for this case"
    thr, res = found
    mod, st = res["modules"][0], res["fused"][0]
    accs = []
    assert [A.gate(accs, a, thr, 1) for a in mod["acc_D"]] == mod["trained"]
    assert st["trained_D"] == sum(mod["trained"]) and st["t_D"] == sum(mod["trained"])
    assert abs(st["acc_D"] - mod["acc_D"][-1]) < 1e-6
    _assert_close(res, check_grad_D=mod["trained"][-1])


# ---- a destroyed dataset invalidates the captured device-fed steps ------------------------------------------------------
@pytest.mark.parametrize("kind", ["32", "s16", "c2f32"])
def test_recreated_dataset_does_not_replay_a_stale_graph(fg, kind):
    """The device-fed multi-iteration graph holds the dataset's device buffers and size.  Destroy the dataset after the
    graph is captured and replayed, create one of another size (its host object often lands at the same address),
    and call again with the same (B, d, g, hyper): the step must draw from the new dataset, bitwise as the host-fed
    step on the inputs rebuilt from it."""
    from face_generator_b200.dataset import DeviceDataset
    B, C, d, g = 32, 3, 2, 1
    imgs1 = np.random.default_rng(70).integers(0, 256, (300, 3, 64, 64), dtype=np.uint8)
    imgs2 = np.random.default_rng(71).integers(0, 256, (37, 3, 64, 64), dtype=np.uint8)
    res = []
    for mode in ("device", "host"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net, _, bn = _trainer(fg, kind, ctx)
        _init(net, 72)
        hyper = fg.hyper_default()
        ds = DeviceDataset(ctx, imgs1)
        for seed in (1, 2, 3):  # eager, captured, replayed: both modes alike
            _dataset_call(fg, kind, net, ds, hyper, B, d, g, seed)
        ds.close()
        ds = DeviceDataset(ctx, imgs2)
        stats = []
        for seed in (4, 5):
            if mode == "device":
                stats.append(_dataset_call(fg, kind, net, ds, hyper, B, d, g, seed))
            else:
                stats.append(_call_iters(net, kind, hyper, B, d, g, _rebuilt_inputs(ctx, ds, kind, net, B, d, g, seed), seed))
        res.append((stats, _state(net, bn)))
        ds.close()
        if net is not ctx:
            net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])


# ---- (2) / (6) composition on the --scale 16 and coarse-to-fine nets ---------------------------------------------------
NO_PEN = dict(D_L1=0.0, D_L2=0.0, G_L1=0.0, G_L2=0.0, D_clamp=0.0, G_clamp=0.0)  # raw gradients on both paths


def _s16_compose(net, hyper, real, nD, nG, mD, mG):
    """fevalD / fevalG_on_D per iteration from the fg_s16_* L-net calls, optim.adam steps by fg_adam_step"""
    from face_generator_b200.adversarial_c2f import AdamState
    from face_generator_b200.lib import NET_D, NET_G
    ctx = net.ctx
    Bh = real.shape[1]
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)]).astype(np.float32)
    opt = {k: AdamState(net, k) for k in (NET_D, NET_G)}
    for j in range(real.shape[0]):
        fake = net.G_forward(nD[j])
        net.zero_grads(NET_D)
        out = net.D_forward(np.concatenate([real[j], fake]), masks=mD[j])
        net.D_backward(ctx.bce_backward(out, targets), want_wgrad=True, want_dimg=False)
        opt[NET_D].step(hyper)
    for j in range(nG.shape[0]):
        net.zero_grads(NET_G)
        img = net.G_forward(nG[j])
        out = net.D_forward(img, masks=mG[j])
        net.G_backward(net.D_backward(ctx.bce_backward(out, np.ones(2 * Bh, np.float32)), want_wgrad=False, want_dimg=True))
        opt[NET_G].step(hyper)
    for o in opt.values():
        o.close()


def _stack(first, rng, make, n):
    return np.ascontiguousarray(np.stack([first] + [make(rng) for _ in range(n - 1)]), np.float32)


def _close_pair(a, b, steps):
    """a, b: (params D, params G, grads D, grads G[, bn]) of the fused call and the composition"""
    for x, y in zip(a[2:4], b[2:4]):
        assert PU.relerr(x, y) < 2e-5, PU.relerr(x, y)
    for x, y in zip(a[:2], b[:2]):
        dd = np.abs(x.astype(np.float64) - y)
        # sign flips of noise-level gradients move a parameter by 2*lr per optimizer step
        assert dd.max() < 2.1e-3 * steps and np.mean(dd > 1e-5) < 0.01, (dd.max(), np.mean(dd > 1e-5))
    if len(a) > 4:
        assert PU.relerr(a[4], b[4]) < 1e-5, PU.relerr(a[4], b[4])


@pytest.mark.parametrize("B,d,g", [(8, 2, 1), (8, 1, 2), (8, 3, 2), (256, 2, 1)])
def test_s16_fused_iters_equal_lnet_composition(fg, B, d, g):
    import s16_utils as SU
    from oracle import oracle_s16 as OS
    from face_generator_b200.lib import NET_D, NET_G
    C = 3
    case = SU.make_case(B, C, seed=300 + 10 * d + g, init="smooth")
    rng = np.random.default_rng(301)
    mask = lambda r: r.random((B, OS.MASK_PER_SAMPLE)) < 0.5
    real = _stack(case["real"], rng, lambda r: r.random((B // 2, C, 16, 16)), d)
    nD = _stack(case["noise_D"], rng, lambda r: r.uniform(-1, 1, (B // 2, 100)), d)
    nG = _stack(case["noise_G"], rng, lambda r: r.uniform(-1, 1, (B, 100)), g)
    mD, mG = _stack(case["masks_D"], rng, mask, d), _stack(case["masks_G"], rng, mask, g)
    hyper = fg.hyper_default(**NO_PEN)
    res = {}
    for mode in ("fused", "modules"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net = fg.S16(ctx)
        net.set_params(NET_G, case["PG"])
        net.set_params(NET_D, case["PD"])
        if mode == "fused":
            st = net.train_step_iters(hyper, B, d, g, real, nD, nG, mD, mG)
            assert st["trained_D"] == d and st["t_D"] == d and st["t_G"] == g and sum(st["conf"]) == d * B
        else:
            _s16_compose(net, hyper, real, nD, nG, mD, mG)
        res[mode] = (net.get_params(NET_D), net.get_params(NET_G), net.get_grads(NET_D), net.get_grads(NET_G),
                     net.get_bn_state())
        net.close()
        ctx.close()
    _close_pair(res["fused"], res["modules"], max(d, g))


@pytest.mark.parametrize("S,d,g", [(32, 2, 1), (32, 1, 2), (32, 3, 2), (16, 2, 1)])
def test_c2f_fused_iters_equal_lnet_composition(fg, S, d, g):
    from face_generator_b200 import adversarial_c2f as AC
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_D, NET_G
    B, C = 8, 3
    rng = np.random.default_rng(400 + S + 10 * d + g)
    probe = fg.Context(0, max_batch=B, channels=C)
    pnet = fg.C2f(probe, S)
    mps, nG_, nD_ = pnet.mask_per_sample, pnet.count(NET_G), pnet.count(NET_D)
    pnet.close()
    probe.close()
    PG = np.ascontiguousarray(LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.0, slope=1.0), np.float32)
    PD_full = LY.trained_like_init(LY.c2f_D_layout(C), rng, 0.8, slope=1.0) if S == 32 else None
    PD = np.ascontiguousarray(PD_full if PD_full is not None else rng.standard_normal(nD_) * 0.02, np.float32)
    assert PG.size == nG_ and PD.size == nD_

    def pairs(n):
        if S == 32:
            return LY.c2f_pairs(n, C, rng)
        return (rng.uniform(-0.3, 0.3, (n, C, S, S)).astype(np.float32), rng.random((n, C, S, S)).astype(np.float32))

    f = lambda a: np.ascontiguousarray(np.stack(a), np.float32)
    rd, cD, zD, cG, zG = [], [], [], [], []
    for _ in range(d):
        diff, cr = pairs(B // 2)
        _, cf = pairs(B // 2)
        rd.append(diff)
        cD.append(np.concatenate([cr, cf]))
        zD.append(rng.uniform(-1, 1, (B // 2, 1, S, S)))
    for _ in range(g):
        cG.append(pairs(B)[1])
        zG.append(rng.uniform(-1, 1, (B, 1, S, S)))
    rd, cD, zD, cG, zG = (f(a) for a in (rd, cD, zD, cG, zG))
    mD = f([rng.random((B, mps)) < 0.5 for _ in range(d)])
    mG = f([rng.random((B, mps)) < 0.5 for _ in range(g)])
    hyper = fg.hyper_default(**NO_PEN)
    res = {}
    for mode in ("fused", "modules"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net = fg.C2f(ctx, S)
        net.set_params(NET_G, PG)
        net.set_params(NET_D, PD)
        if mode == "fused":
            st = AC.train_batch_iters(net, hyper, rd, cD, zD, cG, zG, mD, mG)
            assert st["trained_D"] == d and st["t_D"] == d and st["t_G"] == g and sum(st["conf"]) == d * B
        else:
            AC.train_batch_iters_modules(net, hyper, rd, cD, zD, cG, zG, mD, mG)
        res[mode] = (net.get_params(NET_D), net.get_params(NET_G), net.get_grads(NET_D), net.get_grads(NET_G))
        net.close()
        ctx.close()
    _close_pair(res["fused"], res["modules"], max(d, g))


# ---- (2) every iteration of the composition against the fp64 oracle ----------------------------------------------------
@pytest.mark.parametrize("d,g", [(2, 1), (1, 2), (3, 2)])
def test_lnet_composition_iterations_match_fp64_oracle(fg, d, g):
    """Each D and G iteration of the composition (which the fused call matches, above) against the fp64 oracle's G / D
    forward / backward and BCE on the parameters that iteration ran on, at the project's 1e-4 bar; G's BatchNorm
    running statistics after all d + g training-mode G forwards, restated in fp64 alongside."""
    from face_generator_b200 import adversarial as A
    from face_generator_b200.lib import NET_D, NET_G
    from oracle import oracle as O
    B, C = 8, 3
    case = _iters_case(B, C, d, g, 500 + 10 * d + g)
    bn = PU.fresh_state(case)["bnG"]
    Bh = B // 2
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)])
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_params(NET_G, case["PG"])
    ctx.set_params(NET_D, case["PD"])
    checked = []

    def hook(kind, j, outputs):
        Gf, Df = O.f64.G(), O.f64.D()
        PG, PD = ctx.get_params(NET_G), ctx.get_params(NET_D)
        if kind == "D":
            fake = Gf.forward(PG, case["noises_D"][j], C, True, bn)
            out = Df.forward(PD, np.concatenate([case["reals"][j].astype(np.float64), fake]), case["masks_Ds"][j])
            ref, _ = Df.backward(O.f64.bce_bwd(out, targets), want_dimg=False)
            got = ctx.get_grads(NET_D)
        else:
            img = Gf.forward(PG, case["noises_G"][j], C, True, bn)
            out = Df.forward(PD, img, case["masks_Gs"][j])
            _, dimg = Df.backward(O.f64.bce_bwd(out, np.ones(B)), want_dP=False)
            ref = Gf.backward(dimg)
            got = ctx.get_grads(NET_G)
        assert PU.relerr(outputs.reshape(-1), out) < 1e-4, (kind, j, PU.relerr(outputs.reshape(-1), out))
        assert PU.relerr(got, ref) < 1e-4, (kind, j, PU.relerr(got, ref))
        checked.append((kind, j))

    A.train_batch_iters_modules(ctx, fg.hyper_default(), case["reals"], case["noises_D"], case["noises_G"],
                                case["masks_Ds"], case["masks_Gs"], hook=hook)
    assert checked == [("D", j) for j in range(d)] + [("G", j) for j in range(g)]
    assert PU.relerr(ctx.get_bn_state(), bn) < 1e-4, PU.relerr(ctx.get_bn_state(), bn)
    ctx.close()


# ---- (7) data parallel on two GPUs ----------------------------------------------------------------------------------
def _gpu_count():
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for line in out.splitlines() if line.startswith("GPU "))
    except Exception:
        return 0


def _dp_worker(rank, world, port, q):
    import torch.distributed as dist
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C, d, g = 16, 3, 2, 1
    base = _iters_case(B, C, d, g, 600)
    calls = [_iters_case(B, C, d, g, 601 + rank + 10 * s) for s in range(2)]  # rank-distinct shards
    res = []
    for overlap in (1, 0):
        ctx = fg.Context(rank, max_batch=B, channels=C)
        ctx.set_option("dp_overlap", overlap)
        ctx.set_params(NET_G, base["PG"])
        ctx.set_params(NET_D, base["PD"])
        ids = [ctx.dp_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        ctx.dp_init(ids[0], world, rank)
        ctx.dp_broadcast_params()
        sts = [ctx.train_step_iters(fg.hyper_default(), B, d, g, c["reals"], c["noises_D"], c["noises_G"], c["masks_Ds"],
                                    c["masks_Gs"], 3 + s) for s, c in enumerate(calls)]
        res.append((ctx.get_params(NET_D), ctx.get_params(NET_G), [list(s["conf"]) for s in sts],
                    [s["trained_D"] for s in sts]))
        dist.barrier()
        ctx.close()
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def test_dp_two_gpus_iters_keep_replicas_identical():
    """(2, 1) on two GPUs, dp_overlap on and off: every D iteration all-reduces before its gate and optimizer, so the
    replicas end bit-identical; conf is global and sums over the D iterations"""
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_dp_worker, args=(r, world, 29791, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r = q.get(timeout=600)
        got[r[0]] = r[1]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for mode in (0, 1):
        np.testing.assert_array_equal(got[0][mode][0], got[1][mode][0])
        np.testing.assert_array_equal(got[0][mode][1], got[1][mode][1])
        assert got[0][mode][2] == got[1][mode][2] and all(sum(c) == 2 * 16 * world for c in got[0][mode][2])
        assert got[0][mode][3] == [2, 2]
