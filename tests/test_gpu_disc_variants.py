"""GPU: create_D32 on the 32x32 nets and create_D16 / _b / _c on the --scale 16 nets against the float64 restatement
(tests/dbr_ref.py) at the 1e-4 normwise bar, and their train steps: bit-reproducible, graph replay equal to the eager
first call, device-fed, scored in chunks, and the side check."""
import ctypes as C

import numpy as np
import pytest
import torch

import dbr_ref as R

NAMES = ["create_D32", "create_D16", "create_D16_b", "create_D16_c"]
BAR = 1e-4
MARGIN = 1e-5  # pooling windows whose top two float64 candidates lie closer (relative to the layer's max) take the GPU's


def relerr(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def make(name, C_, max_batch):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=max_batch, channels=C_, discriminator=name if R.NETS[name][0] == 32 else "create_D32b")
    net = ctx if R.NETS[name][0] == 32 else fg.S16(ctx, discriminator=name)
    return ctx, net


def close(ctx, net):
    if net is not ctx:
        net.close()
    ctx.close()


def gpu_route(net_gpu, P, zget=None):
    """route hook of dbr_ref.MaxPool: the window's arg-max as the GPU took it (fp32 PReLU of its own pre-activation,
    first strict maximum) wherever the float64 top two lie within MARGIN.  zget(name): the GPU's pre-activation
    "<branch>.z<i>" (default: the "D.*" debug tensor of net_gpu's last D forward)"""
    if zget is None:
        zget = lambda n: net_gpu.debug_tensor("D." + n)

    def route(name, win, idx):
        bname, i = name.split(".")
        z = zget("%s.z%s" % (bname, i))
        B, Cc, Ho, Wo, _ = win.shape
        z = z[:B * Ho * 2 * Wo * 2 * Cc].reshape(B, Ho * 2, Wo * 2, Cc).transpose(0, 3, 1, 2)
        a = np.float32(P[slope_off[name]])
        h = np.where(z > 0, z, a * z).astype(np.float32)
        gw = R.MaxPool.windows(torch.from_numpy(h.astype(np.float64)))
        gidx = R.first_max(gw)
        w = win.numpy()
        top = np.sort(w, axis=-1)
        amb = (top[..., 3] - top[..., 2]) <= MARGIN * max(np.abs(w).max(), 1e-30)
        out = idx.clone()
        out[torch.from_numpy(amb)] = gidx[torch.from_numpy(amb)]
        route.count += int(amb.sum())
        return out
    route.count = 0
    slope_off = {}
    return route, slope_off


def pool_slopes(net):
    """MaxPool name -> offset of the PReLU slope in front of it"""
    out = {}
    for _, mods, _ in net.branches:
        for j, m in enumerate(mods):
            if isinstance(m, R.MaxPool):
                out[m.name] = mods[j - 1].off
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("C_", [1, 3])
@pytest.mark.parametrize("B", [6, 256])
def test_gpu_disc_forward_backward_against_float64(name, C_, B):
    ref = R.Net(name, C_)
    ctx, net = make(name, C_, 256)
    try:
        assert net.nD == ref.n_params and net.mask_per_sample == ref.mask
        rng = np.random.default_rng(B * 10 + C_)
        P = R.make_params(ref, 11 + C_)
        PG = rng.uniform(-0.05, 0.05, net.nG).astype(np.float32)
        net.set_params(1, P.astype(np.float32))
        net.set_params(0, PG)
        x = rng.uniform(0, 1, (B, C_, ref.side, ref.side)).astype(np.float32)
        keep = (rng.uniform(0, 1, (B, ref.mask)) >= 0.5).astype(np.float32)
        dout = rng.standard_normal(B).astype(np.float32)
        # evaluate()
        out_e = net.D_forward(x, training=False)
        route, offs = gpu_route(net, P)
        offs.update(pool_slopes(ref))
        ref_e, _, _, _ = R.run(ref, P, x, None, route=route)
        assert relerr(out_e, ref_e) < BAR
        # training with the given flags, forward and backward
        net.zero_grads(1)
        out = net.D_forward(x, masks=keep, training=True)
        dx = net.D_backward(dout, want_wgrad=True, want_dimages=True) if net is ctx else \
            net.D_backward(dout, want_wgrad=True, want_dimg=True)
        g = net.get_grads(1)
        route, offs = gpu_route(net, P)
        offs.update(pool_slopes(ref))
        ref_out, ref_dx, ref_g, rc = R.run(ref, P, x, keep, dout, route=route)
        errs = {"out": relerr(out, ref_out), "dx": relerr(dx, ref_dx)}
        for pname, off, n in ref.param_tensors():
            if pname.endswith(".a"):  # a PReLU slope: one sum of signed terms, whose rounding scales with the sum of their sizes
                errs[pname] = abs(float(g[off]) - ref_g[off]) / max(abs(ref_g[off]), rc.gabs[off], 1e-30)
            else:
                errs[pname] = relerr(g[off:off + n], ref_g[off:off + n])
        bad = {k: v for k, v in errs.items() if not v < BAR}
        assert not bad, (bad, route.count)
    finally:
        close(ctx, net)


def _state(net, seed):
    rng = np.random.default_rng(seed)
    ref = R.Net(net.discriminator, net.C)
    return dict(PD=R.make_params(ref, seed, near=False).astype(np.float32),
                PG=rng.uniform(-0.05, 0.05, net.nG).astype(np.float32))


def _reset(net, st):
    net.set_params(1, st["PD"])
    net.set_params(0, st["PG"])
    for k in (0, 1):
        z = np.zeros(net.count(k), np.float32)
        net.set_adam_state(k, z, z, 0)
    net.set_bn_state(np.concatenate([np.zeros(256), np.ones(256), np.zeros(128), np.ones(128)]).astype(np.float32))


def _snapshot(net, stats):
    m, v, t = net.get_adam_state(1)
    return [net.get_params(1), net.get_params(0), m, v, np.array(stats["conf"]), np.array([stats["loss_D"], stats["loss_G"]])]


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_disc_train_steps_are_bit_reproducible(name):
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset
    C_, B = 3, 16
    ctx, net = make(name, C_, B)
    try:
        S = R.NETS[name][0]
        st = _state(net, 5)
        rng = np.random.default_rng(3)
        real = rng.uniform(0, 1, (2, B // 2, C_, S, S)).astype(np.float32)
        nD = rng.uniform(-1, 1, (2, B // 2, 100)).astype(np.float32)
        nG = rng.uniform(-1, 1, (1, B, 100)).astype(np.float32)
        h = fg.hyper_default()
        runs = []
        for graph in (1, 1, 1, 0):  # eager first call (captured), two replays, no graph
            ctx.set_option("use_graph", graph)
            _reset(net, st)
            runs.append(_snapshot(net, net.train_step_iters(h, B, 2, 1, real, nD, nG, seed=9)))
        for r in runs[1:]:
            for a, b in zip(runs[0], r):
                np.testing.assert_array_equal(a, b)
        assert not np.array_equal(runs[0][0], st["PD"])  # D was stepped
        # device-fed: the captured step replays bit for bit
        imgs = rng.integers(0, 256, (40, C_, 32, 32), dtype=np.uint8)
        ds = DeviceDataset(ctx, imgs)
        ctx.set_option("use_graph", 1)
        feed = []
        for _ in range(3):
            _reset(net, st)
            feed.append(_snapshot(net, ds.train_step(h, B, 21) if net is ctx else net.train_step_dataset(ds, h, B, 21)))
        for r in feed[1:]:
            for a, b in zip(feed[0], r):
                np.testing.assert_array_equal(a, b)
        ds.close()
    finally:
        close(ctx, net)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_disc_score_equals_chunked_forward(name):
    from face_generator_b200.lib import _ptr
    C_, N, chunk = 3, 20, 8
    ctx, net = make(name, C_, chunk)
    try:
        S = R.NETS[name][0]
        net.set_params(1, _state(net, 2)["PD"])
        imgs = np.random.default_rng(1).uniform(0, 1, (N, C_, S, S)).astype(np.float32)
        preds = np.empty(N, np.float32)
        fn = ctx.lib.fg_D_score if net is ctx else ctx.lib.fg_s16_D_score
        for training in (0, 1):
            assert fn(net.h, _ptr(imgs), N, chunk, training, 77, _ptr(preds)) == 0
            for s in range(0, N, chunk):
                got = net.D_forward(imgs[s:s + chunk], training=bool(training), seed=77 + s)
                np.testing.assert_array_equal(preds[s:s + chunk], got)
    finally:
        close(ctx, net)


@pytest.mark.gpu
def test_gpu_disc_reported_and_side_checked():
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=8, channels=3)
    lib = ctx.lib
    assert lib.fg_get_disc(ctx.h) == 1 and ctx.nD == lib.fg_param_count(1, 3)
    s16 = fg.S16(ctx)
    assert lib.fg_s16_get_disc(s16.h) == 2 and s16.nD == lib.fg_s16_param_count(1, 3)
    h = C.c_void_p()
    assert lib.fg_s16_create_disc(ctx.h, 3, C.byref(h)) == -4 and not h.value  # create_D32 on the 16x16 nets
    assert b"32x32" in lib.fg_last_error()
    with pytest.raises(fg.FGError):
        fg.S16(ctx, discriminator="create_D32b")
    for name, disc in (("create_D16", 4), ("create_D16_b", 5), ("create_D16_c", 6)):
        n = fg.S16(ctx, discriminator=name)
        assert lib.fg_s16_get_disc(n.h) == disc
        n.close()
    s16.close()
    ctx.close()
    c32 = fg.Context(0, max_batch=8, channels=1, discriminator="create_D32")
    assert lib.fg_get_disc(c32.h) == 3 and c32.nD == lib.fg_disc_param_count(3, 1)
    c32.close()


# ---- one fused step against a float64 iteration: the oracle's G and the restated D ----------------------------------
NO_PEN = dict(D_L1=0.0, D_L2=0.0, G_L1=0.0, G_L2=0.0, D_clamp=0.0, G_clamp=0.0)  # raw gradients on both paths


def _compose_f64(name, C_, B, d, g, PG, PD, real, nD, nG, mD, mG, hp, routes=None):
    """adversarial.lua's loop body in float64: d D iterations (fevalD on real + G's fakes, Adam) then g G iterations
    (fevalG_on_D, Adam), G from the oracle, D from dbr_ref"""
    from oracle import oracle as O
    from oracle import oracle_s16 as OS
    T, S, Bh = O.f64, R.NETS[name][0], B // 2
    Gn = O.f64.G() if S == 32 else OS.f64.G()
    bn = np.concatenate([np.zeros(256), np.ones(256), np.zeros(128), np.ones(128)])
    gfwd = (lambda P, z: Gn.forward(P, z, C_, True, bn)) if S == 32 else (lambda P, z: Gn.forward(P, z, C_, bn))
    ref = R.Net(name, C_)
    st = dict(PD=PD.astype(np.float64), PG=PG.astype(np.float64))
    for k in ("mD", "vD", "mG", "vG"):
        st[k] = np.zeros(st["P" + k[1]].size)
    conf = np.zeros(4, np.int64)
    tgt = np.concatenate([np.ones(Bh), np.zeros(Bh)])
    adam = lambda x, gr, m, v, t, lr: T.adam(x, np.ascontiguousarray(gr, np.float64), m, v, t, lr, hp.beta1, hp.beta2, hp.eps)
    for j in range(d):
        x = np.concatenate([real[j], gfwd(st["PG"], nD[j])])
        rt = (routes or {}).get(("D", j))
        out = R.run(ref, st["PD"], x, mD[j], route=rt)[0]
        _, _, gD, _ = R.run(ref, st["PD"], x, mD[j], T.bce_bwd(out, tgt), route=rt)
        pred = out > 0.5
        conf += [np.sum(pred[:Bh]), np.sum(~pred[:Bh]), np.sum(pred[Bh:]), np.sum(~pred[Bh:])]
        adam(st["PD"], gD, st["mD"], st["vD"], j + 1, hp.lr_D)
    for j in range(g):
        img = gfwd(st["PG"], nG[j])
        rt = (routes or {}).get(("G", j))
        out = R.run(ref, st["PD"], img, mG[j], route=rt)[0]
        _, dx, _, _ = R.run(ref, st["PD"], img, mG[j], T.bce_bwd(out, np.ones(B)), route=rt)
        gG = Gn.backward(dx) if S == 16 else Gn.backward(dx, want_dnoise=False)
        adam(st["PG"], gG, st["mG"], st["vG"], j + 1, hp.lr_G)
    return st, conf


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("d,g", [(1, 1), (2, 1)])
def test_gpu_disc_train_step_iters_against_float64(name, d, g):
    import face_generator_b200 as fg
    import parity_utils as PU
    import s16_utils as SU
    C_, B = 3, 8
    S = R.NETS[name][0]
    ref = R.Net(name, C_)
    rng = np.random.default_rng(40 + d)
    PG = (PU.make_case(B, C_, seed=41, init="smooth") if S == 32 else SU.make_case(B, C_, seed=41, init="smooth"))["PG"]
    PD = R.make_params(ref, 42).astype(np.float32)
    real = rng.uniform(0, 1, (d, B // 2, C_, S, S)).astype(np.float32)
    nD = rng.uniform(-1, 1, (d, B // 2, 100)).astype(np.float32)
    nG = rng.uniform(-1, 1, (g, B, 100)).astype(np.float32)
    mD = (rng.uniform(0, 1, (d, B, ref.mask)) >= 0.5).astype(np.float32)
    mG = (rng.uniform(0, 1, (g, B, ref.mask)) >= 0.5).astype(np.float32)
    hp = fg.hyper_default(**NO_PEN)
    ctx, net = make(name, C_, B)
    try:
        net.set_params(0, np.ascontiguousarray(PG, np.float32))
        net.set_params(1, PD)
        ctx.set_option("debug_keep", 1)  # the D iteration's pre-activations ("Dstep.*")
        stats = net.train_step_iters(hp, B, d, g, real, nD, nG, mD, mG, seed=3)
        # the GPU's own pooling decisions where the float64 candidates tie: the G iteration's D forward is the last
        # one ("D.*"); with one D iteration "Dstep.*" holds its pre-activations
        pools = [n for _, mods, _ in ref.branches for n in (m.name for m in mods if isinstance(m, R.MaxPool))]
        zs = {("G", 0): {n: net.debug_tensor("D." + k) for n in pools for k in [n.replace(".", ".z")]}}
        if d == 1:
            zs[("D", 0)] = {n: net.debug_tensor("Dstep." + k) for n in pools for k in [n.replace(".", ".z")]}
        assert stats["trained_D"] == d and stats["t_D"] == d and stats["t_G"] == g
        got = dict(PD=net.get_params(1), PG=net.get_params(0))
        got["mD"], got["vD"], _ = net.get_adam_state(1)
        got["mG"], got["vG"], _ = net.get_adam_state(0)
    finally:
        close(ctx, net)
    routes = {}
    for key, z in zs.items():
        rt, offs = gpu_route(None, PD if key[0] == "D" else got["PD"], zget=lambda k, z=z: z[k.replace(".z", ".")])
        offs.update(pool_slopes(ref))
        routes[key] = rt
    want, conf = _compose_f64(name, C_, B, d, g, PG, PD, real, nD, nG, mD, mG, hp, routes)
    assert list(stats["conf"]) == list(conf)
    for k in ("mD", "vD", "mG", "vG"):
        assert relerr(got[k], want[k]) < 1e-4, (k, relerr(got[k], want[k]))
    for k, steps in (("PD", d), ("PG", g)):
        dd = np.abs(got[k].astype(np.float64) - want[k])
        # a sign flip of a noise-level gradient moves a parameter by up to 2 lr per Adam step
        assert dd.max() < 2.1e-3 * steps and np.mean(dd > 1e-5) < 0.01, (k, dd.max(), np.mean(dd > 1e-5))


# ---- the device-fed step equals the host-fed step on the same draws ------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_disc_device_fed_step_equals_host_fed(name):
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset, noise_uniform
    from face_generator_b200.lib import iteration_root
    C_, B, d, g = 3, 16, 2, 1
    S, Bh, m = R.NETS[name][0], B // 2, 2 ** 64
    imgs = np.random.default_rng(30).integers(0, 256, (100, C_, 32, 32), dtype=np.uint8)
    res = []
    for mode in ("device", "host"):
        ctx, net = make(name, C_, B)
        st = _state(net, 31)
        _reset(net, st)
        ds = DeviceDataset(ctx, imgs)
        h = fg.hyper_default()
        stats = []
        for seed in (6, 7, 8):  # eager, captured, replayed
            if mode == "device":
                s = ds.train_step_iters(h, B, d, g, seed) if net is ctx else net.train_step_dataset_iters(ds, h, B, d, g, seed)
            else:
                r = [iteration_root(seed, j) for j in range(max(d, g))]
                real = np.stack([ds.gather(ds.draw((4 * r[j]) % m, Bh), S) for j in range(d)])
                zD = np.stack([noise_uniform(ctx, (4 * r[j] + 1) % m, (Bh, 100)) for j in range(d)])
                zG = np.stack([noise_uniform(ctx, (4 * r[j] + 2) % m, (B, 100)) for j in range(g)])
                s = net.train_step_iters(h, B, d, g, np.ascontiguousarray(real, np.float32),
                                         np.ascontiguousarray(zD, np.float32), np.ascontiguousarray(zG, np.float32),
                                         seed=seed)
            stats.append(s)
        m1, v1, _ = net.get_adam_state(1)
        res.append((stats, [net.get_params(1), net.get_params(0), m1, v1]))
        ds.close()
        close(ctx, net)
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1], res[1][1]):
        np.testing.assert_array_equal(a, b)


# ---- checkpoints: an adversarial.net with create_D32 loads into a create_D32 context only -------------------------
@pytest.mark.gpu
def test_gpu_disc_reference_checkpoint_loads_into_its_context(tmp_path):
    import face_generator_b200 as fg
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200 import layouts as LY
    from test_t7 import G_CLASSES, cuda_net
    from test_disc_variants_cpu import disc_tree, write_root
    C_ = 3
    rng = np.random.default_rng(12)
    gl, ng = LY.G_layout(C_)
    PG = rng.standard_normal(ng).astype(np.float32)
    PD = rng.standard_normal(R.Net("create_D32", C_).n_params).astype(np.float32)
    p = tmp_path / "adversarial.net"
    write_root(p, {"G": cuda_net(PG, gl, G_CLASSES), "D": disc_tree("create_D32", C_, PD), "epoch": 9})
    ctx = fg.Context(0, max_batch=8, channels=C_, discriminator="create_D32")
    with pytest.warns(UserWarning):  # the tree written here carries no BatchNorm statistics
        assert CK.load_reference_checkpoint(ctx, p) == 9
    np.testing.assert_array_equal(ctx.get_params(1), PD)
    np.testing.assert_array_equal(ctx.get_params(0), PG)
    ctx.close()
    ctx = fg.Context(0, max_batch=8, channels=C_)
    with pytest.raises(fg.FGError, match="checkpoint D is create_D32; this 32x32 net has create_D32b"):
        with pytest.warns(UserWarning):
            CK.load_reference_checkpoint(ctx, p)
    ctx.close()
