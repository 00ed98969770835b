"""Option "bwd_streams" (default 1) runs the weight gradients of the 32x32 D (D.L3 to D.C2), G.C3's and G.C1's on a
stream of their own, next to the data-gradient chain of the backward (D32::backward in nets.cu, gen_backward in gen.cu).  Only the
order in which independent launches reach the GPU changes, so a step with it is held bitwise to the same step with
bwd_streams 0 and to the step run with timing on (per-launch timers keep everything on one stream).

Three contexts go through the same calls: (D, G iterations) (1, 1), (2, 1) and (1, 2), host- and device-fed, three calls
each (the two untimed contexts run them eager, captured and replayed).  After every call: parameters, gradients,
optimizer moments and step counters, BatchNorm running state, losses and confusion counts.  The 32x32 and --scale 16
trainers share G's backward; the 32x32 trainer with create_D32 shows that G's half holds with another discriminator.
The direct D and G backward entry points, with their weight gradients, are held to the serial context too.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

pytestmark = pytest.mark.gpu

ITERS = [(1, 1), (2, 1), (1, 2)]


@pytest.fixture(scope="module")
def fg():
    import face_generator_b200 as fg
    return fg


def _state(net):
    from face_generator_b200.lib import NET_D, NET_G
    out = []
    for k in (NET_G, NET_D):
        m, v, t = net.get_adam_state(k)
        out += [net.get_params(k), net.get_grads(k), m, v, np.array([t])]
    return out + [net.get_bn_state()]


def _same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), "%s: array %d differs" % (what, i)


def _contexts(fg, kind, B, C, imgs):
    """(ctx, net, dataset) with bwd_streams 1, with bwd_streams 0 and with timing on; the same parameters"""
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    p0 = np.random.default_rng(51)
    PG = PD = None
    runs = []
    for mode in ("streams", "one stream", "timed"):
        ctx = fg.Context(0, max_batch=B, channels=C, discriminator="create_D32" if kind == "d32" else "create_D32b")
        assert ctx.get_option("bwd_streams") == 1
        if mode == "one stream":
            ctx.set_option("bwd_streams", 0)
            assert ctx.get_option("bwd_streams") == 0
        ctx.timing_enable(mode == "timed")
        net = fg.S16(ctx) if kind == "s16" else ctx
        if PG is None:
            PG = (p0.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32)
            PD = (p0.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32)
        net.set_params(NET_G, PG)
        net.set_params(NET_D, PD)
        runs.append((ctx, net, DeviceDataset(ctx, imgs)))
    return runs


def _close(runs):
    for ctx, net, ds in runs:
        ds.close()
        if net is not ctx:
            net.close()
        ctx.close()


@pytest.mark.parametrize("kind,B", [("32", 256), ("32", 130), ("s16", 256), ("s16", 130), ("d32", 256)])
def test_step_with_wgrad_stream_is_the_serial_step(fg, kind, B):
    C, S = 3, 16 if kind == "s16" else 32
    imgs = np.random.default_rng(50).integers(0, 256, (400, 3, 64, 64), dtype=np.uint8)
    runs = _contexts(fg, kind, B, C, imgs)
    hyper = fg.hyper_default()
    rng = np.random.default_rng(52)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    seed = 200
    try:
        for d, g in ITERS:
            for fed in ("host", "device"):
                for call in range(3):
                    seed += 1
                    inp = [f(rng.random((d, B // 2, C, S, S))), f(rng.uniform(-1, 1, (d, B // 2, 100))),
                           f(rng.uniform(-1, 1, (g, B, 100)))]
                    stats = []
                    for ctx, net, ds in runs:
                        if fed == "host":
                            stats.append(net.train_step_iters(hyper, B, d, g, *inp, None, None, seed))
                        elif kind == "s16":
                            stats.append(net.train_step_dataset_iters(ds, hyper, B, d, g, seed))
                        else:
                            stats.append(ds.train_step_iters(hyper, B, d, g, seed))
                    what = "%s B=%d (%d, %d) %s-fed call %d" % (kind, B, d, g, fed, call)
                    states = [_state(net) for _, net, _ in runs]
                    for i in (1, 2):
                        assert stats[0] == stats[i], "%s: stats vs context %d" % (what, i)
                        _same(states[0], states[i], "%s: vs context %d" % (what, i))
    finally:
        _close(runs)


@pytest.mark.parametrize("kind", ["32", "s16"])
def test_backward_entries_with_wgrad_stream(fg, kind):
    from face_generator_b200.lib import NET_D, NET_G
    B, C = 256, 3
    S = 16 if kind == "s16" else 32
    imgs = np.random.default_rng(60).integers(0, 256, (64, 3, 64, 64), dtype=np.uint8)
    runs = _contexts(fg, kind, B, C, imgs)
    rng = np.random.default_rng(61)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    try:
        for rep in range(2):
            x = f(rng.random((B, C, S, S)))
            dout = f(rng.standard_normal(B))
            noise = f(rng.uniform(-1, 1, (B, 100)))
            dimg = f(rng.standard_normal((B, C, S, S)) * 0.1)
            outs = []
            for _, net, _ in runs:
                net.zero_grads(NET_D)
                net.zero_grads(NET_G)
                net.D_forward(x, seed=7 + rep)
                dx = net.D_backward(dout)
                net.G_forward(noise)
                dn = net.G_backward(dimg, True)
                outs.append([np.asarray(dx), np.asarray(dn), net.get_grads(NET_D), net.get_grads(NET_G)])
            for i in (1, 2):
                _same(outs[0], outs[i], "%s backward entries, round %d, vs context %d" % (kind, rep, i))
    finally:
        _close(runs)


def test_option_range(fg):
    ctx = fg.Context(0, max_batch=8, channels=3)
    try:
        with pytest.raises(fg.FGError):
            ctx.set_option("bwd_streams", 2)
        assert ctx.get_option("bwd_streams") == 1
    finally:
        ctx.close()
