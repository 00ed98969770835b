"""The 32x32 and --scale 16 train steps with one GPU run the first G iteration's generator forward on a second stream,
next to the D iterations (step_body, netpair.cu).  Only the order in which independent launches reach the GPU changes,
so the overlapped step is held bitwise to the serial one: the step run with timing on (per-launch timers keep it on one
stream).

Both contexts go through the same calls: (D, G iterations) (1, 1), (2, 1), (1, 2) and (2, 2), host- and device-fed,
three calls each (the overlapped context runs them eager, captured and replayed).  After every call: parameters,
gradients, optimizer moments and step counters, BatchNorm running state, losses and confusion counts.  After each
group of calls: the "G.*" debug rows (they describe the G iteration's forward, B samples), an eval-mode G forward and,
for the 32x32 nets, fg_sample.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

pytestmark = pytest.mark.gpu

ITERS = [(1, 1), (2, 1), (1, 2), (2, 2)]
G_ROWS = ["G." + n for n in ("z0", "h0", "z1", "h1", "z2", "h2", "z3", "y", "dz2", "dz1", "dz0", "bn_mean1", "bn_istd1",
                              "bn_mean2", "bn_istd2")]


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


@pytest.mark.parametrize("kind", ["32", "s16"])
@pytest.mark.parametrize("B", [256, 130])
def test_overlapped_step_is_the_serial_step(fg, kind, B):
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    C, S = 3, 32 if kind == "32" else 16
    imgs = np.random.default_rng(50).integers(0, 256, (400, 3, 64, 64), dtype=np.uint8)
    p0 = np.random.default_rng(51)
    PG = None
    runs = []  # (ctx, net, dataset): overlapped, serial
    for serial in (False, True):
        ctx = fg.Context(0, max_batch=B, channels=C)
        ctx.timing_enable(serial)
        net = ctx if kind == "32" else fg.S16(ctx)
        if PG is None:
            PG = (p0.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32)
            PD = (p0.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32)
        net.set_params(NET_G, PG)
        net.set_params(NET_D, PD)
        runs.append((ctx, net, DeviceDataset(ctx, imgs)))
    hyper = fg.hyper_default()
    rng = np.random.default_rng(52)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    seed = 100
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
                        elif kind == "32":
                            stats.append(ds.train_step_iters(hyper, B, d, g, seed))
                        else:
                            stats.append(net.train_step_dataset_iters(ds, hyper, B, d, g, seed))
                    what = "%s B=%d (%d, %d) %s-fed call %d" % (kind, B, d, g, fed, call)
                    assert stats[0] == stats[1], what
                    _same(_state(runs[0][1]), _state(runs[1][1]), what)
                rows = [[net.debug_tensor(n) for n in G_ROWS] for _, net, _ in runs]
                _same(rows[0], rows[1], "G.* rows after " + what)
                assert rows[0][G_ROWS.index("G.y")].size == B * S * S * C  # the G iteration's B samples
                noise = f(rng.uniform(-1, 1, (B, 100)))
                out = [net.G_forward(noise, False) for _, net, _ in runs]
                _same(out[:1], out[1:], "eval G forward after " + what)
                if kind == "32":
                    out = [ctx.sample(noise, 64) for ctx, _, _ in runs]
                    _same(out[:1], out[1:], "fg_sample after " + what)
    finally:
        for ctx, net, ds in runs:
            ds.close()
            if net is not ctx:
                net.close()
            ctx.close()
