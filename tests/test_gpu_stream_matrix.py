"""The two-stream train step against the one-stream step, bit for bit, on every numeric path and discriminator.

The 32x32 and --scale 16 train steps overlap work on two more streams: the first G iteration's generator forward runs
on side_stream beside the last D iteration (step_body, netpair.cu), and with option bwd_streams the weight gradients of
the 32x32 D and of G.C3 / G.C1 run on wgrad_stream (OnWgradStream, convl.cu).  Which buffers each launch reads and
writes differs between the numeric paths (3xFP16 or 3xTF32 operands, producers that write the operand split themselves,
the FFMA kernels and their split-K workspaces, the separate BatchNorm statistics pass, the round-1 edge kernels, the
merged G backward), so each path and each discriminator is held to the serial step here.

Per case three contexts start from the same parameters with the same options:
  A  both streams (the defaults),
  B  bwd_streams 0: only the side-stream G forward is left,
  C  timing on: one stream throughout.
A != B points at the weight-gradient stream, B != C at the side-stream generator forward.  A race in the side-stream
forward runs in A and B alike, so in one run it may also show as A != B; the message names what differs either way.

All three are made with max_batch 256 and run the same calls: batches 256, 130, 4 (the smallest the step accepts) and
256 again, (D, G iterations) (1, 1), (2, 1) and (1, 2), host- and device-fed, three calls each.  A and B run the three
calls eager, captured and replayed (unless the case sets use_graph 0), which the test checks through the context's
count of graph launches.  Each batch round adds six step keys (three iteration pairs, two feeds) and the step-graph
cache keeps the newest eight (net_graph_run, netpair.cu), so the first round's graphs are gone when the last
batch-256 round starts, and that round captures them again.  After every call: parameters, gradients, optimizer state
and step counters, BatchNorm running state, losses, confusion counts and gate decisions.  After every three calls: an
eval-mode G forward.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MAX_BATCH = 256
BATCHES = [256, 130, 4, 256]
ITERS = [(1, 1), (2, 1), (1, 2)]
MODES = ("A (both streams)", "B (bwd_streams 0)", "C (serial)")
BLAME = ("they differ in the weight-gradient stream", "they differ in the side-stream G forward")
# per-iteration accuracy gate (adversarial.lua:154-178 with accs_interval 1): D trains while its accuracy on the
# iteration's batch is below 0.6.  From random parameters it starts near 0.5 and soon tells the uniform-noise reals
# from the generator's images, so some D updates are skipped while the side-stream G forward still runs beside them.
GATE = dict(D_maxAcc=0.6, accs_interval=1)

CASES = [("32", "create_D32b", o) for o in (
    {}, {"mma_f16": 0}, {"conv_impl": 0}, {"conv_impl": 1}, {"bn_epilogue": 0}, {"edge_impl": 0}, {"bwd_merge": 0},
    {"bwd_merge": 2}, {"use_graph": 0}, {"optimizer": ("adagrad", 0.0)}, {"optimizer": ("sgd", 0.9)}, {"hyper": GATE})]
CASES += [("32", "create_D32", o) for o in ({}, {"mma_f16": 0}, {"conv_impl": 0})]
CASES += [("s16", "create_D16_d", o) for o in (
    {}, {"mma_f16": 0}, {"conv_impl": 0}, {"conv_impl": 1}, {"bn_epilogue": 0}, {"bwd_merge": 2})]
CASES += [("s16", d, o) for d in ("create_D16", "create_D16_b", "create_D16_c")
          for o in ({}, {"mma_f16": 0}, {"conv_impl": 0})]


def _case_id(case):
    kind, disc, opts = case
    words = []
    for k, v in opts.items():
        if k == "optimizer":
            words.append(v[0])
        elif k == "hyper":
            words.append("gate")
        else:
            words.append("%s=%s" % (k, v))
    return "-".join([disc] + (words or ["default"]))


OPTIMIZERS = ["adam", "adagrad", "sgd"]  # option optimizer_D / optimizer_G
STATE = ["G.params", "G.grads", "G.m", "G.v", "G.t", "D.params", "D.grads", "D.m", "D.v", "D.t", "G.bn_running"]


@pytest.fixture(scope="module")
def fg():
    import face_generator_b200 as fg
    return fg


def _state(ctx, net):
    """STATE as CUDA tensors, copied on the device (host copies of every array after every call would take most of
    the test's time)"""
    from face_generator_b200.lib import NET_D, NET_G, _ptr
    dev = lambda n: torch.empty(n, dtype=torch.float32, device="cuda")
    out = []
    for k in (NET_G, NET_D):
        P, g, m, v = (dev(net.count(k)) for _ in range(4))
        t = ctypes.c_int(0)
        net._call("get_params", k, _ptr(P.data_ptr()))
        net._call("get_grads", k, _ptr(g.data_ptr()))
        net._call("get_adam_state", k, _ptr(m.data_ptr()), _ptr(v.data_ptr()), ctypes.byref(t))
        out += [P, g, m, v, torch.tensor([t.value])]
    bn = dev(768)
    net._call("get_bn_state", _ptr(bn.data_ptr()))
    ctx.sync()  # copies to device memory are asynchronous on the context's stream
    return out + [bn]


def _bits(x):
    """x as a tensor whose equality is bitwise equality"""
    x = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
    return x.view({4: torch.int32, 8: torch.int64}[x.element_size()]) if x.is_floating_point() else x


def _first_difference(a, b, names):
    """None, or where a and b (lists of arrays or tensors) first differ"""
    for name, x, y in zip(names, a, b):
        bx, by = _bits(x), _bits(y)
        if bx.shape != by.shape:
            return "%s: shapes %s vs %s" % (name, tuple(bx.shape), tuple(by.shape))
        if not torch.equal(bx, by):
            bad = (bx != by).flatten().nonzero().flatten()
            i = int(bad[0])
            fx, fy = (torch.as_tensor(np.asarray(z)) if not torch.is_tensor(z) else z for z in (x, y))
            return "%s differs at %d of %d elements, first [%d]: %r vs %r" % (
                name, bad.numel(), bx.numel(), i, fx.flatten()[i].item(), fy.flatten()[i].item())
    return None


def _agree(per_mode, names, what):
    """per_mode: one list of arrays per context (A, B, C); every context must hold the same bits"""
    msgs = []
    for i, blame in enumerate(BLAME):
        d = _first_difference(per_mode[i], per_mode[i + 1], names)
        if d:
            msgs.append("%s vs %s (%s): %s" % (MODES[i], MODES[i + 1], blame, d))
    assert not msgs, "%s: %s" % (what, "; ".join(msgs))


def _contexts(fg, kind, disc, opts, imgs):
    """(ctx, net, dataset) for A, B and C; the same parameters and options"""
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    p0 = np.random.default_rng(71)
    PG = PD = None
    runs = []  # [ctx, net, dataset]
    try:
        for mode in MODES:
            ctx = fg.Context(0, max_batch=MAX_BATCH, channels=3, discriminator=disc if kind == "32" else "create_D32b")
            runs.append([ctx, ctx, None])
            for k, v in opts.items():
                if k == "optimizer":
                    for which in (NET_G, NET_D):
                        ctx.set_optimizer(which, *v)
                    assert ctx.get_option("optimizer_D") == ctx.get_option("optimizer_G") == OPTIMIZERS.index(v[0])
                elif k != "hyper":
                    ctx.set_option(k, v)
                    assert ctx.get_option(k) == v
            if mode != MODES[0]:
                ctx.set_option("bwd_streams", 0)
            assert ctx.get_option("bwd_streams") == (mode == MODES[0])
            ctx.timing_enable(mode == MODES[2])
            if kind == "s16":
                runs[-1][1] = fg.S16(ctx, discriminator=disc)
            net = runs[-1][1]
            if PG is None:
                PG = (p0.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32)
                PD = (p0.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32)
            net.set_params(NET_G, PG)
            net.set_params(NET_D, PD)
            runs[-1][2] = DeviceDataset(ctx, imgs)
    except BaseException:
        _close(runs)
        raise
    return runs


def _close(runs):
    for ctx, net, ds in runs:
        if ds is not None:
            ds.close()
        if net is not ctx:
            net.close()
        ctx.close()


@pytest.mark.parametrize("kind,disc,opts", CASES, ids=[_case_id(c) for c in CASES])
def test_concurrent_step_is_the_serial_step(fg, kind, disc, opts):
    C, S = 3, 32 if kind == "32" else 16
    imgs = np.random.default_rng(70).integers(0, 256, (400, 3, 64, 64), dtype=np.uint8)
    hyper = fg.hyper_default(**opts.get("hyper", {}))
    rng = np.random.default_rng(72)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    seed = 300
    gate = []  # (D iterations, trained_D) of every call
    runs = _contexts(fg, kind, disc, opts, imgs)
    try:
        for rnd, B in enumerate(BATCHES):
            for d, g in ITERS:
                for fed in ("host", "device"):
                    what = "%s, batch %d (round %d), (%d, %d) %s-fed" % (_case_id((kind, disc, opts)), B, rnd, d, g, fed)
                    graphs = [ctx.get_option("step_graph_launches") for ctx, _, _ in runs]
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
                        at = "%s call %d" % (what, call)
                        keys = sorted(stats[0])
                        _agree([[np.array(s[k]) for k in keys] for s in stats], ["stats." + k for k in keys], at)
                        _agree([_state(ctx, net) for ctx, net, _ in runs], STATE, at)
                        assert stats[0]["t_G"] > 0 and np.isfinite(stats[0]["loss_D"]), (at, stats[0])
                        gate.append((d, stats[0]["trained_D"]))
                    # a key new to the cache: eager, then captured and launched, then replayed
                    graphs = [ctx.get_option("step_graph_launches") - n for (ctx, _, _), n in zip(runs, graphs)]
                    assert graphs == ([0, 0, 0] if opts.get("use_graph") == 0 else [2, 2, 0]), (what, graphs)
                    noise = f(rng.uniform(-1, 1, (B, 100)))
                    _agree([[net.G_forward(noise, training=False)] for _, net, _ in runs], ["eval G forward"],
                           "after " + what)
    finally:
        _close(runs)
    if "hyper" in opts:
        assert any(t < d for d, t in gate) and any(t > 0 for d, t in gate), \
            "D_maxAcc %.2f never closed or never opened the gate: %s" % (GATE["D_maxAcc"], gate)
