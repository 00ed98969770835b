"""Every BatchNorm statistics path against the float64 restatement of tests/bn_ref.py, channel by channel.

BatchNorm's numerics run through three implementations: the per-tile partials of the tensor-core convolution's
epilogue (option bn_epilogue = 1, G.C1 / G.C2 of the 32x32 and --scale 16 generators), the separate double-precision
pass (bn_reduce4_kernel for C % 4 == 0, 16 <= C <= 1024, 256 % (C/4) == 0; bn_stats_kernel otherwise; also behind the
L-op fg_bn_forward_train) and the backward's reduce / apply kernels.  Trained-looking parameters give every channel
|mean| <~ sigma and sigma^2 >> eps, where any of them looks exact, so the data here adds channels whose mean is 100 to
1000 times their spread, near-constant channels (sigma^2 < eps) and an exactly constant channel, and every bar is held
per channel: one bad channel among 256 is not diluted by the rest.

a. the L-ops over C = 1 .. 1024 (both statistics kernels, both apply kernels, one-lane blocks) and batch tails;
b. G's own tensors at batch 256 and 131 (the last epilogue tile partly valid) under every option that changes the
   statistics path, on a "stress set" of parameters."""
import functools

import numpy as np
import pytest

import bn_ref as R
import parity_utils as PU
from oracle import oracle as O
from oracle import oracle_s16 as OS

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = torch.nn.functional
KTOL = 1e-5  # one launch against fp64 on identical inputs (tests/test_gpu_headline.py)
F32_ULP = 2.0 ** -23


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def chan_max(t):
    """per-channel max|t| of an NC... tensor -> [C]"""
    return t.abs().transpose(0, 1).reshape(t.shape[1], -1).max(1).values


def chan_err(a, b):
    """per-channel max|a - b| / max|b| -> [C]"""
    return chan_max(a - b) / chan_max(b).clamp_min(1e-300)


def worst(err, what):
    """assert message: the worst channels of a per-channel error vector"""
    e = err.double().cpu().numpy()
    idx = np.argsort(-e)[:4]
    return "%s: worst channels %s" % (what, ", ".join("%d: %.2e" % (i, e[i]) for i in idx))


def dz_scale(dz, gamma, istd, g):
    """per-channel scale of a BatchNorm input gradient dz = gamma istd (g - mean(g) - xhat mean(g xhat)): max|dz|,
    unless the three terms cancel (max|dz| < 0.1 gamma istd max|g|, e.g. two pixels per channel, where
    1 - xhat^2 = eps / (var + eps)); there max|dz| says nothing about the rounding of the terms, and the bar is taken
    against gamma istd max|g| instead"""
    m = chan_max(dz)
    t = gamma.abs() * istd * chan_max(g)
    return torch.where(m < 0.1 * t, t, m).clamp_min(1e-300)


def check_stats(mean, istd, ref, mean_tol, istd_tol, what):
    """save_mean within 2^-23 |mu| + mean_tol * sqrt(var + eps); save_istd within istd_tol relative"""
    m, s = dev(mean), dev(istd)
    mu, var = ref["mean"], ref["var"]
    em = (m - mu).abs() / (F32_ULP * mu.abs() + mean_tol * torch.sqrt(var + R.EPS))
    assert float(em.max()) <= 1.0, worst(em, what + " mean / bar")
    es = (s - ref["istd"]).abs() / ref["istd"]
    assert float(es.max()) < istd_tol, worst(es, what + " istd")


def check_running(got_m, got_v, rm0, rv0, ref, n, tol, what):
    """running mean relative to the size of its two terms, running variance relative (got_v None: not checked)"""
    rm0, rv0 = dev(rm0), dev(rv0)
    m, v = R.running_update(rm0, rv0, ref["mean"], ref["var"], max(n, 2))
    em = (dev(got_m) - m).abs() / ((1 - R.MOMENTUM) * rm0.abs() + R.MOMENTUM * ref["mean"].abs())
    assert float(em.max()) < tol, worst(em, what + " running mean")
    if got_v is None:
        return
    ev = (dev(got_v) - v).abs() / v
    assert float(ev.max()) < tol, worst(ev, what + " running var")


# ------------------------------------------------------------------------------------------------ a. L-ops
@pytest.fixture(scope="module")
def ctx():
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=8, channels=3)
    yield c
    c.close()


def lop_case(N, C, HW, seed):
    """NCHW data whose channels cycle through: mean ~ sigma; +1e3 sigma; -1e3 sigma; sigma = 1e-3 (sigma^2 < eps).
    The last channel (C >= 3) is exactly constant at 3.3, a value with no short binary expansion."""
    rng = np.random.default_rng(seed)
    sig = rng.uniform(0.5, 2.0, C)
    off = rng.standard_normal(C) * sig
    kind = np.arange(C) % 4
    off[kind == 1] += 1e3 * sig[kind == 1]
    off[kind == 2] -= 1e3 * sig[kind == 2]
    sig[kind == 3] = 1e-3
    x = off[None, :, None] + sig[None, :, None] * rng.standard_normal((N, C, HW))
    if C >= 3:
        x[:, C - 1] = 3.3
    f = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(x=f(x), g=f(rng.uniform(0.5, 1.5, C)), be=f(rng.standard_normal(C) * 0.5), dy=f(rng.standard_normal((N, C, HW))),
                rm=f(rng.standard_normal(C)), rv=f(rng.uniform(0.5, 2.0, C)), dg=f(rng.standard_normal(C)),
                db=f(rng.standard_normal(C)))


def run_lop(ctx, k, N, C, HW, running=True, grads=True, on_device=False):
    """fg_bn_forward_train + fg_bn_backward on case k; host arrays, or device tensors when on_device.
    The running statistics and dgamma / dbeta buffers start from k's non-zero values (None: NULL pointers)."""
    from face_generator_b200.lib import _ptr
    lib, h = ctx.lib, ctx.h
    if on_device:
        t = lambda a: torch.as_tensor(a, device="cuda").contiguous()
        out = lambda shape: torch.empty(shape, dtype=torch.float32, device="cuda")
        p = lambda a: None if a is None else _ptr(a.data_ptr())
        host = lambda a: a.cpu().numpy()
    else:
        t = lambda a: a.copy()
        out = lambda shape: np.empty(shape, np.float32)
        p, host = _ptr, (lambda a: a)
    x, g, be, dy = t(k["x"]), t(k["g"]), t(k["be"]), t(k["dy"])
    rm, rv = (t(k["rm"]), t(k["rv"])) if running else (None, None)
    dg, db = (t(k["dg"]), t(k["db"])) if grads else (None, None)
    y, sm, si, dx = out((N, C, HW)), out(C), out(C), out((N, C, HW))
    if on_device:
        torch.cuda.synchronize()  # the library runs on its own stream
    assert lib.fg_bn_forward_train(h, p(x), p(g), p(be), p(y), p(sm), p(si), p(rm), p(rv), N, C, HW) == 0, lib.fg_last_error()
    assert lib.fg_bn_backward(h, p(x), p(g), p(sm), p(si), p(dy), p(dx), p(dg), p(db), N, C, HW) == 0, lib.fg_last_error()
    r = dict(y=y, mean=sm, istd=si, dx=dx, rm=rm, rv=rv, dg=dg, db=db)
    return {n: (None if a is None else host(a)) for n, a in r.items()}


LOP_C = [1, 3, 12, 16, 24, 64, 128, 256, 512, 768, 1000, 1024]
LOP_NHW = [(1, 1), (2, 1), (3, 49), (5, 7)]


@pytest.mark.parametrize("C,N,HW", [(C, N, HW) for C in LOP_C for N, HW in LOP_NHW] + [(64, 64, 4096)])
def test_lop_batchnorm_per_channel(ctx, C, N, HW):
    """(64, 64, 4096): 262144 rows pass the sm_count * 8 grid cap of bn_reduce4_kernel, with rows left over after its
    4-row unroll"""
    k = lop_case(N, C, HW, seed=C * 1000 + N * 10 + HW)
    got = run_lop(ctx, k, N, C, HW)
    P = N * HW
    for n, v in got.items():
        assert np.isfinite(v).all(), n
    z, g, be, dy = dev(k["x"]), dev(k["g"]), dev(k["be"]), dev(k["dy"])
    ref = R.forward_train(z, g, be)
    check_stats(got["mean"], got["istd"], ref, 1e-6, 1e-6, "L-op C=%d P=%d" % (C, P))
    # y and dx against the reference taken about the kernel's own fp32 mean (its rounding is checked just above)
    gm = dev(got["mean"])
    y_ref = R.forward_train(z, g, be, mean=gm)["u"]
    dz, dgam, dbet, _ = R.backward(z, g, be, gm, ref["istd"], dy)
    if P == 1:  # x_hat = 0: y is beta exactly, and dx is 0
        assert np.array_equal(got["y"], np.broadcast_to(k["be"][None, :, None], got["y"].shape))
        assert not got["dx"].any()
    e = chan_err(dev(got["y"]), y_ref)
    assert float(e.max()) < KTOL, worst(e, "y")
    e = chan_max(dev(got["dx"]) - dz) / dz_scale(dz, g, ref["istd"], dy)
    assert float(e.max()) < KTOL, worst(e, "dx")
    # running statistics from non-zero values; at P = 1 THNN divides by n - 1 = 0, so only the mean is defined
    check_running(got["rm"], got["rv"] if P > 1 else None, k["rm"], k["rv"], ref, P, 1e-6, "L-op")
    # dgamma / dbeta are accumulated into the given buffers
    assert PU.relerr(got["dg"] - k["dg"].astype(np.float64), dgam.cpu().numpy()) < KTOL
    assert PU.relerr(got["db"] - k["db"].astype(np.float64), dbet.cpu().numpy()) < KTOL


@pytest.mark.parametrize("C", [24, 64])
def test_lop_batchnorm_pointers_null_buffers_and_refusal(ctx, C):
    """host and device pointers give the same bits; NULL running statistics and NULL dgamma / dbeta change nothing
    else; dgamma / dbeta are added (+=) to what the buffers held; C = 1025 is refused and the context stays usable"""
    from face_generator_b200.lib import _ptr
    N, HW = 3, 49
    k = lop_case(N, C, HW, seed=77 + C)
    host = run_lop(ctx, k, N, C, HW)
    devp = run_lop(ctx, k, N, C, HW, on_device=True)
    for n in host:
        assert np.array_equal(host[n], devp[n]), n
    bare = run_lop(ctx, k, N, C, HW, running=False, grads=False)
    for n in ("y", "mean", "istd", "dx"):
        assert np.array_equal(bare[n], host[n]), n
    assert bare["rm"] is None and bare["dg"] is None
    # from zeroed buffers the kernels write (float) sum; into k's buffers they add it in fp32
    z = dict(k, dg=np.zeros(C, np.float32), db=np.zeros(C, np.float32))
    fresh = run_lop(ctx, z, N, C, HW)
    assert np.array_equal(host["dg"], k["dg"] + fresh["dg"]) and np.array_equal(host["db"], k["db"] + fresh["db"])
    # refusal
    lib, h = ctx.lib, ctx.h
    Cb = 1025
    x = np.ones((1, Cb, 2), np.float32)
    v = np.ones(Cb, np.float32)
    y, dx = np.empty_like(x), np.empty_like(x)
    assert lib.fg_bn_forward_train(h, _ptr(x), _ptr(v), _ptr(v), _ptr(y), _ptr(v.copy()), _ptr(v.copy()), None, None, 1, Cb, 2) != 0
    assert lib.fg_bn_backward(h, _ptr(x), _ptr(v), _ptr(v), _ptr(v), _ptr(x), _ptr(dx), None, None, 1, Cb, 2) != 0
    again = run_lop(ctx, k, N, C, HW)
    for n in host:
        assert np.array_equal(again[n], host[n]), n


# ------------------------------------------------------------------------------------------------ b. inside G
NETS = {"32": (32, O.G_layout, O.G_param_count), "s16": (16, OS.G_layout, OS.G_param_count)}
OPTIONS = {"default": None, "bn_epilogue=0": ("bn_epilogue", 0), "mma_f16=0": ("mma_f16", 0),
           "conv_impl=1": ("conv_impl", 1), "conv_impl=0": ("conv_impl", 0)}
CH = 3


def open_net(net, B, option=None):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=B + (B & 1), channels=CH)  # max_batch is even; the batch itself need not be
    if option:
        ctx.set_option(*option)
    return ctx, (ctx if net == "32" else fg.S16(ctx))


def close_net(ctx, g):
    if g is not ctx:
        g.close()
    ctx.close()


def nchw(flat, B, H, C):
    """NHWC debug tensor -> float64 NCHW tensor on the GPU"""
    return dev(flat.reshape(B, H, H, C)).permute(0, 3, 1, 2).contiguous()


def split(P, layout):
    return {k: dev(P[o:o + int(np.prod(s))]).reshape(s) for k, (o, s) in layout.items()}


@functools.lru_cache(maxsize=None)
def stress_params(net, B):
    """trained_like_init, then in both BatchNorm layers (mean mu, spread sigma per channel from one default GPU
    forward): 16 channels shifted by +100 sigma, 16 by +1000 sigma and 8 by -1000 sigma through C.b; 8 near-constant
    channels (C.W row x 1e-3, bias 0.7 / 3.3 / 10.1); 1 exactly constant channel (zero C.W row, bias 10.1).
    Such channels: a conv channel whose weights decayed while its bias drifted, or one loaded from a checkpoint."""
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_G
    S, layout, count = NETS[net]
    L = layout(CH)
    rng = np.random.default_rng(5000 + B + S)
    P = LY.trained_like_init((L, count(CH)), rng)
    noise = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
    ctx, g = open_net(net, B)
    g.set_params(NET_G, P)
    g.G_forward(noise)
    z = {1: g.debug_tensor("G.z1").reshape(-1, 256).astype(np.float64), 2: g.debug_tensor("G.z2").reshape(-1, 128).astype(np.float64)}
    close_net(ctx, g)
    for i in (1, 2):
        sd = z[i].std(0)
        (ow, sw), (ob, _) = L["C%dW" % i], L["C%db" % i]
        Cc, fan = sw[0], int(np.prod(sw[1:]))
        W, b = P[ow:ow + Cc * fan].reshape(Cc, fan), P[ob:ob + Cc]
        perm = rng.permutation(Cc)
        for ch, k in zip(perm[:40], [100] * 16 + [1000] * 16 + [-1000] * 8):
            b[ch] += k * sd[ch]
        for j, ch in enumerate(perm[40:48]):
            W[ch] *= 1e-3
            b[ch] = (0.7, 3.3, 10.1)[j % 3]
        W[perm[48]] = 0.0
        b[perm[48]] = 10.1
    return P, noise


def bn_state0(seed):
    """non-trivial running statistics [mean1 256][var1 256][mean2 128][var2 128]"""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.standard_normal(256), rng.uniform(0.5, 2, 256), rng.standard_normal(128),
                           rng.uniform(0.5, 2, 128)]).astype(np.float32)


def gpu_pos(z, mean, istd, gamma, beta):
    """the sign of the pre-activation exactly as the CUDA kernels form it: u = fma(gamma, fl(fl(z - mean) * istd), beta)"""
    f32 = lambda t: t.to(torch.float32)
    cv = lambda v: v.view(1, -1, 1, 1)
    t = f32(f32(f32(z) - f32(cv(mean))) * f32(cv(istd)))
    return (f32(cv(gamma)).double() * t.double() + f32(cv(beta)).double()) > 0


@pytest.mark.parametrize("option", list(OPTIONS))
@pytest.mark.parametrize("B", [256, 131])
@pytest.mark.parametrize("net", list(NETS))
def test_G_batchnorm_per_channel(net, B, option):
    """G's BatchNorm statistics, outputs, running statistics, evaluate mode and backward on its own tensors.  At
    B = 131 the last epilogue tile is partly valid: box (8, 8, 2) of the 32x32 G.C1 and --scale 16 G.C2, box (4, 4, 8)
    of the --scale 16 G.C1."""
    from face_generator_b200.lib import NET_G
    S, layout, _ = NETS[net]
    L = layout(CH)
    P, noise = stress_params(net, B)
    p = split(P, L)
    ctx, g = open_net(net, B, OPTIONS[option])
    try:
        g.set_params(NET_G, P)
        bn0 = bn_state0(B + S)
        g.set_bn_state(bn0)
        g.G_forward(noise)
        T = {"z1": nchw(g.debug_tensor("G.z1"), B, S // 2, 256), "h1": nchw(g.debug_tensor("G.h1"), B, S // 2, 256),
             "z2": nchw(g.debug_tensor("G.z2"), B, S, 128), "h2": nchw(g.debug_tensor("G.h2"), B, S, 128),
             "y": nchw(g.debug_tensor("G.y"), B, S, CH)}
        st = {k: dev(g.debug_tensor("G.bn_" + k)) for k in ("mean1", "istd1", "mean2", "istd2")}
        bn1 = g.get_bn_state()
        layers = ((1, 256, S // 2, "a2", 0), (2, 128, S, "a3", 512))
        ref = {}
        for i, Cc, H, a, o in layers:
            what = "%s B=%d %s BN%d" % (net, B, option, i)
            z, gm, be = T["z%d" % i], p["g%d" % i], p["be%d" % i]
            r = R.forward_train(z, gm, be, p[a], mean=st["mean%d" % i])
            ref[i] = r
            check_stats(st["mean%d" % i].cpu().numpy(), st["istd%d" % i].cpu().numpy(), r, 1e-5, 1e-5, what)
            e = chan_err(T["h%d" % i], r["h"])
            assert float(e.max()) < KTOL, worst(e, what + " h")
            check_running(bn1[o:o + Cc], bn1[o + Cc:o + 2 * Cc], bn0[o:o + Cc], bn0[o + Cc:o + 2 * Cc], r, z.numel() // Cc,
                          1e-5, what)
        # ---- backward: dz of each BatchNorm + PReLU against bn_ref's backward of the GPU's z, with the reference dh
        # built in fp64 from the GPU's dz of the layer above ----
        dout = np.random.default_rng(B + 1).standard_normal((B, CH, S, S)).astype(np.float32)
        g.zero_grads(NET_G)
        g.G_backward(dout)
        grads = g.get_grads(NET_G)
        dz_gpu = {1: nchw(g.debug_tensor("G.dz1"), B, S // 2, 256), 2: nchw(g.debug_tensor("G.dz2"), B, S, 128)}
        up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")
        pool = lambda t: F.avg_pool2d(t, 2, 2) * 4  # backward of the nearest upsample: 2x2 sum
        dz3 = dev(dout) * T["y"] * (1 - T["y"])
        dh = {2: torch.nn.grad.conv2d_input(T["h2"].shape, p["C3W"], dz3, padding=1),
              1: pool(torch.nn.grad.conv2d_input(up(T["h1"]).shape, p["C2W"], dz_gpu[2], padding=2))}
        blk = lambda k: grads[L[k][0]:L[k][0] + int(np.prod(L[k][1]))]
        for i, Cc, H, a, o in layers:
            what = "%s B=%d %s BN%d" % (net, B, option, i)
            z, gm, be, r = T["z%d" % i], p["g%d" % i], p["be%d" % i], ref[i]
            mean = st["mean%d" % i]
            pos = R.kink_pos(r["u"], gpu_pos(z, mean, st["istd%d" % i], gm, be), PU.KINK_MARGIN)
            dz, dgam, dbet, dsl = R.backward(z, gm, be, mean, r["istd"], dh[i], p[a], pos=pos)
            e = chan_max(dz_gpu[i] - dz) / dz_scale(dz, gm, r["istd"], torch.where(pos, dh[i], p[a] * dh[i]))
            assert float(e.max()) < 5 * KTOL, worst(e, what + " dz")
            assert PU.relerr(blk("g%d" % i), dgam.cpu().numpy()) < KTOL, what + " dgamma"
            assert PU.relerr(blk("be%d" % i), dbet.cpu().numpy()) < KTOL, what + " dbeta"
            assert PU.relerr(blk(a), [float(dsl)]) < 3e-4, what + " slope gradient"
        # ---- evaluate mode with the running statistics the training forward left ----
        g.G_forward(noise, training=False)
        for i, Cc, H, a, o in layers:
            rm, rv = dev(bn1[o:o + Cc]), dev(bn1[o + Cc:o + 2 * Cc])
            z, h = nchw(g.debug_tensor("G.z%d" % i), B, H, Cc), nchw(g.debug_tensor("G.h%d" % i), B, H, Cc)
            e = chan_err(h, R.forward_eval(z, p["g%d" % i], p["be%d" % i], rm, rv, p[a]))
            assert float(e.max()) < KTOL, worst(e, "%s B=%d %s BN%d evaluate h" % (net, B, option, i))
    finally:
        close_net(ctx, g)


@pytest.mark.parametrize("B", [256, 131])
@pytest.mark.parametrize("net", list(NETS))
def test_G_epilogue_statistics_agree_with_separate_pass(net, B):
    """the statistics from the convolution epilogue (default) and from the separate double pass (bn_epilogue = 0)
    give the same istd per channel on the stress set"""
    from face_generator_b200.lib import NET_G
    P, noise = stress_params(net, B)
    ctx, g = open_net(net, B)
    try:
        g.set_params(NET_G, P)
        istd = {}
        for v in (1, 0):
            ctx.set_option("bn_epilogue", v)
            g.G_forward(noise)
            istd[v] = [g.debug_tensor("G.bn_istd%d" % i).astype(np.float64) for i in (1, 2)]
        for i in range(2):
            e = np.abs(istd[1][i] - istd[0][i]) / istd[0][i]
            assert e.max() < 1e-5, worst(torch.as_tensor(e), "%s B=%d BN%d istd, epilogue vs separate pass" % (net, B, i + 1))
    finally:
        close_net(ctx, g)
