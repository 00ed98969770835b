"""GPU: the optimizer update held to float64 (tests/optim_ref.py), elementwise, at every step.

adam_kernel (k_elem.cu) runs the grad scale, penalty, clamp and the Adam / Adagrad / SGD update of every parameter of
every net, with the step size prepared by gate_prep_kernel, optim_prep_kernel, adam_prep_kernel or fg_adam_step.  The
tests write chosen float32 gradients straight into the library's gradient buffer (fg_*grads_ptr + fg_memcpy), set the
parameters and the optimizer state through the C entry points, run one step and read back the consumed gradient
(the library writes the penalised, clamped gradient back), m, v, t and the parameters.  Each step is checked from
the state the GPU held before it, so errors cannot build up over a run; the references run in float64 on the device.

Bars, in float32 ulps (the spacing of float32 at a magnitude; 2^-149 at and below the subnormals):
  consumed gradient, m   2 ulp of the largest term of the sum (g*scale, the penalty, the result; b1*m, (1-b1)*g):
                         a sum of two terms of opposite sign can cancel to far below its terms, and its float32
                         rounding error is bounded by the terms, not by the result
  v                      3 ulp of v (all terms are >= 0)
  parameters             2 ulp(p) + 1e-5 |dp| + 2^-149/denom (the update dp = step*m/denom, denom = sqrt(v)+eps,
                         carries a few roundings; the product step*m is rounded before the division, and where it
                         is subnormal its absolute error 2^-150 is scaled by 1/denom)
m and v are checked against the float64 update of the consumed gradient the GPU returned, and the parameters
against the float64 update from the m and v the GPU returned, so each bar covers one stage: the moments of a sum
that cancelled would otherwise carry their float32 rounding into the parameters at many ulps of a small p.
Measured on an H100 80GB HBM3 (700 W power limit): the consumed gradient and m within 1.0 ulp, v within 1.5 ulp,
parameters within 0.36 of their bar (fg_dn_train_step's two chained updates: m within 2.6 ulp).  The worst error of each quantity is printed (run with -s)."""
import ctypes as C

import numpy as np
import pytest

import optim_ref as R

pytestmark = pytest.mark.gpu

G_BAR, M_BAR, V_BAR, P_ULP, P_REL = 2.0, 2.0, 3.0, 2.0, 1e-5
SPECIAL = 97  # every 97th element from offset k holds special value k (_grads)


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.init()
    return torch


def _vp(t):
    return C.c_void_p(t.data_ptr())


def _ctx_of(pair):
    return pair if hasattr(pair, "max_batch") else pair.ctx


class Vec:
    """the flat parameter vector of one net of a pair (Context, C2f, S16) with its gradient and optimizer state,
    read and written as float32 CUDA tensors through the pair's C entry points"""

    def __init__(self, torch, pair, net):
        self.torch, self.pair, self.net, self.n = torch, pair, net, pair.count(net)
        self.ctx = _ctx_of(pair)
        self.gptr = getattr(pair.lib, pair._prefix + "grads_ptr")(pair.h, net)
        assert self.gptr

    def _sync(self):
        from face_generator_b200.lib import _check
        _check(self.pair.lib.fg_sync(self.ctx.h), "fg_sync")

    def put(self, P=None, m=None, v=None, t=None, g=None):
        from face_generator_b200.lib import _check
        self.torch.cuda.synchronize()  # the library's stream does not wait for torch's
        if P is not None:
            self.pair._call("set_params", self.net, _vp(P))
        if t is not None:
            self.pair._call("set_adam_state", self.net, None if m is None else _vp(m), None if v is None else _vp(v), int(t))
        if g is not None:
            _check(self.pair.lib.fg_memcpy(self.ctx.h, C.c_void_p(self.gptr), _vp(g), 4 * self.n), "fg_memcpy")

    def state(self):
        torch = self.torch
        P, g, m, v = (torch.empty(self.n, dtype=torch.float32, device="cuda") for _ in range(4))
        t = C.c_int(0)
        self.pair._call("get_params", self.net, _vp(P))
        self.pair._call("get_grads", self.net, _vp(g))
        self.pair._call("get_adam_state", self.net, _vp(m), _vp(v), C.byref(t))
        self._sync()
        return dict(P=P, g=g, m=m, v=v, t=t.value)


def _grads(torch, n, gen, lo=1e-30, hi=1e3, specials=(0.0, -0.0, 1e-40, -3e-42, 1.4e-45, -1.4e-45)):
    """fresh float32 gradients: magnitudes log-uniform over [lo, hi] with random signs, and every SPECIAL-th
    element from offset k set to specials[k] (zeros, -0.0, subnormals)"""
    e = torch.rand(n, generator=gen, dtype=torch.float64, device="cuda") * (np.log10(hi) - np.log10(lo)) + np.log10(lo)
    s = torch.where(torch.rand(n, generator=gen, device="cuda") < 0.5, -1.0, 1.0).double()
    g = (s * torch.pow(10.0, e)).float()
    for k, val in enumerate(specials):
        g[k::SPECIAL] = val
    return g


def _params(torch, n, gen, scale=0.05):
    """float32 parameters ~ N(0, scale^2), some exactly 0 and -0.0 (sign(0) = 0 in the L1 penalty)"""
    P = (torch.randn(n, generator=gen, device="cuda", dtype=torch.float64) * scale).float()
    P[10::SPECIAL] = 0.0
    P[11::SPECIAL] = -0.0
    return P


def _ulp(torch, x):
    """spacing of float32 at |x| (x float64); 2^-149 for |x| below the normal range"""
    _, e = torch.frexp(x.abs())
    u = torch.pow(torch.full_like(x, 2.0), (e - 24).clamp_min(-149).to(x.dtype))
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -149), u)


def _worst(torch, what, got, ref, unit, bar, report, mask=None):
    """max |got - ref| / unit; fails when an element exceeds bar (NaN counts as exceeding)"""
    r = (got.double() - ref).abs() / unit
    if mask is not None:
        r = r[mask]
    bad = ~(r <= bar)
    if bad.any():
        i = int(torch.nonzero(bad)[0])
        idx = torch.nonzero(mask)[i] if mask is not None else i
        idx = int(idx)
        pytest.fail("%s: %d elements beyond %.3g (first at %d: got %r, float64 %r, %.3g units)" %
                    (what, int(bad.sum()), bar, idx, float(got.double()[idx]), float(ref[idx]), float(r[i])))
    w = float(r.max()) if r.numel() else 0.0
    report[what] = max(report.get(what, 0.0), w)
    return w


class Rule:
    """the update rule, its hyper-parameters and the net's penalty / clamp, as the library is configured"""

    def __init__(self, name, hy, is_D, mom=0.0):
        self.name, self.hy, self.is_D, self.mom = name, hy, is_D, mom
        self.lr = hy.lr_D if is_D else hy.lr_G
        self.l1, self.l2 = R.penalty_terms(is_D, hy.D_L1, hy.D_L2) if is_D else R.penalty_terms(False, hy.G_L1, hy.G_L2)
        self.clamp = hy.D_clamp if is_D else hy.G_clamp

    def consumed(self, g, p, scale):
        return R.consumed_grad(g, p, scale, self.l1, self.l2, self.clamp)

    def param(self, p, g, m, v, t):
        """(parameters, denominator or None) of step t from the updated m, v (or gradient g), all float64"""
        hy = self.hy
        if self.name == "adam":
            return R.adam_param(p, m, v, t, self.lr, hy.beta1, hy.beta2, hy.eps), R._sqrt(v) + R.f32(hy.eps)
        if self.name == "adagrad":
            return R.adagrad_param(p, g, v, self.lr), R._sqrt(v) + R.f32(1e-10)
        return p - R.f32(self.lr) * (m if self.mom else g), None

    def update(self, p, g, m, v, t):
        """(p, m, v, t) after one step from (p, m, v, t) with consumed gradient g, all float64"""
        hy = self.hy
        if self.name == "adam":
            return R.adam(p, g, m, v, t, self.lr, hy.beta1, hy.beta2, hy.eps)
        if self.name == "adagrad":
            p, v, t = R.adagrad(p, g, v, t, self.lr)
            return p, m, v, t
        p, m, t = R.sgd(p, g, m, t, self.lr, self.mom)
        return p, m, v, t


def check_step(torch, rule, pre, g_in, post, scale, report, mask=None):
    """post (the GPU state after one step) against the float64 step from pre (the GPU state before it) with raw
    gradient g_in; mask selects the elements compared"""
    f = lambda a: a.double()
    p0, m0, v0 = f(pre["P"]), f(pre["m"]), f(pre["v"])
    g_ref = rule.consumed(f(g_in), p0, scale)
    pen = (R._sign(p0) * R.f32(rule.l1) + p0 * R.f32(rule.l2)).abs()
    mag = torch.maximum(torch.maximum((f(g_in) * R.f32(scale)).abs(), pen), g_ref.abs())
    if rule.clamp:  # a clamped element is +-clamp exactly
        c = R.f32(rule.clamp)
        mag = torch.where(rule.consumed(f(g_in), p0, scale).abs() >= c, torch.full_like(mag, c), mag)
    _worst(torch, "grad", post["g"], g_ref, _ulp(torch, mag), G_BAR, report, mask)
    g = f(post["g"])
    p, m, v, t = rule.update(p0, g, m0, v0, pre["t"])
    assert post["t"] == t, (post["t"], t)
    if rule.name == "adam" or (rule.name == "sgd" and rule.mom != 0):
        b = R.f32(rule.hy.beta1 if rule.name == "adam" else rule.mom)
        mag = torch.maximum(torch.maximum((m0 * b).abs(), ((1 - b) * g).abs()), m.abs())
        if rule.name == "sgd" and pre["t"] == 0:
            mag = m.abs()
        _worst(torch, "m", post["m"], m, _ulp(torch, mag), M_BAR, report, mask)
    else:
        assert torch.equal(post["m"], pre["m"]), "m changed under " + rule.name
    if rule.name in ("adam", "adagrad"):
        _worst(torch, "v", post["v"], v, _ulp(torch, v), V_BAR, report, mask)
    else:
        assert torch.equal(post["v"], pre["v"]), "v changed under sgd"
    _check_param(torch, rule, p0, g, post, t, report, mask)


def _check_param(torch, rule, p0, g, post, t, report, mask=None):
    """the parameters after step t against the float64 update from p0 and the g, m, v the GPU returned"""
    p, denom = rule.param(p0, g, post["m"].double(), post["v"].double(), t)
    unit = P_ULP * _ulp(torch, p) + P_REL * (p - p0).abs()
    if denom is not None:
        unit = unit + 2.0 ** -149 / denom
    _worst(torch, "param", post["P"], p, unit, 1.0, report, mask)


def optim_run(torch, ctx, net, rule, steps, gen, scale=1.0, grads=None):
    """`steps` fg_optim_step calls on the ctx's own vectors, each with fresh gradients and checked"""
    x = Vec(torch, ctx, net)
    report = {}
    pre = x.state()
    for _ in range(steps):
        g = grads(x.n) if grads else _grads(torch, x.n, gen)
        x.put(g=g)
        ctx.optim_step(net, rule.hy, scale)
        post = x.state()
        check_step(torch, rule, pre, g, post, scale, report)
        pre = post
    return report


def _hyper(**kw):
    import face_generator_b200 as fg
    # every penalty weight nonzero and G_L1 != G_L2, so that G's quirk (its L1 term weighted by G_L2) shows
    base = dict(D_L1=2e-4, D_L2=1e-4, G_L1=3e-4, G_L2=1e-4)
    base.update(kw)
    return fg.hyper_default(**base)


# ---- 200 consecutive steps of each rule, on D and G, 1 and 3 channels -------------------------------------------------
@pytest.mark.parametrize("C_", [1, 3])
@pytest.mark.parametrize("method,mom", [("adam", 0.0), ("adagrad", 0.0), ("sgd", 0.9)])
def test_optim_step_200_steps(torch, method, mom, C_):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(100 + C_)
    ctx = fg.Context(0, max_batch=4, channels=C_)
    lr = {"adam": 1e-3, "adagrad": 1e-3, "sgd": 0.02}[method]
    hy = _hyper(lr_D=lr, lr_G=lr)
    try:
        for net in (NET_D, NET_G):
            ctx.set_optimizer(net, method, mom)
            x = Vec(torch, ctx, net)
            x.put(P=_params(torch, x.n, gen))
            rep = optim_run(torch, ctx, net, Rule(method, hy, net == NET_D, mom), 200, gen)
            print("200 steps %s C=%d %s (n=%d): worst %s" % (method, C_, "DG"[net], x.n, rep))
    finally:
        ctx.close()


# ---- resumed states --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t0", [1, 2, 10 ** 4, 10 ** 6])
def test_adam_resumed(torch, t0):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(t0)
    ctx = fg.Context(0, max_batch=4, channels=3)
    hy = _hyper()
    try:
        for net in (NET_D, NET_G):
            x = Vec(torch, ctx, net)
            m0 = (torch.randn(x.n, generator=gen, device="cuda") * 1e-2).float()
            v0 = (torch.rand(x.n, generator=gen, device="cuda") * 1e-4).float()
            m0[12::SPECIAL], v0[12::SPECIAL] = 0.0, 0.0
            x.put(P=_params(torch, x.n, gen), m=m0, v=v0, t=t0)
            rep = optim_run(torch, ctx, net, Rule("adam", hy, net == NET_D), 3, gen)
            print("adam resumed at t=%d %s: worst %s" % (t0, "DG"[net], rep))
    finally:
        ctx.close()


def test_adagrad_resumed_large_variance(torch):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(7)
    ctx = fg.Context(0, max_batch=4, channels=3)
    hy = _hyper(D_clamp=0.0, G_clamp=0.0)
    try:
        for net in (NET_D, NET_G):
            ctx.set_optimizer(net, "adagrad")
            x = Vec(torch, ctx, net)
            v0 = torch.pow(10.0, torch.rand(x.n, generator=gen, device="cuda", dtype=torch.float64) * 36).float()  # 1 .. 1e36
            x.put(P=_params(torch, x.n, gen), m=torch.zeros(x.n, device="cuda"), v=v0, t=12345)
            rep = optim_run(torch, ctx, net, Rule("adagrad", hy, net == NET_D), 3, gen,
                            grads=lambda n: _grads(torch, n, gen, hi=1e18))
            print("adagrad resumed, large variance %s: worst %s" % ("DG"[net], rep))
    finally:
        ctx.close()


@pytest.mark.parametrize("mom", [0.5, 0.9])
@pytest.mark.parametrize("t0", [0, 5])
def test_sgd_resumed(torch, mom, t0):
    """evalCounter 0: the momentum buffer the state holds is ignored and replaced by the gradient (the reference has
    no state.dfdx before its first evaluation); evalCounter 5: it is blended"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(int(mom * 10) + t0)
    ctx = fg.Context(0, max_batch=4, channels=3)
    hy = _hyper(lr_D=0.02, lr_G=0.02)
    try:
        for net in (NET_D, NET_G):
            ctx.set_optimizer(net, "sgd", mom)
            x = Vec(torch, ctx, net)
            m0 = (torch.randn(x.n, generator=gen, device="cuda") * 0.3).float()
            x.put(P=_params(torch, x.n, gen), m=m0, v=torch.zeros(x.n, device="cuda"), t=t0)
            rep = optim_run(torch, ctx, net, Rule("sgd", hy, net == NET_D, mom), 3, gen)
            print("sgd mom %.1f resumed at t=%d %s: worst %s" % (mom, t0, "DG"[net], rep))
    finally:
        ctx.close()


# ---- penalty, clamp and grad scale ----------------------------------------------------------------------------------
def _edge_grads(torch, n, gen, clamp, scale):
    """gradients spread over 1e-30 .. 1e3 plus, every SPECIAL-th element, exactly +-clamp, one ulp beyond and inside
    it, +-clamp/scale (on the clamp after scaling), and +-Inf when a clamp is on"""
    c = np.float32(clamp if clamp else 1.0)
    vals = [c, -c, np.nextafter(c, np.float32(np.inf)), -np.nextafter(c, np.float32(np.inf)), np.nextafter(c, np.float32(0)),
            np.float32(c / np.float32(scale)), -np.float32(c / np.float32(scale)), 0.0, -0.0, 1e-40]
    if clamp:
        vals += [np.inf, -np.inf]
    return _grads(torch, n, gen, specials=tuple(float(v) for v in vals))


@pytest.mark.parametrize("scale", [1.0, 0.5, 1.0 / 3.0])
@pytest.mark.parametrize("clamp", [1.0, 5.0, 0.0])
def test_penalty_clamp_scale(torch, clamp, scale):
    """grad_scale applies first, then the penalty (P exactly 0 / -0.0 in places), then the clamp"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(int(clamp * 10 + scale * 100))
    ctx = fg.Context(0, max_batch=4, channels=3)
    hy = _hyper(D_clamp=clamp, G_clamp=clamp, D_L1=1e-2, D_L2=3e-2, G_L1=5e-3, G_L2=2e-2)
    try:
        for net in (NET_D, NET_G):
            x = Vec(torch, ctx, net)
            x.put(P=_params(torch, x.n, gen, scale=1.0))
            rep = optim_run(torch, ctx, net, Rule("adam", hy, net == NET_D), 2, gen, scale,
                            grads=lambda n: _edge_grads(torch, n, gen, clamp, scale))
            if clamp:
                g = x.state()["g"]
                assert float(g.abs().max()) == np.float32(clamp)
            print("penalty/clamp %.3g scale %.4g %s: worst %s" % (clamp, scale, "DG"[net], rep))
    finally:
        ctx.close()


def test_nan_gradient_under_clamp_becomes_minus_clamp(torch):
    """pins fminf(fmaxf(NaN, -c), c) = -c (fg_b200.h, fg_optim_step); Torch's CPU clamp would keep the NaN.  Without a
    clamp the NaN is consumed as it is."""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(5)
    ctx = fg.Context(0, max_batch=4, channels=1)
    try:
        for clamp in (1.0, 0.0):
            hy = _hyper(D_clamp=clamp, G_clamp=clamp)
            for net in (NET_D, NET_G):
                x = Vec(torch, ctx, net)
                x.put(P=_params(torch, x.n, gen))
                g = _grads(torch, x.n, gen, hi=1.0)
                g[::1000] = float("nan")
                x.put(g=g)
                ctx.optim_step(net, hy)
                got = x.state()["g"][::1000]
                if clamp:
                    assert bool((got == -np.float32(clamp)).all()), got[:8]
                else:
                    assert bool(torch.isnan(got).all())
    finally:
        ctx.close()


def test_fp32_overflow_of_v(torch):
    """clamp off and huge gradients.  v += (1-beta2)*g*g is evaluated left to right, ((1-beta2)*g)*g, as Torch's
    addcmul does on FloatTensors (interruptable_optimizers.lua:82), so |g| = 1e20 gives a finite v = 1e37 (checked
    in float64 with the rest) while |g| = 1e21 overflows: there v = inf and the update m/(sqrt(v)+eps) is 0"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    gen = torch.Generator(device="cuda").manual_seed(11)
    ctx = fg.Context(0, max_batch=4, channels=3)
    hy = _hyper(D_clamp=0.0, G_clamp=0.0)
    try:
        for net in (NET_D, NET_G):
            x = Vec(torch, ctx, net)
            x.put(P=_params(torch, x.n, gen), m=(torch.randn(x.n, generator=gen, device="cuda") * 1e-3).float(),
                  v=torch.rand(x.n, generator=gen, device="cuda").float() * 1e-4, t=3)
            pre = x.state()
            g = _grads(torch, x.n, gen)
            g[50::2 * SPECIAL] = 1e20
            g[50 + SPECIAL::2 * SPECIAL] = -1e20
            over = torch.zeros(x.n, dtype=torch.bool, device="cuda")
            over[51::SPECIAL] = True
            g[51::2 * SPECIAL] = 1e21
            g[51 + SPECIAL::2 * SPECIAL] = -1e21
            x.put(g=g)
            ctx.optim_step(net, hy)
            post = x.state()
            assert bool(torch.isinf(post["v"][over]).all())
            assert torch.equal(post["P"][over], pre["P"][over])
            assert bool(torch.isfinite(post["m"][over]).all())
            assert float(post["v"][50::SPECIAL].min()) > 9e36 and bool(torch.isfinite(post["v"][50::SPECIAL]).all())
            check_step(torch, Rule("adam", hy, net == NET_D), pre, g, post, 1.0, {}, mask=~over)
    finally:
        ctx.close()


# ---- fg_adam_step: the raw-pointer entry, at the block and grid-cap edges ------------------------------------------
@pytest.mark.parametrize("where", ["device", "pinned"])
def test_adam_step_sizes(torch, where):
    """n around one block (256 threads) and the grid cap (132*8 blocks of 256 = 270 336 threads), and 5 000 003
    (the grid-stride loop wraps 18 times); one element past n must stay untouched.  "pinned": the four vectors live
    in page-locked host memory, which the kernel reads through the unified address space."""
    import face_generator_b200 as fg
    from face_generator_b200.lib import PinnedArray, _check
    gen = torch.Generator(device="cuda").manual_seed(3)
    ctx = fg.Context(0, max_batch=4, channels=1)
    lr, b1, b2, eps, l1, l2, clamp = 1e-3, 0.9, 0.999, 1e-8, 1e-4, 2e-4, 1.0
    hy = fg.hyper_default(lr_D=lr, D_L1=l1, D_L2=l2, D_clamp=clamp)
    rule = Rule("adam", hy, True)
    report = {}
    try:
        for n in (1, 255, 256, 257, 270335, 270336, 270337, 5000003):
            for t in (1, 2, 10 ** 4):
                vecs = [_params(torch, n + 1, gen), _grads(torch, n + 1, gen),
                        (torch.randn(n + 1, generator=gen, device="cuda") * 1e-2).float(),
                        (torch.rand(n + 1, generator=gen, device="cuda") * 1e-4).float()]
                pre = dict(P=vecs[0].clone(), m=vecs[2].clone(), v=vecs[3].clone(), t=t - 1)
                g_in = vecs[1].clone()
                if where == "pinned":
                    pins = [PinnedArray((n + 1,)) for _ in range(4)]
                    for a, b in zip(pins, vecs):
                        a.array[:] = b.cpu().numpy()
                    ptrs = [C.c_void_p(a.addr) for a in pins]
                else:
                    ptrs = [_vp(a) for a in vecs]
                torch.cuda.synchronize()
                _check(ctx.lib.fg_adam_step(ctx.h, ptrs[0], ptrs[1], ptrs[2], ptrs[3], n, lr, b1, b2, eps, t, l1, l2, clamp,
                                            1.0), "fg_adam_step")
                ctx.sync()
                if where == "pinned":
                    out = [torch.from_numpy(a.array.copy()).cuda() for a in pins]
                    for a in pins:
                        a.free()
                else:
                    out = vecs
                post = dict(P=out[0][:n], g=out[1][:n], m=out[2][:n], v=out[3][:n], t=t)
                for k, a in zip(("P", "g", "m", "v"), out):
                    ref = (pre[k] if k != "g" else g_in)[n]
                    assert torch.equal(a[n], ref), "fg_adam_step wrote %s[%d] past n" % (k, n)
                check_step(torch, rule, {k: (v[:n] if k != "t" else v) for k, v in pre.items()}, g_in[:n], post, 1.0, report)
        print("fg_adam_step %s: worst %s" % (where, report))
    finally:
        ctx.close()


# ---- each trainer's wiring: one step from a resumed state --------------------------------------------------------
T_RESUME = 5000


def _resume(torch, x, gen):
    m0 = (torch.randn(x.n, generator=gen, device="cuda") * 1e-3).float()
    v0 = (torch.rand(x.n, generator=gen, device="cuda") * 1e-5).float()
    x.put(m=m0, v=v0, t=T_RESUME)
    return x.state()


def _check_trainer_update(torch, x, pre, rule, what):
    """the step's update of x from its resumed state with the gradient the step consumed, which must respect the
    clamp; the carried t must be used"""
    post = x.state()
    assert post["t"] == T_RESUME + 1, (what, post["t"])
    if rule.clamp:
        assert float(post["g"].abs().max()) <= np.float32(rule.clamp), what
    g = post["g"]
    p, m, v, t = rule.update(pre["P"].double(), g.double(), pre["m"].double(), pre["v"].double(), pre["t"])
    report = {}
    b = R.f32(rule.hy.beta1)
    _worst(torch, "m", post["m"], m, _ulp(torch, torch.maximum(torch.maximum((pre["m"].double() * b).abs(),
                                                                             ((1 - b) * g.double()).abs()), m.abs())),
           M_BAR, report)
    _worst(torch, "v", post["v"], v, _ulp(torch, v), V_BAR, report)
    _check_param(torch, rule, pre["P"].double(), g.double(), post, t, report)
    print("%s: worst %s" % (what, report))


def test_train_step_wiring_32(torch):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    import parity_utils as PU
    B, C_ = 8, 3
    case = PU.make_case(B, C_, seed=41)
    gen = torch.Generator(device="cuda").manual_seed(41)
    ctx = fg.Context(0, max_batch=B, channels=C_)
    hy = fg.hyper_default(**PU.HYPER)
    try:
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        xs = {net: Vec(torch, ctx, net) for net in (NET_D, NET_G)}
        pre = {net: _resume(torch, x, gen) for net, x in xs.items()}
        st = ctx.train_step(hy, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        assert st["trained_D"] == 1 and st["t_D"] == st["t_G"] == T_RESUME + 1
        for net, x in xs.items():
            _check_trainer_update(torch, x, pre[net], Rule("adam", hy, net == NET_D), "fg_train_step " + "GD"[net])
    finally:
        ctx.close()


def test_train_step_wiring_s16(torch):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    import s16_utils as SU
    B, C_ = 8, 3
    case = SU.make_case(B, C_, seed=42)
    gen = torch.Generator(device="cuda").manual_seed(42)
    ctx = fg.Context(0, max_batch=B, channels=C_)
    net16 = fg.S16(ctx)
    hy = fg.hyper_default(**SU.HYPER)
    try:
        net16.set_params(NET_G, case["PG"])
        net16.set_params(NET_D, case["PD"])
        xs = {net: Vec(torch, net16, net) for net in (NET_D, NET_G)}
        pre = {net: _resume(torch, x, gen) for net, x in xs.items()}
        st = net16.train_step(hy, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        assert st["trained_D"] == 1 and st["t_D"] == st["t_G"] == T_RESUME + 1
        for net, x in xs.items():
            _check_trainer_update(torch, x, pre[net], Rule("adam", hy, net == NET_D), "fg_s16_train_step " + "GD"[net])
    finally:
        net16.close()
        ctx.close()


def test_train_step_wiring_c2f(torch):
    """train_c2f.lua's defaults (D_L1 = 1e-7) and optim.adam without the accuracy gate: D_maxAcc = 0 would close the
    gate of the 32x32 loop, and D still steps"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    import c2f_utils as CU
    B, C_ = 4, 3
    case = CU.make_case(B, C_, seed=43)
    gen = torch.Generator(device="cuda").manual_seed(43)
    ctx = fg.Context(0, max_batch=B, channels=C_)
    c2f = fg.C2f(ctx)
    hy = fg.hyper_default(**CU.HYPER, D_maxAcc=0.0)
    try:
        c2f.set_params(NET_G, case["PG"])
        c2f.set_params(NET_D, case["PD"])
        xs = {net: Vec(torch, c2f, net) for net in (NET_D, NET_G)}
        pre = {net: _resume(torch, x, gen) for net, x in xs.items()}
        st = c2f.train_step(hy, B, case["real_diff"], case["cond_D"], case["noise_D"], case["cond_G"], case["noise_G"],
                            case["masks_D"], case["masks_G"])
        assert st["t_D"] == st["t_G"] == T_RESUME + 1
        for net, x in xs.items():
            _check_trainer_update(torch, x, pre[net], Rule("adam", hy, net == NET_D), "fg_c2f_train_step " + "GD"[net])
    finally:
        c2f.close()
        ctx.close()


def _shared_state_check(torch, what, hy_rule, P0, m0, v0, t0, grads, P1, m1, v1, t1):
    """optim.adam steps on parameter vectors P0[i] in turn, each with its consumed gradient grads[i], sharing one
    (m, v, t): the state after the last step and each vector's parameters"""
    m, v, t = m0.double(), v0.double(), t0
    report = {}
    for i, (p0, g) in enumerate(zip(P0, grads)):
        b = R.f32(hy_rule.hy.beta1)
        mprev = m
        p, m, v, t = R.adam(p0.double(), g.double(), m, v, t, hy_rule.lr, hy_rule.hy.beta1, hy_rule.hy.beta2, hy_rule.hy.eps)
        _worst(torch, "param", P1[i], p, P_ULP * _ulp(torch, p) + P_REL * (p - p0.double()).abs(), 1.0, report)
        if i == len(P0) - 1:
            mag = torch.maximum(torch.maximum((mprev * b).abs(), ((1 - b) * g.double()).abs()), m.abs())
            # two chained updates: the first one's float32 rounding of m and v carries into the second
            _worst(torch, "m", m1, m, _ulp(torch, mag), 2 * M_BAR, report)
            _worst(torch, "v", v1, v, _ulp(torch, v), 2 * V_BAR, report)
        else:
            m, v = m.float().double(), v.float().double()  # the state between the two steps is float32 on the GPU
    assert t1 == t0 + len(P0), (what, t1)
    print("%s: worst %s" % (what, report))


class _Cfg:
    def __init__(self, h):
        self.hy = h
        self.lr = h.lr


def test_train_step_wiring_denoiser(torch):
    """train_denoiser.lua: AE1's and AE2's optim.adam steps share one state (m, v, t), AE1 first; the clamp holds on
    both consumed gradients.  The m / v between the two steps is not visible, so AE1's parameters are checked against
    the float64 first step and the final m / v against both steps with the intermediate state rounded to float32."""
    import face_generator_b200 as fg
    from face_generator_b200.denoiser import Denoiser, dn_hyper_default
    ctx = fg.Context(0, max_batch=8, channels=3)
    dn = Denoiser(ctx, size=16)
    rng = np.random.default_rng(44)
    gen = torch.Generator(device="cuda").manual_seed(44)
    hy = dn_hyper_default()
    try:
        n = dn.n
        m0 = (torch.randn(n, generator=gen, device="cuda") * 1e-3).float()
        v0 = (torch.rand(n, generator=gen, device="cuda") * 1e-5).float()
        dn.set_adam_state(m0.cpu().numpy(), v0.cpu().numpy(), T_RESUME)
        P0 = [torch.from_numpy(dn.get_params(k)).cuda() for k in (0, 1)]
        st = dn.train_step(hy, rng.random((8, 3, 16, 16)).astype(np.float32), seed=5)
        grads = [torch.from_numpy(dn.get_grads(k)).cuda() for k in (0, 1)]
        for g in grads:
            assert float(g.abs().max()) <= np.float32(hy.clamp)
        m1, v1, t1 = dn.get_adam_state()
        P1 = [torch.from_numpy(dn.get_params(k)).cuda() for k in (0, 1)]
        assert st["t"] == t1
        _shared_state_check(torch, "fg_dn_train_step", _Cfg(hy), P0, m0, v0, T_RESUME, grads, P1,
                            torch.from_numpy(m1).cuda(), torch.from_numpy(v1).cuda(), t1)
    finally:
        dn.close()
        ctx.close()


def test_train_step_wiring_autoencoder(torch):
    import face_generator_b200 as fg
    from face_generator_b200.autoencoder import Autoencoder, ae_hyper_default
    ctx = fg.Context(0, max_batch=8, channels=1)
    ae = Autoencoder(ctx, size=32)
    rng = np.random.default_rng(45)
    gen = torch.Generator(device="cuda").manual_seed(45)
    hy = ae_hyper_default()
    try:
        n = ae.n
        m0 = (torch.randn(n, generator=gen, device="cuda") * 1e-3).float()
        v0 = (torch.rand(n, generator=gen, device="cuda") * 1e-5).float()
        ae.set_adam_state(m0.cpu().numpy(), v0.cpu().numpy(), T_RESUME)
        P0 = torch.from_numpy(ae.get_params()).cuda()
        st = ae.train_step(hy, rng.random((8, 1, 32, 32)).astype(np.float32), seed=5)
        g = torch.from_numpy(ae.get_grads()).cuda()
        m1, v1, t1 = ae.get_adam_state()
        assert st["t"] == t1
        _shared_state_check(torch, "fg_ae_train_step", _Cfg(hy), [P0], m0, v0, T_RESUME, [g],
                            [torch.from_numpy(ae.get_params()).cuda()], torch.from_numpy(m1).cuda(),
                            torch.from_numpy(v1).cuda(), t1)
    finally:
        ae.close()
        ctx.close()


# ---- fg_optim_step next to the fused steps: no gate, no accuracy history ------------------------------------------
def test_optim_step_after_train_step_is_not_gated(torch):
    """fg_optim_step(D) right after a fused step, without zeroing the gradients: the step's confusion counts are still
    in the buffer, and they are not an accuracy.  D moves by the float64 Adam step at t = 2 and t_D is 2."""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    import parity_utils as PU
    B, C_ = 64, 3
    case = PU.make_case(B, C_, seed=46)
    ctx = fg.Context(0, max_batch=B, channels=C_)
    hy = fg.hyper_default()
    try:
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        st = ctx.train_step(hy, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        assert st["trained_D"] == 1 and st["conf"][0] + st["conf"][3] > 0
        x = Vec(torch, ctx, NET_D)
        pre = x.state()
        assert pre["t"] == 1
        ctx.optim_step(NET_D, hy)
        post = x.state()
        assert post["t"] == 2, "fg_optim_step(D) did not step (t_D = %d)" % post["t"]
        rep = {}
        check_step(torch, Rule("adam", hy, True), pre, pre["g"], post, 1.0, rep)
        print("optim_step after train_step: worst %s" % rep)
    finally:
        ctx.close()


def _gate_sequence(B, case, max_acc2):
    """train_step (accs_interval 2), zero_grads + optim_step on D, train_step with D_maxAcc = max_acc2"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    ctx = fg.Context(0, max_batch=B, channels=3)
    try:
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        hy = fg.hyper_default(accs_interval=2)
        s1 = ctx.train_step(hy, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        ctx.zero_grads(NET_D)
        ctx.optim_step(NET_D, hy)
        hy2 = fg.hyper_default(accs_interval=2, D_maxAcc=max_acc2)
        s2 = ctx.train_step(hy2, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        return s1, s2
    finally:
        ctx.close()


def test_optim_step_keeps_accuracy_history(torch):
    """D's accuracy gate of a fused step averages the accuracies of the fused steps only (adversarial.lua:156-178): a
    module-level optimizer step in between adds nothing to the history.  D_maxAcc of the second step lies strictly
    between the mean with and the mean without a spurious 0, so the gate decision tells them apart."""
    import parity_utils as PU
    B = 64
    case = PU.make_case(B, 3, seed=47)
    s1, s2 = _gate_sequence(B, case, 1.01)  # the accuracies; the gate does not change the D forward of either step
    a1, a2 = s1["acc_D"], s2["acc_D"]
    assert a1 > 0
    with_zero, fused_only = (a2 + 0.0) / 2, (a1 + a2) / 2
    max_acc = (with_zero + fused_only) / 2
    accs, go1 = R.accuracy_gate([], a1, 2, 1.01)
    _, go2 = R.accuracy_gate(accs, a2, 2, max_acc)
    assert go1 and not go2
    t1, t2 = _gate_sequence(B, case, max_acc)
    assert (t1["acc_D"], t2["acc_D"]) == (a1, a2)
    assert t2["trained_D"] == int(go2), (a1, a2, max_acc, t2)
    assert t2["t_D"] == 2 + int(go2)
