"""GPU: the coarse-to-fine nets with models_c2f.lua's other generators and discriminators (fg_c2f_create_nets).

Each new G runs with create_D_c and each new D with create_G_d, at fine sizes 16, 32 and 64, batch 256 and the ragged
130, mma_f16 1 and 0, colour (and grayscale at one size), against tests/c2f_var_ref.py in float64:
 * every forward launch in isolation at 1e-5 (the layer's output against F.conv2d / F.linear of the CUDA path's own
   input), the whole net forward and backward at 1e-4 (PReLU slopes 3e-4), with the kink and max-pool routing rules of
   tests/test_gpu_c2f_s16_headline.py;
 * the kernel each new layer shape takes (fg_conv2d_* and last_conv_kind; D's Linear from the net itself);
 * one train_step_iters (1+1, 2+1) at batch 8 and 256 against a float64 loop body composed from the restatement
   and tests/optim_ref.py;
 * device-fed == host-fed on the same draws, graph replay == eager, same seed == same bits, fg_c2f_refine against the
   restatement, fg_c2f_parzen_dist, and fg_c2f_create_nets with the defaults == fg_c2f_create_sized.
"""
import ctypes

import numpy as np
import pytest

import c2f_var_ref as V
import optim_ref as O
from test_gpu_c2f_s16_headline import (KTOL, TOL, check_losses_and_update, first_max, pool_route, prelu32, within,
                                       windows)
from test_gpu_headline import dev, kink_branch, nchw, rel

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = torch.nn.functional

NEW_G = ["create_G_a", "create_G_b", "create_G_c"]
NEW_D = ["create_D_a", "create_D_b"]
SIZES = [16, 32, 64]
BF = [(256, 1), (256, 0), (130, 1), (130, 0)]
FG_KERNEL_TAPCONV, FG_KERNEL_WGRAD_TC = 1, 2


def _ctx(B, f16, C=3):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_option("conv_impl", 2)
    ctx.set_option("mma_f16", f16)
    return ctx


def _net(ctx, S, gen="create_G_d", disc="create_D_c"):
    import face_generator_b200 as fg
    return fg.C2f(ctx, S, gen, disc)


def check_tensors(got, ref, layout, errs, prefix):
    """per parameter tensor at TOL, a shared PReLU slope (one heavily cancelling sum) at 3 TOL"""
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        e = float(np.abs(got[o:o + n] - ref[o:o + n]).max() / (np.abs(ref[o:o + n]).max() + 1e-300))
        within(errs, prefix + k, e, 3 * TOL if k[0] == "a" else TOL)


def G_cases():
    out = [(g, S, B, f16, 3) for g in NEW_G for S in SIZES for B, f16 in BF]
    return out + [(g, 32, 130, 1, 1) for g in NEW_G]


def D_cases():
    out = [(d, S, B, f16, 3) for d in NEW_D for S in SIZES for B, f16 in BF]
    return out + [(d, 32, 130, 1, 1) for d in NEW_D]


@pytest.mark.parametrize("gen,S,B,f16,C", G_cases(), ids=lambda v: str(v))
def test_G_launches_and_whole_net(gen, S, B, f16, C):
    from face_generator_b200.lib import NET_G
    case = V.make_case(B, C, S, gen, "create_D_c", seed=S + B + f16 + 10 * C)
    noise, cond = case["noise_G"], case["cond_G"]
    dout = np.random.default_rng(B).standard_normal((B, C, S, S)).astype(np.float32)
    ctx = _ctx(B, f16, C)
    net = _net(ctx, S, gen)
    assert net.nG == V.count(V.G_layout(gen, C))
    net.set_params(NET_G, case["PG"])
    out = net.G_forward(noise, cond)
    # the ->C output layer is G's last convolution-type launch: its forward on the wgmma kernels means the layer kept
    # ConvL::pad_out (set once at alloc, it also routes the weight gradient through the swapped-role wgmma launch)
    out_kind, out_tile_n = ctx.get_option("last_conv_kind"), ctx.get_option("last_conv_tile_n")
    convs = V.G_convs(gen, C)
    T = {"x": net.debug_tensor("G.x")}
    T.update({"z%d" % (i + 1): net.debug_tensor("G.z%d" % (i + 1)) for i in range(len(convs))})
    net.zero_grads(NET_G)
    net.G_backward(dout)
    grad = net.get_grads(NET_G)
    net.close()
    ctx.close()
    assert (out_kind, out_tile_n) == (FG_KERNEL_TAPCONV, 64), (out_kind, out_tile_n)
    # every launch on its own input
    import torch_ref as R
    p = R._split(dev(case["PG"]), V.G_layout(gen, C))
    x = nchw(T["x"], B, S, S, C + 1)
    assert torch.equal(x, torch.cat([dev(noise), dev(cond)], 1))  # JoinTable
    errs = {}
    zs = []
    for i, (cin, cout, k) in enumerate(convs):
        z = nchw(T["z%d" % (i + 1)], B, S, S, cout)
        within(errs, "G.c%d" % (i + 1), rel(z, F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=k // 2)), KTOL)
        zs.append(z)
        if i < len(convs) - 1:
            x = prelu32(z, p["a%d" % (i + 1)])
    assert np.array_equal(nchw(T["z%d" % len(convs)], B, S, S, C).cpu().numpy(), out)
    # the whole net
    counts = {}
    g_pos = {"z%d" % (i + 1): zs[i] > 0 for i in range(len(convs) - 1)}
    P = dev(case["PG"]).requires_grad_(True)
    ref = V.G_forward(P, dev(noise), dev(cond), gen, C, branch=kink_branch(g_pos, counts))
    within(errs, "out", rel(out, ref.detach()), TOL)
    ref.backward(dev(dout))
    check_tensors(grad, P.grad.cpu().numpy(), V.G_layout(gen, C), errs, "G.")
    print(gen, S, B, f16, C, errs, counts)


def _D_route(get, P, disc, C, S, B):
    """the CUDA path's branch decisions and max-pool picks from its D pre-activations"""
    import torch_ref as R
    p = R._split(dev(P), V.D_layout(disc, C, S))
    pos, idx = {}, {}
    for i, (cin, cout, H, pool) in enumerate(V.D_convs(disc, C, S)):
        z = nchw(get("z%d" % (i + 1)), B, H, H, cout)
        pos["z%d" % (i + 1)] = z > 0
        if pool:
            idx["p%d" % (i + 1)] = first_max(windows(prelu32(z, p["a%d" % (i + 1)])))
    pos["zl1"] = dev(get("zl1").reshape(B, 512)) > 0
    return pos, idx


@pytest.mark.parametrize("disc,S,B,f16,C", D_cases(), ids=lambda v: str(v))
def test_D_launches_and_whole_net(disc, S, B, f16, C):
    from face_generator_b200.lib import NET_D
    case = V.make_case(B, C, S, "create_G_d", disc, seed=100 + S + B + f16 + 10 * C)
    diff, cond, masks = np.concatenate([case["real_diff"], case["real_diff"]]), case["cond_D"], case["masks_D"]
    dout = np.random.default_rng(B + 7).standard_normal(B).astype(np.float32)
    ctx = _ctx(B, f16, C)
    net = _net(ctx, S, disc=disc)
    assert net.nD == V.count(V.D_layout(disc, C, S)) and net.mask_per_sample == V.mask_per_sample(disc, S)
    net.set_params(NET_D, case["PD"])
    out = net.D_forward(diff, cond, masks=masks)
    convs = V.D_convs(disc, C, S)
    names = ["x", "zl1", "logit"] + ["z%d" % (i + 1) for i in range(len(convs))]
    names += ["p%d" % (i + 1) for i, c in enumerate(convs) if c[3]]
    T = {n: net.debug_tensor("D." + n) for n in names}
    net.zero_grads(NET_D)
    ddiff = net.D_backward(dout)
    grad = net.get_grads(NET_D)
    net.D_forward(diff, cond, training=False)
    linear_kind = ctx.get_option("last_conv_kind")  # D.L1 is the last convolution-type launch of D's forward
    net.close()
    ctx.close()
    assert linear_kind == FG_KERNEL_TAPCONV, linear_kind
    import torch_ref as R
    p = R._split(dev(case["PD"]), V.D_layout(disc, C, S))
    m = dev(masks)
    x = nchw(T["x"], B, S, S, C)
    assert torch.equal(x, dev(diff + cond))  # CAddTable (both exact in float32 here: the sum is formed in float32)
    errs = {}
    for i, (cin, cout, H, pool) in enumerate(convs):
        z = nchw(T["z%d" % (i + 1)], B, H, H, cout)
        within(errs, "D.c%d" % (i + 1), rel(z, F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=1)), KTOL)
        x = prelu32(z, p["a%d" % (i + 1)])
        if pool:
            pooled = nchw(T["p%d" % (i + 1)], B, H // 2, H // 2, cout)
            assert torch.equal(pooled, F.max_pool2d(x, 2, 2))
            x = pooled
    n = x[0].numel()
    zl1 = dev(T["zl1"].reshape(B, 512))
    within(errs, "D.L1", rel(zl1, F.linear(x.reshape(B, n) * m[:, :n] * 2.0, p["L1W"], p["L1b"])), KTOL)
    a = p["a%d" % (len(convs) + 1)]
    ref = F.linear(prelu32(zl1, a) * m[:, n:] * 2.0, p["L2W"], p["L2b"]).reshape(B)
    within(errs, "D.L2", rel(dev(T["logit"]), ref), KTOL)
    # the whole net
    pos, idx = _D_route(lambda k: T[k], case["PD"], disc, C, S, B)
    counts = {}
    P = dev(case["PD"]).requires_grad_(True)
    xd = dev(diff).requires_grad_(True)
    ref = V.D_forward(P, xd, dev(cond), m, disc, C, S, branch=kink_branch(pos, counts), route=pool_route(idx, counts))
    within(errs, "out", rel(out, ref.detach()), TOL)
    ref.backward(dev(dout))
    within(errs, "d(diff)", rel(ddiff, xd.grad), TOL)
    check_tensors(grad, P.grad.cpu().numpy(), V.D_layout(disc, C, S), errs, "D.")
    print(disc, S, B, f16, C, errs, counts)


# ---- the kernel of each new layer shape (fg_conv2d_*: the ConvL dispatch rules, DESIGN.md §7.2) ---------------------
NEW_SHAPES = [(64, 128, 7, 1), (64, 256, 5, 1), (64, 128, 3, 1), (128, 128, 3, 2)]  # (Cin, Cout, k, side divisor)


@pytest.mark.parametrize("f16", [1, 0])
@pytest.mark.parametrize("S", SIZES)
@pytest.mark.parametrize("cin,cout,k,div", NEW_SHAPES, ids=lambda v: str(v))
def test_new_layer_shapes_run_on_the_tensor_cores(cin, cout, k, div, S, f16):
    ctx = _ctx(8, f16)
    N, H = 8, S // div
    g = torch.Generator(device="cuda").manual_seed(S + k)
    x = torch.randn(N, cin, H, H, device="cuda", generator=g)
    w = torch.randn(cout, cin, k, k, device="cuda", generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, device="cuda", generator=g) * 0.1
    dy = torch.randn(N, cout, H, H, device="cuda", generator=g)
    y, dx = torch.empty(N, cout, H, H, device="cuda"), torch.empty(N, cin, H, H, device="cuda")
    dw, db = torch.zeros(cout, cin, k, k, device="cuda"), torch.zeros(cout, device="cuda")
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    kinds = {}
    for fn, args in (("fg_conv2d_forward", (P(x), P(w), P(b), P(y))), ("fg_conv2d_backward_data", (P(dy), P(w), P(dx))),
                     ("fg_conv2d_backward_filter", (P(x), P(dy), P(dw), P(db)))):
        torch.cuda.synchronize()
        assert getattr(ctx.lib, fn)(ctx.h, *args, N, cin, H, H, cout, k) == 0, ctx.lib.fg_last_error()
        ctx.sync()
        kinds[fn] = ctx.get_option("last_conv_kind")
    ctx.close()
    assert kinds == {"fg_conv2d_forward": FG_KERNEL_TAPCONV, "fg_conv2d_backward_data": FG_KERNEL_TAPCONV,
                     "fg_conv2d_backward_filter": FG_KERNEL_WGRAD_TC}, kinds
    xd, wd, dyd = x.double().requires_grad_(True), w.double().requires_grad_(True), dy.double()
    ref = F.conv2d(xd, wd, b.double(), padding=k // 2)
    ref.backward(dyd)
    assert rel(y.double(), ref.detach()) < KTOL
    assert rel(dx.double(), xd.grad) < KTOL
    assert rel(dw.double(), wd.grad) < KTOL


# ---- one loop body against float64 ------------------------------------------------------------------------------
PAIRS = [(g, "create_D_c") for g in NEW_G] + [("create_G_d", d) for d in NEW_D]


def _step_inputs(B, C, S, gen, disc, d_iters, seed):
    """train_step_iters inputs stacked per iteration: D iteration j from make_case(seed + j), the G iteration from
    make_case(seed)"""
    cases = [V.make_case(B, C, S, gen, disc, seed + j) for j in range(d_iters)]
    out = {k: np.stack([c[k] for c in cases]) for k in ("real_diff", "cond_D", "noise_D", "masks_D")}
    out.update({k: cases[0][k][None] for k in ("cond_G", "noise_G", "masks_G")})
    # D's logits and G's diffs of the order of the real pairs': no sample saturates the sigmoid, where the float32
    # output (and so the criterion's gradient) of the CUDA path and the float64 checker part ways
    PG, PD = cases[0]["PG"].copy(), cases[0]["PD"].copy()
    gl, dl = V.G_layout(gen, C), V.D_layout(disc, C, S)
    o, sh = gl["c%dW" % len(V.G_convs(gen, C))]
    PG[o:o + int(np.prod(sh))] *= 0.1
    for k, f in (("L2W", 0.05), ("L2b", 0.0)):
        o, sh = dl[k]
        PD[o:o + int(np.prod(sh))] *= f
    out.update(PG=PG, PD=PD)
    return out


def _train(gen, disc, S, B, d_iters, x, keep):
    import face_generator_b200 as fg
    import c2f_utils as CU
    from face_generator_b200.lib import NET_D, NET_G
    ctx = _ctx(B, 1)
    ctx.set_option("debug_keep", int(keep))
    net = _net(ctx, S, gen, disc)
    net.set_params(NET_G, x["PG"])
    net.set_params(NET_D, x["PD"])
    j = slice(0, d_iters)
    st = net.train_step_iters(fg.hyper_default(**CU.HYPER), B, d_iters, 1, x["real_diff"][j], x["cond_D"][j],
                              x["noise_D"][j], x["cond_G"], x["noise_G"], x["masks_D"][j], x["masks_G"])
    r = dict(st=st, PD=net.get_params(NET_D))
    for k, w in ((NET_D, "D"), (NET_G, "G")):
        r["m" + w], r["v" + w], r["t" + w] = net.get_adam_state(k)
    if keep:
        nd, ng = len(V.D_convs(disc, 3, S)), len(V.G_convs(gen, 3))
        zn = ["z%d" % (i + 1) for i in range(nd)] + ["zl1", "out"]
        r["Dk"] = {n: net.debug_tensor("Dstep." + n) for n in zn}
        r["Dg"] = {n: net.debug_tensor("D." + n) for n in zn}
        r["Gg"] = {"z%d" % (i + 1): net.debug_tensor("G.z%d" % (i + 1)) for i in range(ng - 1)}
    net.close()
    ctx.close()
    return r


@pytest.mark.parametrize("B,d_iters", [(8, 1), (8, 2), (256, 1), (256, 2)])
@pytest.mark.parametrize("gen,disc", PAIRS)
def test_train_step_iters_against_float64(gen, disc, B, d_iters):
    """one fg_c2f_train_step_iters (d_iters D iterations + 1 G iteration of adversarial_c2f.lua:121-187, optim.adam,
    train_c2f.lua's D_L1 = 1e-7) against its float64 composition.  The last D iteration runs on the parameters the
    CUDA path held before it (for 2+1: those after a 1+1 call on the first iteration's inputs) with its kink and pool
    decisions from the "Dstep.*" tensors (option debug_keep); D's Adam moment must be that iteration's consumed
    gradient folded into the moment before it.  The G iteration runs on the CUDA path's post-Adam D parameters.  G's
    gradient passes D's data gradient and then G's backward, two nets' rounding: its tensors are held to 3e-4."""
    import c2f_utils as CU
    import torch_ref as R
    C, S, Bh, hp = 3, 32, B // 2, CU.HYPER
    x = _step_inputs(B, C, S, gen, disc, d_iters, seed=4300 + B)
    got = _train(gen, disc, S, B, d_iters, x, keep=True)
    assert got["tD"] == d_iters and got["tG"] == 1
    b1 = O.f32(hp["beta1"])
    if d_iters == 1:
        PD0, m0 = x["PD"], np.zeros_like(got["mD"])
    else:
        first = _train(gen, disc, S, B, 1, x, keep=False)
        PD0, m0 = first["PD"], first["mD"]
    j = d_iters - 1
    PG = dev(x["PG"]).requires_grad_(True)
    PD = dev(PD0).requires_grad_(True)
    with torch.no_grad():
        fake = V.G_forward(PG, dev(x["noise_D"][j]), dev(x["cond_D"][j][Bh:]), gen, C)
    counts = {}
    pos, idx = _D_route(lambda n: got["Dk"][n], PD0, disc, C, S, B)
    out = V.D_forward(PD, torch.cat([dev(x["real_diff"][j]), fake]), dev(x["cond_D"][j]), dev(x["masks_D"][j]), disc, C,
                      S, branch=kink_branch(pos, counts), route=pool_route(idx, counts))
    out.backward(R.bce_grad(out.detach(), torch.cat([torch.ones(Bh), torch.zeros(Bh)]).double().cuda()))
    P0 = PD0.astype(np.float64)
    gD = O.consumed_grad(PD.grad.cpu().numpy(), P0, l1=hp["D_L1"], l2=hp["D_L2"], clamp=hp["D_clamp"])
    errs = {}
    check_tensors((got["mD"] - b1 * m0) / (1 - b1), gD, V.D_layout(disc, C, S), errs, "gradD.")
    g_pos = {n: nchw(got["Gg"][n], B, S, S, V.G_convs(gen, C)[int(n[1:]) - 1][1]) > 0 for n in got["Gg"]}
    pos, idx = _D_route(lambda n: got["Dg"][n], got["PD"], disc, C, S, B)
    gcounts, dcounts = {}, {}
    diff = V.G_forward(PG, dev(x["noise_G"][0]), dev(x["cond_G"][0]), gen, C, branch=kink_branch(g_pos, gcounts))
    outG = V.D_forward(dev(got["PD"]), diff, dev(x["cond_G"][0]), dev(x["masks_G"][0]), disc, C, S,
                       branch=kink_branch(pos, dcounts), route=pool_route(idx, dcounts))
    outG.backward(R.bce_grad(outG.detach(), torch.ones(B).double().cuda()))
    gG = O.consumed_grad(PG.grad.cpu().numpy(), x["PG"].astype(np.float64), clamp=hp["G_clamp"])
    mG = got["mG"] / (1 - b1)
    for k, (o, s) in V.G_layout(gen, C).items():
        n = int(np.prod(s))
        within(errs, "gradG." + k, float(np.abs(mG[o:o + n] - gG[o:o + n]).max() / np.abs(gG[o:o + n]).max()), 3 * TOL)
    if d_iters == 1:
        check_losses_and_update(errs, got["st"], got["Dk"]["out"], out.detach(), hp["D_L1"] * float(np.abs(P0).sum()),
                                got["Dg"]["out"], outG.detach(), Bh, gD, x["PD"], got["PD"], hp)
    print(gen, disc, B, d_iters, errs, counts, gcounts, dcounts)


# ---- device-fed, graphs, seeds ------------------------------------------------------------------------------------
def _dataset(ctx, n=64, side=64, seed=3):
    from face_generator_b200.dataset import DeviceDataset
    imgs = np.random.default_rng(seed).integers(0, 256, (n, 3, side, side), dtype=np.uint8)
    return DeviceDataset(ctx, imgs)


def _state(net):
    from face_generator_b200.lib import NET_D, NET_G
    out = []
    for k in (NET_G, NET_D):
        m, v, t = net.get_adam_state(k)
        out += [net.get_params(k), m, v, np.array([t])]
    return out


def _run(gen, disc, S, B, steps, use_graph=1, init_seed=8, f16=1):
    """`steps`: a list of callables (net, ds, seed) -> stats; returns the state after them and the stats"""
    from face_generator_b200.lib import NET_D, NET_G
    ctx = _ctx(B, f16)
    ctx.set_option("use_graph", use_graph)
    net = _net(ctx, S, gen, disc)
    rng = np.random.default_rng(init_seed)
    net.set_params(NET_G, V.trained_like(V.G_layout(gen, 3), rng).astype(np.float32))
    net.set_params(NET_D, V.trained_like(V.D_layout(disc, 3, S), rng, 1.0).astype(np.float32))
    ds = _dataset(ctx)
    stats = [f(net, ds, 20 + i) for i, f in enumerate(steps)]
    state = _state(net)
    ds.close()
    net.close()
    ctx.close()
    return state, stats


def _host_inputs(ds, ctx, S, B, seed):
    from face_generator_b200.dataset import noise_uniform
    cs, Bh = S // 2, B // 2
    _, cr, dr = ds.gather_c2f(ds.draw(8 * seed, Bh), cs, S)
    _, cf, _ = ds.gather_c2f(ds.draw(8 * seed + 1, Bh), cs, S)
    _, cg, _ = ds.gather_c2f(ds.draw(8 * seed + 2, B), cs, S)
    nD, nG = noise_uniform(ctx, 8 * seed + 3, (Bh, 1, S, S)), noise_uniform(ctx, 8 * seed + 4, (B, 1, S, S))
    return dr, np.concatenate([cr, cf]), nD, cg, nG


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("B,f16", [(64, 1), (130, 0)])  # 130: an odd half batch of 65
@pytest.mark.parametrize("S", SIZES)
@pytest.mark.parametrize("gen,disc", PAIRS)
def test_device_fed_equals_host_fed_and_graphs_and_seeds(gen, disc, S, B, f16):
    import face_generator_b200 as fg
    h = fg.hyper_default()
    dev_step = lambda net, ds, seed: net.train_step_dataset(ds, h, B, S // 2, seed)
    host_step = lambda net, ds, seed: net.train_step(h, B, *_host_inputs(ds, net.ctx, S, B, seed), None, None, seed)
    a, sa = _run(gen, disc, S, B, [dev_step] * 3, f16=f16)
    b, sb = _run(gen, disc, S, B, [host_step] * 3, f16=f16)
    _same(a, b)
    assert sa == sb
    c, sc = _run(gen, disc, S, B, [dev_step] * 3, use_graph=0, f16=f16)  # eager against captured + replayed
    _same(a, c)
    d, _ = _run(gen, disc, S, B, [dev_step] * 3, f16=f16)  # the same seed twice
    _same(a, d)
    it = lambda net, ds, seed: net.train_step_dataset_iters(ds, h, B, 2, 1, S // 2, seed)
    e, _ = _run(gen, disc, S, B, [it] * 2, f16=f16)
    f, _ = _run(gen, disc, S, B, [it] * 2, use_graph=0, f16=f16)
    _same(e, f)


@pytest.mark.parametrize("S", SIZES)
def test_create_nets_with_the_defaults_is_create_sized(S):
    """fg_c2f_create_nets(ctx, S, FG_C2F_G_D, FG_C2F_D_C) and fg_c2f_create_sized(ctx, S): the same bits over three
    train steps (the net built through the descriptor is the default pair's)"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G, _check
    h = fg.hyper_default()
    B = 64
    states = []
    for how in ("nets", "sized"):
        ctx = _ctx(B, 1)
        hnd = ctypes.c_void_p()
        if how == "nets":
            _check(ctx.lib.fg_c2f_create_nets(ctx.h, S, 1, 1, ctypes.byref(hnd)), "fg_c2f_create_nets")
        else:
            _check(ctx.lib.fg_c2f_create_sized(ctx.h, S, ctypes.byref(hnd)), "fg_c2f_create_sized")
        assert ctx.lib.fg_c2f_get_gen(hnd) == 1 and ctx.lib.fg_c2f_get_disc(hnd) == 1
        net = fg.C2f.__new__(fg.C2f)
        net.ctx, net.lib, net.C, net.h, net.S = ctx, ctx.lib, 3, hnd, S
        net.generator, net.discriminator = "create_G_d", "create_D_c"
        net.nG, net.nD = int(ctx.lib.fg_c2f_param_count(0, 3)), int(ctx.lib.fg_c2f_param_count_sized(1, 3, S))
        net.mask_per_sample = int(ctx.lib.fg_c2f_mask_per_sample_sized(S))
        rng = np.random.default_rng(12)
        net.set_params(NET_G, V.trained_like(V.G_layout("create_G_d", 3), rng).astype(np.float32))
        net.set_params(NET_D, V.trained_like(V.D_layout("create_D_c", 3, S), rng, 1.0).astype(np.float32))
        ds = _dataset(ctx)
        st = [net.train_step_dataset(ds, h, B, S // 2, 30 + i) for i in range(3)]
        states.append((_state(net), st))
        ds.close()
        net.close()
        ctx.close()
    _same(states[0][0], states[1][0])
    assert states[0][1] == states[1][1]


def test_unknown_nets_are_refused_before_allocation():
    from face_generator_b200.lib import FGError
    import face_generator_b200 as fg
    ctx = _ctx(8, 1)
    hnd = ctypes.c_void_p()
    for g, d in ((5, 1), (1, 4), (-1, 1), (1, -1)):
        assert ctx.lib.fg_c2f_create_nets(ctx.h, 32, g, d, ctypes.byref(hnd)) == -4  # FG_ERR_UNSUPPORTED
        assert not hnd.value
    assert ctx.lib.fg_c2f_create_nets(ctx.h, 48, 2, 2, ctypes.byref(hnd)) == -4
    with pytest.raises(FGError, match="unknown c2f generator"):
        fg.C2f(ctx, 32, "create_G_e")
    net = fg.C2f(ctx, 32, "create_G_a", "create_D_b")
    assert (ctx.lib.fg_c2f_get_gen(net.h), ctx.lib.fg_c2f_get_disc(net.h)) == (2, 3)
    with pytest.raises(FGError, match="keep flags"):  # host keep flags are sized against the held D
        net.D_forward(np.zeros((4, 3, 32, 32), np.float32), np.zeros((4, 3, 32, 32), np.float32),
                      masks=np.ones((4, 100), np.float32))
    net.close()
    ctx.close()


# ---- refine and Parzen ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gen,disc", PAIRS)
def test_refine_against_the_restatement(gen, disc):
    from face_generator_b200 import pyramid
    from face_generator_b200.lib import NET_D, NET_G
    C, S, N, T, insz = 3, 32, 6, 4, 16
    rng = np.random.default_rng(77)
    PG = V.trained_like(V.G_layout(gen, C), rng).astype(np.float32)
    PD = V.trained_like(V.D_layout(disc, C, S), rng, 1.0).astype(np.float32)
    images = rng.random((N, C, insz, insz)).astype(np.float32)
    noise = rng.uniform(-1, 1, (N, T, 1, S, S)).astype(np.float32)
    masks = (rng.random((N, T, V.mask_per_sample(disc, S))) < 0.5).astype(np.float32)
    ctx = _ctx(N * T, 1)
    net = _net(ctx, S, gen, disc)
    net.set_params(NET_G, PG)
    net.set_params(NET_D, PD)
    res = [pyramid.refine(net, images, T, chunk, True, 0, noise, masks) for chunk in (1, 4, 6)]
    up = pyramid.image_scale(ctx, images, S)
    net.close()
    ctx.close()
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert np.array_equal(a, b)  # independent of chunk
    out, pick, pred = res[0]
    cond = dev(np.repeat(up, T, axis=0))
    diff = V.G_forward(dev(PG), dev(noise.reshape(N * T, 1, S, S)), cond, gen, C)
    ref = V.D_forward(dev(PD), diff, cond, dev(masks.reshape(N * T, -1)), disc, C, S).reshape(N, T)
    assert rel(pred, ref) < TOL
    top = np.sort(ref.cpu().numpy(), axis=1)
    clear = (top[:, -1] - top[:, -2]) > 1e-4  # where no two tries are within the bar of each other
    ref_pick = ref.argmax(1).cpu().numpy()
    assert np.array_equal(pick[clear], ref_pick[clear])
    want = dev(up) + diff.reshape(N, T, C, S, S)[torch.arange(N), torch.as_tensor(pick).long().cuda()]
    assert rel(out, want) < TOL


def test_parzen_dist_on_a_variant_pair():
    from face_generator_b200.lib import NET_G, _check
    gen, disc, C, S, K = "create_G_b", "create_D_a", 3, 32, 16
    rng = np.random.default_rng(5)
    PG = V.trained_like(V.G_layout(gen, C), rng).astype(np.float32)
    noise = rng.uniform(-1, 1, (K, 1, S, S)).astype(np.float32)
    coarse, fine = rng.random((C, S, S)).astype(np.float32), rng.random((C, S, S)).astype(np.float32)
    ctx = _ctx(K, 1)
    net = _net(ctx, S, gen, disc)
    net.set_params(NET_G, PG)
    d = ctypes.c_float(0)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    _check(ctx.lib.fg_c2f_parzen_dist(net.h, P(noise), P(coarse), P(fine), K, ctypes.byref(d)), "fg_c2f_parzen_dist")
    net.close()
    ctx.close()
    cond = dev(np.repeat(coarse[None], K, axis=0))
    gen_img = V.G_forward(dev(PG), dev(noise), cond, gen, C) + cond
    ref = float((gen_img - dev(fine)[None]).flatten(1).norm(dim=1).min())
    assert abs(d.value - ref) / ref < TOL
