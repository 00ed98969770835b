"""Every launch of the 32x32 discriminator held to float64 on its own inputs, forward and backward.

One fg_D_forward(training, masks) and one fg_D_backward(dout, want_wgrad=1) per case, with option debug_keep, so
that the backward's scratch tensors are kept per layer ("Dbwd.*").  Each launch is compared with tests/d_ref.py (the
float64 restatement, pinned to the C++ oracle by tests/test_d_ref_cpu.py) computed on the CUDA path's own input
tensors, so errors do not accumulate and PReLU's branch is never ambiguous.  Both operand splits run (mma_f16 = 1:
3xFP16, mma_f16 = 0: 3xTF32 with the TF32 hi/lo split written by the act/pool kernels themselves), at batch 256 and
130 (several grid-stride passes, the 1056-block cap of the backward reductions) and at batch 7 and 1 (grids smaller
than one wave).

The data reaches the edges: a band of the image is zero and D.C1's bias is 0, so z1 is exactly 0 under the band, whole
pooled pixels of p1 are 0 and, with half of D.C2's bias at 0, z2 has exact zeros too (PReLU's `z > 0` rule forward
and backward); each layer's SpatialDropout flags have their own density (0.2, 0.5, 0.8, 0.65, one sample's D.C2
plane all dropped) and so do the two Dropout rows, so a flag read at another layer's offset changes the result.

Bars (err / bar is what the tests compare with 1):
  * elementwise outputs (p, h, dz, dzl, dh, dlogit, out): max|err| <= ETOL * max|ref| per channel of an NHWC tensor
    and per sample of a [B][512] or [B] tensor (a reference that is exactly 0 there must be matched exactly);
  * convolution and Linear launches: KTOL normwise; weight gradients per output channel, against WTOL;
  * reductions (PReLU slope, bias and D.L3 gradients, the BCE loss): |got - ref| <= RTOL * sum|terms|, per channel for
    bias gradients (the loss adds BCE's eps, which fp32 drops next to an output of order 1).
The largest err / bar of each family measured on the H100 is in DESIGN.md section 5.

The sigmoid + BCE of the train step runs with D.L3W = 0 and D.L3b = 0, +100 and -100: logits exactly 0 give y = 0.5,
which counts as "predicted 0", and a loss of log 2; +-100 saturate y to exactly 1 or 0, so D's gradients are exactly
0 and Adam leaves D bitwise unchanged.  fg_prelu_backward, the shared PReLU backward with its ordered slope reduction
over up to 1056 blocks, runs from 1 element to 2^24 + 3, with an accumulating dslope, host and device pointers, and
twice to show the slope sum is bit-reproducible.

Deliberate bugs this file catches (each made once in k_elem.cu, run on the H100 and reverted; the test that turned
red in brackets):
  1. block_colsum_rows' last block sums gridDim.x - 1 rows  [test_D_launches: c<i>b and a<i> gradients]
  2. d_act_pool_bwd_kernel takes v == 0 as positive  [test_D_launches: dz1 / dz2 at the exact zeros]
  3. d_act_pool_fwd_kernel reads the SpatialDropout flags at the previous layer's offset  [test_D_launches: p2..p4]
  4. lin_act_drop_bwd_kernel drops the 1/(1-p) scale  [test_D_launches: dzl1 / dzl2]
  5. gemv_wgrad_kernel sums b < B - 1  [test_D_launches: L3W gradient]
  6. sigmoid_bce_kernel counts y >= 0.5 as predicted 1  [test_train_step_sigmoid_bce: L3b = 0]
  7. prelu_bwd_kernel's last block sums min(gridDim.x, 132) rows  [test_prelu_backward_lop: n > 33 792]
"""
import numpy as np
import pytest

import d_ref as R
import parity_utils as PU
import torch_ref as TR
from oracle import oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
C = 3
ETOL = 1e-6  # elementwise: a few fp32 roundings
KTOL = 1e-5  # one convolution / Linear launch on identical inputs (tests/test_gpu_headline.py)
WTOL = 3e-5  # a weight gradient per output channel (a channel of small gradients; measured up to 4.1e-6)
RTOL = 1e-5  # reductions, relative to the sum of |terms|: 16-term fp32 partials summed in double
FLT_MIN = float(np.finfo(np.float32).tiny)  # below it fp32 holds no relative precision (sigmoid(-100) is 0)
DEV = "cuda"


@pytest.fixture(scope="module")
def fg():
    import face_generator_b200 as fg
    return fg


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)


def _ratio(d, s):
    """d / s elementwise, with 0 / 0 = 0 and d / 0 = inf (a reference of exactly 0 must be matched exactly)"""
    return torch.where(s > 0, d / s.clamp_min(1e-300), torch.where(d > 0, float("inf"), 0.0))


def elem_err(got, ref, per="last"):
    """max|err| / max|ref| per group: per channel of an NHWC tensor (per="last"), per row of a [B][N] tensor
    (per="row"), per element of a vector (per="elem", where an error below FLT_MIN always passes); the largest over
    the groups"""
    d, r = (got - ref).abs(), ref.abs()
    if per == "last":
        d, r = d.reshape(-1, d.shape[-1]).max(0).values, r.reshape(-1, r.shape[-1]).max(0).values
    elif per == "row":
        d, r = d.reshape(d.shape[0], -1).max(1).values, r.reshape(r.shape[0], -1).max(1).values
    else:
        r = r.clamp_min(FLT_MIN / ETOL)
    return float(_ratio(d, r).max())


def norm_err(got, ref):
    return float(_ratio((got - ref).abs().max(), ref.abs().max()))


def red_err(got, ref, cond):
    return float(_ratio((got - ref).abs(), torch.as_tensor(cond, dtype=torch.float64, device=DEV)).max())


def masks_for(B, rng):
    """keep flags with a different density per layer and row, and one sample's D.C2 plane all dropped"""
    m = np.zeros((B, O.MASK_PER_SAMPLE), np.float32)
    for i, dens in enumerate((0.2, 0.5, 0.8, 0.65)):
        m[:, R.MOFF[i]:R.MOFF[i] + R.COUT[i]] = rng.random((B, R.COUT[i])) < dens
    m[:, R.MOFF_L1:R.MOFF_L1 + 512] = rng.random((B, 512)) < 0.3
    m[:, R.MOFF_L2:R.MOFF_L2 + 512] = rng.random((B, 512)) < 0.7
    if B > 1:
        m[B // 2, R.MOFF[1]:R.MOFF[1] + R.COUT[1]] = 0
    return m


def edge_case(B, seed):
    """parameters, image and dout with exact zeros: rows 0..7 of every image and D.C1's bias are 0, so z1 is exactly 0
    in rows 0..6 and p1 in rows 0..2; half of D.C2's bias is 0, so z2 is exactly 0 there in rows 0..1"""
    rng = np.random.default_rng(seed)
    L = O.D_layout(C)
    P = TR.trained_like_D(C, rng).astype(np.float32)
    o, s = L["c1b"]
    P[o:o + s[0]] = 0
    o, s = L["c2b"]
    P[o:o + s[0]:2] = 0
    img = rng.random((B, C, 32, 32)).astype(np.float32)
    img[:, :, :8, :] = 0
    return P, img, masks_for(B, rng), rng.standard_normal(B).astype(np.float32)


def run_D(fg, B, f16, training, seed):
    from face_generator_b200.lib import NET_D
    P, img, masks, dout = edge_case(B, seed)
    ctx = fg.Context(0, max_batch=max(4, B + B % 2), channels=C)  # a context holds an even batch of at least 4
    ctx.set_option("mma_f16", f16)
    ctx.set_option("debug_keep", 1)
    ctx.set_params(NET_D, P)
    ctx.D_forward(img, masks=masks if training else None, training=training)
    ctx.zero_grads(NET_D)
    ctx.D_backward(dout)
    T = {}
    shapes = {"z%d" % (i + 1): (R.HW[i], R.COUT[i]) for i in range(4)}
    shapes.update({"p%d" % (i + 1): (R.HW[i] // 2, R.COUT[i]) for i in range(4)})
    for k, (H, Cc) in shapes.items():
        T[k] = dev(ctx.debug_tensor("D." + k).reshape(B, H, H, Cc))
    for k in ("zl1", "hl1", "zl2", "hl2"):
        T[k] = dev(ctx.debug_tensor("D." + k).reshape(B, 512))
    for k in ("logit", "out", "dlogit"):
        T[k] = dev(ctx.debug_tensor("D." + k))
    T["dx"] = dev(ctx.debug_tensor("D.dx").reshape(B, 32, 32, C))
    for k in ("dh3", "dzl2", "dh2", "dzl1"):
        T[k] = dev(ctx.debug_tensor("Dbwd." + k).reshape(B, 512))
    for i in range(4):
        H, Cc = R.HW[i], R.COUT[i]
        T["dp%d" % (i + 1)] = dev(ctx.debug_tensor("Dbwd.dp%d" % (i + 1)).reshape(B, H // 2, H // 2, Cc))
        T["dz%d" % (i + 1)] = dev(ctx.debug_tensor("Dbwd.dz%d" % (i + 1)).reshape(B, H, H, Cc))
    gD = ctx.get_grads(NET_D)
    ctx.close()
    p = TR._split(dev(P), O.D_layout(C))
    g = TR._split(dev(gD), O.D_layout(C))
    return T, p, g, dev(img).permute(0, 2, 3, 1).contiguous(), dev(masks) if training else None, dev(dout)


def D_launch_errors(T, p, g, x, m, dout):
    """{check: (err / bar)} for every launch of one D forward and backward"""
    e = {}
    ins = [x] + [T["p%d" % i] for i in (1, 2, 3)]
    # ---- forward ----
    for i in range(4):
        n = i + 1
        e["fwd.z%d" % n] = norm_err(T["z%d" % n], R.conv_fwd(ins[i], p["c%dW" % n], p["c%db" % n])) / KTOL
        e["fwd.p%d" % n] = elem_err(T["p%d" % n], R.act_pool_fwd(T["z%d" % n], p["a%d" % n], m, R.MOFF[i])) / ETOL
    e["fwd.zl1"] = norm_err(T["zl1"], R.view2048(T["p4"]) @ p["L1W"].t() + p["L1b"]) / KTOL
    e["fwd.hl1"] = elem_err(T["hl1"], R.lin_act_drop_fwd(T["zl1"], p["a5"], m, R.MOFF_L1), "row") / ETOL
    e["fwd.zl2"] = norm_err(T["zl2"], T["hl1"] @ p["L2W"].t() + p["L2b"]) / KTOL
    e["fwd.hl2"] = elem_err(T["hl2"], R.lin_act_drop_fwd(T["zl2"], p["a6"], m, R.MOFF_L2), "row") / ETOL
    w3 = p["L3W"].reshape(512)
    e["fwd.logit"] = norm_err(T["logit"], R.gemv_fwd(T["hl2"], w3, p["L3b"])) / KTOL
    e["fwd.out"] = elem_err(T["out"], torch.sigmoid(T["logit"]), "elem") / ETOL
    # ---- backward: D.L3 ----
    e["bwd.dlogit"] = elem_err(T["dlogit"], R.sigmoid_grad(dout, T["out"]), "elem") / ETOL
    r = R.gemv_wgrad(T["hl2"], T["dlogit"])
    e["bwd.L3W"] = red_err(g["L3W"].reshape(512), r["dw"], r["dw_cond"]) / RTOL
    e["bwd.L3b"] = red_err(g["L3b"], r["db"], r["db_cond"]) / RTOL
    e["bwd.dh3"] = elem_err(T["dh3"], R.gemv_dgrad(T["dlogit"], w3), "row") / ETOL
    # ---- D.L2 and D.L1, each behind its PReLU + Dropout ----
    for dh, zl, dzl, hin, W, b, a, moff, dout_name in (
            ("dh3", "zl2", "dzl2", T["hl1"], "L2W", "L2b", "a6", R.MOFF_L2, "dh2"),
            ("dh2", "zl1", "dzl1", R.view2048(T["p4"]), "L1W", "L1b", "a5", R.MOFF_L1, "dp4")):
        r = R.lin_act_drop_bwd(T[dh], T[zl], p[a], m, moff)
        e["bwd." + dzl] = elem_err(T[dzl], r["dz"], "row") / ETOL
        e["bwd." + a] = red_err(g[a], r["dslope"], r["dslope_cond"]) / RTOL
        dz = T[dzl]
        e["bwd." + W] = elem_err(g[W], dz.t() @ hin, "row") / WTOL
        e["bwd." + b] = red_err(g[b], dz.sum(0), dz.abs().sum(0)) / RTOL
        dx = dz @ p[W]
        e["bwd." + dout_name] = norm_err(T[dout_name], R.view2048_bwd(dx) if W == "L1W" else dx) / KTOL
    # ---- D.C4 .. D.C1: act/pool backward (+ slope and bias sums), then the convolution's gradients ----
    for i in range(3, -1, -1):
        n = i + 1
        r = R.act_pool_bwd(T["dp%d" % n], T["z%d" % n], p["a%d" % n], m, R.MOFF[i])
        e["bwd.dz%d" % n] = elem_err(T["dz%d" % n], r["dz"]) / ETOL
        e["bwd.a%d" % n] = red_err(g["a%d" % n], r["dslope"], r["dslope_cond"]) / RTOL
        e["bwd.c%db" % n] = red_err(g["c%db" % n], r["dbias"], r["dbias_cond"]) / RTOL
        dz = T["dz%d" % n]
        W = p["c%dW" % n]
        e["bwd.c%dW" % n] = elem_err(g["c%dW" % n], R.conv_wgrad(ins[i], W.shape, dz), "row") / WTOL
        e["bwd.%s" % ("dp%d" % i if i else "dx")] = norm_err(T["dp%d" % i if i else "dx"], R.conv_dgrad(ins[i].shape, W, dz)) / KTOL
    return e


def report(tag, e):
    worst = max(e, key=e.get)
    print("\n[d-launches] %s worst %s %.3g | %s" % (tag, worst, e[worst], " ".join("%s=%.3g" % kv for kv in sorted(e.items()))))


CASES = [(256, 1, 1), (256, 0, 1), (130, 1, 1), (130, 0, 1), (7, 1, 1), (7, 0, 1), (1, 1, 1), (1, 0, 1), (130, 1, 0), (7, 0, 0)]


@pytest.mark.parametrize("B,f16,training", CASES, ids=["B%d-f16_%d-%s" % (b, f, "train" if t else "eval") for b, f, t in CASES])
def test_D_launches(fg, B, f16, training):
    T, p, g, x, m, dout = run_D(fg, B, f16, training, seed=7000 + B)
    # the edge data did what it is for: exact zeros in z1, whole pooled pixels of p1 and z2
    assert bool((T["z1"][:, :7] == 0).all()) and bool((T["p1"][:, :3] == 0).all())
    assert bool((T["z2"][:, :2, :, ::2] == 0).all())
    e = D_launch_errors(T, p, g, x, m, dout)
    report("B=%d mma_f16=%d training=%d" % (B, f16, training), e)
    bad = {k: v for k, v in e.items() if not v <= 1.0}
    assert not bad, bad


@pytest.mark.parametrize("B", [256, 130])
@pytest.mark.parametrize("L3b", [0.0, 100.0, -100.0, None], ids=["L3b_0", "L3b_+100", "L3b_-100", "random"])
def test_train_step_sigmoid_bce(fg, B, L3b):
    """loss_D, loss_G and the confusion counts of fg_train_step against d_ref.sigmoid_bce on the kept logits"""
    from face_generator_b200.lib import NET_D, NET_G
    if L3b is None and B != 130:
        pytest.skip("the ordinary case runs at the odd half-batch 65")
    case = PU.make_case(B, C, seed=7100 + B, init="trained")
    PD = case["PD"].astype(np.float32)
    if L3b is not None:
        L = O.D_layout(C)
        PD[L["L3W"][0]:L["L3W"][0] + 512] = 0
        PD[L["L3b"][0]] = L3b
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_option("debug_keep", 1)
    ctx.set_params(NET_G, case["PG"])
    ctx.set_params(NET_D, PD)
    hyper = fg.hyper_default(D_L1=0.0, D_L2=0.0)
    st = ctx.train_step(hyper, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
    kept = {k: dev(ctx.debug_tensor(k)) for k in ("Dstep.logit", "Dstep.out", "D.logit", "D.out", "D.dlogit")}
    gD, PD_after = ctx.get_grads(NET_D), ctx.get_params(NET_D)
    ctx.close()
    e = {}
    for what, logit, out, n_ones, loss in (("D", "Dstep.logit", "Dstep.out", B // 2, st["loss_D"]),
                                           ("G", "D.logit", "D.out", B, st["loss_G"])):
        e["out_" + what] = elem_err(kept[out], torch.sigmoid(kept[logit]), "elem") / ETOL
        r = R.sigmoid_bce(kept[logit], n_ones, y=kept[out])
        # + 2 eps: the kernel adds eps to log's argument in fp32, where it vanishes next to an argument x >= 1/2 and
        # so moves that term by at most eps / x
        e["loss_" + what] = abs(loss - float(r["loss"])) / (RTOL * float(r["loss_cond"]) + 2 * R.BCE_EPS)
        if what == "D":
            assert st["conf"] == r["conf"], (st["conf"], r["conf"])
        else:
            e["dlogit_G"] = elem_err(kept["D.dlogit"], r["dlogit"], "elem") / ETOL
    report("train step B=%d L3b=%s" % (B, L3b), e)
    bad = {k: v for k, v in e.items() if not v <= 1.0}
    assert not bad, bad
    if L3b == 0.0:
        assert bool((kept["Dstep.logit"] == 0).all()) and bool((kept["Dstep.out"] == 0.5).all())
        assert st["conf"] == [0, B // 2, 0, B // 2]  # y = 0.5 is "predicted 0"
        assert abs(st["loss_D"] - np.log(2)) < 1e-6
    elif L3b is not None:
        sat = 1.0 if L3b > 0 else 0.0
        assert bool((kept["Dstep.out"] == sat).all()) and bool((kept["D.out"] == sat).all())
        assert bool((kept["D.dlogit"] == 0).all())
        assert not np.any(gD), "saturated D: every D gradient is exactly 0"
        assert np.array_equal(PD_after.view(np.uint32), PD.view(np.uint32)), "Adam moved D on zero gradients"
        assert st["conf"] == ([B // 2, 0, B // 2, 0] if L3b > 0 else [0, B // 2, 0, B // 2])


@pytest.mark.parametrize("n", [1, 255, 257, 270337, 2 ** 24 + 3])
@pytest.mark.parametrize("where", ["host", "device"])
def test_prelu_backward_lop(fg, n, where):
    """fg_prelu_backward = prelu_bwd_kernel, whose ordered slope sum runs over up to 1056 blocks (270 337 elements is
    one past a full 1056 x 256 grid): dx elementwise, dslope (accumulating onto 0.75) against the condition-aware bar,
    and two identical calls bitwise equal"""
    from face_generator_b200.lib import _ptr
    gen = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, generator=gen, device="cuda", dtype=torch.float32)
    x[::7] = 0.0  # PReLU's kink: the slope branch, adding 0 to dslope
    dy = torch.randn(n, generator=gen, device="cuda", dtype=torch.float32)
    a, ds0 = 0.25, 0.75
    ctx = fg.Context(0, max_batch=8, channels=C)
    lib, h = ctx.lib, ctx.h
    torch.cuda.synchronize()
    outs = []
    for _ in range(2):
        if where == "host":
            xs, dys = x.cpu().numpy(), dy.cpu().numpy()
            sl, dx, ds = np.array([a], np.float32), np.empty(n, np.float32), np.array([ds0], np.float32)
            assert lib.fg_prelu_backward(h, _ptr(xs), _ptr(sl), _ptr(dys), _ptr(dx), _ptr(ds), n) == 0, lib.fg_last_error()
            outs.append((torch.as_tensor(dx, device="cuda"), float(ds[0])))
        else:
            sl = torch.tensor([a], device="cuda")
            dx = torch.empty(n, device="cuda")
            ds = torch.tensor([ds0], device="cuda")
            torch.cuda.synchronize()
            assert lib.fg_prelu_backward(h, _ptr(x.data_ptr()), _ptr(sl.data_ptr()), _ptr(dy.data_ptr()), _ptr(dx.data_ptr()),
                                         _ptr(ds.data_ptr()), n) == 0, lib.fg_last_error()
            ctx.sync()
            outs.append((dx, float(ds.item())))
    ctx.close()
    x64, dy64 = x.double(), dy.double()
    pos = x64 > 0
    t = torch.where(pos, torch.zeros_like(x64), dy64 * x64)
    ref_dx = torch.where(pos, dy64, a * dy64)
    (dx, ds), (dx2, ds2) = outs
    e = dict(dx=norm_err(dx.double(), ref_dx) / ETOL,
             dslope=abs(ds - (ds0 + float(t.sum()))) / (RTOL * (ds0 + float(t.abs().sum()))))
    report("prelu_bwd n=%d %s" % (n, where), e)
    assert e["dx"] <= 1.0 and e["dslope"] <= 1.0, e
    assert np.float32(ds).view(np.uint32) == np.float32(ds2).view(np.uint32), (ds, ds2)
    assert torch.equal(dx, dx2)
