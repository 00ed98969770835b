"""tests/d_ref.py (the per-launch float64 yardstick of tests/test_gpu_d_launches.py) chained into the whole 32x32 D,
forward and backward, and pinned to the C++ oracle's D (O.f64.D()) at batch 4, in training and evaluate mode; its
BCE, confusion counts and the conditions it returns checked on their own."""
import numpy as np
import pytest

import d_ref as R
import torch_ref as TR
from oracle import oracle as O

torch = pytest.importorskip("torch")
TOL = 1e-12
C = 3


def t64(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64)


def rel(a, b):
    a, b = t64(a), t64(b)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def d_chain(P, img, masks, dout):
    """the whole D forward and backward composed from d_ref's launches: (out, dP, dimg), img NCHW like the oracle's"""
    p = TR._split(P, O.D_layout(C))
    x =img.permute(0, 2, 3, 1).contiguous()
    zs, ins = [], []
    cur = x
    for i in range(4):
        ins.append(cur)
        z = R.conv_fwd(cur, p["c%dW" % (i + 1)], p["c%db" % (i + 1)])
        zs.append(z)
        cur = R.act_pool_fwd(z, p["a%d" % (i + 1)], masks, R.MOFF[i])
    p4 = cur
    zl1 = R.view2048(p4) @ p["L1W"].t() + p["L1b"]
    hl1 = R.lin_act_drop_fwd(zl1, p["a5"], masks, R.MOFF_L1)
    zl2 = hl1 @ p["L2W"].t() + p["L2b"]
    hl2 = R.lin_act_drop_fwd(zl2, p["a6"], masks, R.MOFF_L2)
    logit = R.gemv_fwd(hl2, p["L3W"].reshape(512), p["L3b"])
    out = R.sigmoid_out(logit)
    g = {k: torch.zeros_like(v) for k, v in p.items()}
    dlogit = R.sigmoid_grad(dout, out)
    wg = R.gemv_wgrad(hl2, dlogit)
    g["L3W"][:], g["L3b"][:] = wg["dw"].reshape(1, 512), wg["db"]
    dh = R.gemv_dgrad(dlogit, p["L3W"].reshape(512))
    for zl, hin, W, b, a, moff in ((zl2, hl1, "L2W", "L2b", "a6", R.MOFF_L2), (zl1, R.view2048(p4), "L1W", "L1b", "a5", R.MOFF_L1)):
        r = R.lin_act_drop_bwd(dh, zl, p[a], masks, moff)
        g[a][:] = r["dslope"]
        g[W][:], g[b][:] = r["dz"].t() @ hin, r["dz"].sum(0)
        dh = r["dz"] @ p[W]
    dp = R.view2048_bwd(dh)
    for i in range(3, -1, -1):
        r = R.act_pool_bwd(dp, zs[i], p["a%d" % (i + 1)], masks, R.MOFF[i])
        g["a%d" % (i + 1)][:], g["c%db" % (i + 1)][:] = r["dslope"], r["dbias"]
        Wn = "c%dW" % (i + 1)
        g[Wn][:] = R.conv_wgrad(ins[i], p[Wn].shape, r["dz"])
        dp = R.conv_dgrad(ins[i].shape, p[Wn], r["dz"])
    dP = torch.cat([g[k].reshape(-1) for k in O.D_layout(C)])
    return out, dP, dp.permute(0, 3, 1, 2)


def case(seed, B=4):
    rng = np.random.default_rng(seed)
    P = TR.trained_like_D(C, rng)
    img = rng.random((B, C, 32, 32))
    masks = TR.make_masks(B, rng)
    dout = rng.standard_normal(B)
    return P, img, masks, dout


@pytest.mark.parametrize("training", [True, False])
def test_chain_matches_oracle(training):
    P, img, masks, dout = case(5 + training)
    D = O.f64.D()
    ref_out = D.forward(P, img, masks if training else None, training=training)
    ref_dP, ref_dimg = D.backward(dout)
    out, dP, dimg = d_chain(t64(P), t64(img), t64(masks) if training else None, t64(dout))
    assert rel(out, ref_out) < TOL
    assert rel(dimg, ref_dimg) < TOL
    for k, (o, s) in O.D_layout(C).items():
        n = int(np.prod(s))
        assert rel(dP[o:o + n], ref_dP[o:o + n]) < TOL, k


def test_view2048_is_torch_flatten_of_nchw():
    p4 = torch.randn(3, 2, 2, 512, dtype=torch.float64)
    assert torch.equal(R.view2048(p4), p4.permute(0, 3, 1, 2).reshape(3, 2048))
    assert torch.equal(R.view2048_bwd(R.view2048(p4)), p4)


def test_sigmoid_bce_matches_oracle_and_counts_ties_as_predicted_0():
    logit = t64([0.0, 0.0, 3.0, -2.0, 100.0, -200.0, 1e-3, -1e-3])
    r = R.sigmoid_bce(logit, 4)
    y = r["y"].numpy()
    t = np.array([1, 1, 1, 1, 0, 0, 0, 0], np.float64)
    assert y[0] == 0.5 and y[4] == 1.0 and y[5] == 0.0
    assert abs(float(r["loss"]) - O.f64.bce_fwd(y, t)) < 1e-14
    assert rel(r["dlogit"], O.f64.bce_bwd(y, t) * y * (1 - y)) < 1e-14
    # y = 0.5 is "predicted 0" for both targets; y(100) = 1 is predicted 1, y(-200) = 0 predicted 0
    assert r["conf"] == [1, 3, 2, 2]
    assert float(r["dlogit"][4]) == 0.0 and float(r["dlogit"][5]) == 0.0  # saturated: exactly 0
    half = R.sigmoid_bce(torch.zeros(6, dtype=torch.float64), 3)
    assert abs(float(half["loss"]) - np.log(2)) < 1e-11 and half["conf"] == [0, 3, 0, 3]


def test_conditions_are_sums_of_absolute_terms():
    g = torch.Generator().manual_seed(1)
    z = torch.randn(2, 4, 4, 8, generator=g, dtype=torch.float64)
    z[0, 0, 0, :] = 0.0
    dp = torch.randn(2, 2, 2, 8, generator=g, dtype=torch.float64)
    masks = (torch.rand(2, 1984, generator=g) < 0.5).double()
    r = R.act_pool_bwd(dp, z, 0.25, masks, 64)
    gg = dp.repeat_interleave(2, 1).repeat_interleave(2, 2) * 0.25 * masks[:, 64:72].reshape(2, 1, 1, 8)
    neg = ~(z > 0)
    assert torch.allclose(r["dslope_cond"], (gg * z).abs()[neg].sum(), rtol=1e-14, atol=0)
    assert torch.equal(r["dz"][0, 0, 0], 0.25 * gg[0, 0, 0])  # z == 0 takes the slope branch
    assert torch.allclose(r["dbias_cond"], r["dz"].abs().sum((0, 1, 2)), rtol=1e-14, atol=0)
    assert bool((r["dbias"].abs() <= r["dbias_cond"]).all()) and abs(float(r["dslope"])) <= float(r["dslope_cond"])
    h, dl = torch.randn(5, 16, generator=g, dtype=torch.float64), torch.randn(5, generator=g, dtype=torch.float64)
    w = R.gemv_wgrad(h, dl)
    assert torch.allclose(w["dw_cond"], (h * dl[:, None]).abs().sum(0), rtol=1e-14, atol=0)
    assert float(w["db_cond"]) == float(dl.abs().sum())
