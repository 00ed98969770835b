"""Shared helpers for the parity tests: seeded cases, oracle runs, error norms."""
import numpy as np

from oracle import oracle as O
from face_generator_b200 import layouts as LY

HYPER = dict(lr_D=1e-3, lr_G=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, D_L1=0.0, D_L2=1e-4, G_L1=0.0, G_L2=0.0,
             D_clamp=1.0, G_clamp=5.0)


def relerr(a, b):
    """normwise relative error max|a-b| / max|b| (the parity bar is 1e-4, BASELINE.json north_star)."""
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def make_masks(B, rng):
    m = np.zeros((B, O.MASK_PER_SAMPLE))
    m[:, :960] = rng.random((B, 960)) < 0.8
    m[:, 960:] = rng.random((B, 1024)) < 0.5
    return m


def make_case(B, C, seed, init="trained"):
    rng = np.random.default_rng(seed)
    if init in ("trained", "smooth"):
        # "smooth": all PReLU slopes = 1 (identity) -> the loss is differentiable everywhere, so gradients can be
        # compared strictly; with real slopes a pre-activation within fp32 noise of 0 may take the other branch
        sl = 1.0 if init == "smooth" else 0.25
        PG = LY.trained_like_init(LY.G_layout(C), rng, slope=sl)
        PD = LY.trained_like_init(LY.D_layout(C), rng, 1.4, slope=sl)
        if init == "smooth":
            # with slopes 1 nothing damps D's activations: shrink its last layer so that the logits stay O(1).  With
            # |logit| > 17 the fp32 sigmoid saturates, the reference's composed gradient is exactly 0 (SURVEY.md appendix
            # 12) and a "strict gradient" case would compare nothing but zeros / near-saturation rounding noise
            o, shape = LY.D_layout(C)[0]["L3W"]
            PD[o:o + int(np.prod(shape))] *= 0.1
    else:  # the reference's own init: N(0, 0.005^2) weights (incl. BN gamma, PReLU slope), N(0, 0.001^2) biases
        PG, PD = LY.reference_init(LY.G_layout(C), rng), LY.reference_init(LY.D_layout(C), rng)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(PG=f(PG), PD=f(PD), real=f(rng.random((B // 2, C, 32, 32))),
                noise_D=f(rng.uniform(-1, 1, (B // 2, 100))), noise_G=f(rng.uniform(-1, 1, (B, 100))),
                masks_D=f(make_masks(B, rng)), masks_G=f(make_masks(B, rng)))


def fresh_state(case, dtype=np.float64):
    PD, PG = case["PD"].astype(dtype), case["PG"].astype(dtype)
    return dict(PD=PD, PG=PG, mD=np.zeros_like(PD), vD=np.zeros_like(PD), mG=np.zeros_like(PG), vG=np.zeros_like(PG),
                tD=0, tG=0, bnG=np.concatenate([np.zeros(256), np.ones(256), np.zeros(128), np.ones(128)]).astype(dtype))


def oracle_iteration(case, B, C, hyper=None, state=None):
    st = state or fresh_state(case)
    res = O.f64.train_iteration(B, C, hyper or HYPER, case["real"], case["noise_D"], case["noise_G"], case["masks_D"],
                                case["masks_G"], st)
    res["state"] = st
    return res


# ---- strict gradient parity across PReLU kinks (replaces seed-shopping) -------------------------------------------
# PReLU's derivative jumps at 0.  Among ~1e6 pre-activations a handful lie within fp32 rounding noise of 0 and two
# correct implementations may take different branches there; the batch-summed gradients then differ at 1e-3..1e-2.
# Instead of retrying seeds, the oracle lists the AMBIGUOUS elements (|x| < margin*max|x| per layer, decided from
# oracle data only), the test reads the branch the CUDA path took for exactly those elements, and the oracle's
# backward is re-run with those branches forced (oracle.kink).  Every other element keeps the oracle's own branch,
# so a wrong x<=0 branch, a wrong slope gradient or a wrong mask shows up at the strict 1e-4 bar.  The tests also
# assert that the ambiguous set is tiny (<= KINK_MAX_FRAC of a layer) and that the CUDA pre-activations of those
# elements are indeed ~0 (which also proves the NCHW->NHWC index mapping).
KINK_MARGIN = 2e-5      # single-net passes: the tensor-core path is within ~5e-6 of the oracle (normwise)
KINK_MAX_FRAC = 2e-3


def nchw_to_nhwc_index(idx, Cc, H, W):
    idx = np.asarray(idx, np.int64)
    b, r = np.divmod(idx, Cc * H * W)
    ch, r = np.divmod(r, H * W)
    y, x = np.divmod(r, W)
    return ((b * H + y) * W + x) * Cc + ch


def bn_preact_gpu(z_nhwc, mean, istd, gamma, beta):
    """BN output exactly as bn_prelu_apply_kernel / the BN backward kernels compute its sign:
    u = fma(gamma, fl32(fl32(z - mean) * istd), beta)  (k_elem.cu); evaluated for selected elements only."""
    t = ((z_nhwc.astype(np.float32) - mean.astype(np.float32)).astype(np.float32) * istd.astype(np.float32)).astype(np.float32)
    return gamma.astype(np.float64) * t.astype(np.float64) + beta.astype(np.float64)


def kink_overrides(calls, first_call, gpu_preacts, shapes, margin=KINK_MARGIN, label=""):
    """calls: oracle.kink.calls(); gpu_preacts[i]: callable(idx_nhwc) -> CUDA-path pre-activation values of layer i
    (flat NHWC indexing); shapes[i] = (C, H, W) of that layer.  Registers the overrides and returns the number of
    ambiguous elements."""
    from oracle import oracle as O
    total = 0
    for i, (get, (Cc, H, W)) in enumerate(zip(gpu_preacts, shapes)):
        n, mx, idx = calls[first_call + i]
        assert idx.size <= max(8, KINK_MAX_FRAC * n), "%s layer %d: %d of %d pre-activations within %.0e of 0" % (
            label, i, idx.size, n, margin)
        if idx.size == 0:
            O.kink.set_override(first_call + i, idx, np.zeros(0, np.int8))
            continue
        v = np.asarray(get(nchw_to_nhwc_index(idx, Cc, H, W)), np.float64)
        # the CUDA path's values of these elements must be ~0 as well (forward parity + index mapping)
        assert np.abs(v).max() <= 10 * margin * mx + 1e-30, "%s layer %d: CUDA pre-activation %.3e at an oracle zero" % (
            label, i, np.abs(v).max())
        O.kink.set_override(first_call + i, idx, (v > 0).astype(np.int8))
        total += idx.size
    return total


def oracle_gstep(PG, PD, noise_G, masks_G, B, C, hyper=None, bn_state=None, forward_only=False):
    """fevalG_on_D (adversarial.lua:187-231) composed from the fp64 oracle's nets: G fwd -> D fwd (train mode) ->
    BCE vs targets=1 -> D bwd (gradInput only) -> G bwd -> penalty (the :223 quirk: L1 gradient term scaled by G_L2)
    -> clamp.  Used with the CUDA path's own post-Adam D parameters, so that the G step is compared on identical
    inputs (after one Adam step a parameter whose gradient is rounding noise may have moved by +lr or -lr: the D
    parameters of two correct implementations differ by 2*lr in a few places, SURVEY.md 7.5)."""
    hp = hyper or HYPER
    g, d = O.f64.G(), O.f64.D()
    fake = g.forward(PG, noise_G, C, True, bn_state)
    out = d.forward(PD, fake, masks_G)
    t = np.ones(B)
    loss = O.f64.bce_fwd(out, t)
    if forward_only:
        return dict(lossG=loss, fake=fake, outD=out)
    _, dimg = d.backward(O.f64.bce_bwd(out, t), want_dP=False)
    gG = g.backward(dimg)
    loss += O.f64.penalty_clamp(np.asarray(PG, np.float64), gG, hp["G_L1"], hp["G_L2"], hp["G_L2"], hp["G_clamp"])
    return dict(lossG=loss, gradG=gG, fake=fake, outD=out)


def oracle_dstep(PD, real, fake, masks_D, B, C, hyper=None):
    """fevalD (adversarial.lua:83-179) + interruptableAdam at t=1 composed from the fp64 oracle's ops, given the
    fake half of the batch: D fwd -> BCE (first B/2 targets 1) -> D bwd -> penalty -> clamp -> Adam."""
    hp = hyper or HYPER
    d = O.f64.D()
    out = d.forward(PD, np.concatenate([real, fake]), masks_D)
    t = np.concatenate([np.ones(B // 2), np.zeros(B // 2)])
    loss = O.f64.bce_fwd(out, t)
    gD, _ = d.backward(O.f64.bce_bwd(out, t), want_dimg=False)
    P = np.array(PD, np.float64)
    loss += O.f64.penalty_clamp(P, gD, hp["D_L1"], hp["D_L1"], hp["D_L2"], hp["D_clamp"])
    m, v = np.zeros_like(P), np.zeros_like(P)
    O.f64.adam(P, gD, m, v, 1, hp["lr_D"], hp["beta1"], hp["beta2"], hp["eps"])
    return dict(lossD=loss, gradD=gD, mD=m, vD=v, PD=P, outD=out)
