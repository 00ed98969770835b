"""The --scale 16 nets (models.lua:27-51 create_G_decoder_upsampling16, :279-316 create_D16_d) and the adversarial.lua
loop on them, plus cudnn.SpatialConvolutionUpsample with factor != 1 (layers/cudnnSpatialConvolutionUpsample.lua).

CPU: the C ABI reports the oracle's parameter counts.
GPU (-m gpu): fg_s16_* / fg_scu_* through the C ABI against the fp64 oracle on the same seeded inputs, both conv
implementations (0 = fp32 FFMA kernels, 2 = wgmma 3-term split).  Tolerance 1e-4 relative (BASELINE.json north_star).
Gradients are compared strictly on the "smooth" (PReLU slopes 1) and "near" (slopes 1 - k*1e-3, see s16_utils) inits;
the "trained" init (slopes 0.25) holds the forward values to 1e-4 and the gradients to the kink bar."""
import numpy as np
import pytest

import parity_utils as PU
import s16_utils as SU
from oracle import oracle as O
from oracle import oracle_s16 as OS

TOL = 1e-4
KINK_TOL = 2e-2


def _layer_errs(got, ref, layout):
    """per-tensor relative errors.  A convolution bias in front of a training-mode BatchNorm (G's C1b, C2b) has an
    exactly-zero gradient: both sides hold rounding noise there, which is compared with the scale of all gradients."""
    out = {}
    scale = np.abs(ref).max()
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        if k in ("C1b", "C2b"):
            out[k] = max(np.abs(got[o:o + n]).max(), np.abs(ref[o:o + n]).max()) / scale
        else:
            out[k] = PU.relerr(got[o:o + n], ref[o:o + n])
    return out


# ------------------------------------------------------------------------------------------ CPU
def test_s16_param_counts_match_oracle():
    from face_generator_b200.lib import load_library, S16_MASK_PER_SAMPLE
    lib = load_library()
    for C in (1, 3):
        assert lib.fg_s16_param_count(0, C) == OS.G_param_count(C)
        assert lib.fg_s16_param_count(1, C) == OS.D_param_count(C)
    assert lib.fg_s16_mask_per_sample() == OS.MASK_PER_SAMPLE == S16_MASK_PER_SAMPLE


def test_oracle_reproduces_s16_golden():
    """the committed vectors (tests/golden/make_golden_s16.py) pin the oracle's --scale 16 iteration"""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s16_train_color_b8.npz"), allow_pickle=False)
    B, C = int(g["B"]), int(g["C"])
    case = SU.make_case(B, C, seed=int(g["seed"]), init=str(g["init"]))
    assert abs(sum(np.abs(case[k]).sum() for k in sorted(case)) - float(g["input_checksum"])) < 1e-5
    res = SU.oracle_iteration(case, B, C)
    assert abs(res["lossD"] - float(g["lossD"])) < 1e-10 and abs(res["lossG"] - float(g["lossG"])) < 1e-10
    np.testing.assert_array_equal(res["conf"], g["conf"])
    assert PU.relerr(res["gradD"][::1009], g["gradD"]) < 1e-9 and PU.relerr(res["gradG"][::1009], g["gradG"]) < 1e-9
    assert PU.relerr(res["PD"][::1009], g["PD"]) < 1e-12 and PU.relerr(res["bn"], g["bn"]) < 1e-12


# ------------------------------------------------------------------------------------------ GPU
def _ctx(B, C, impl):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_option("conv_impl", impl)
    return ctx, fg.S16(ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 1])
@pytest.mark.parametrize("impl", [0, 2])
@pytest.mark.parametrize("init", ["near", "trained"])
def test_gpu_s16_G_forward_backward(C, impl, init):
    from face_generator_b200.lib import NET_G
    B = 6
    case = SU.make_case(2 * B, C, seed=900 + C, init=init)
    rng = np.random.default_rng(11)
    noise = case["noise_G"][:B]
    dout = rng.standard_normal((B, C, 16, 16)).astype(np.float32)
    g = OS.f64.G()
    bn = SU.bn_init()
    ref_img = g.forward(case["PG"], noise, C, bn)
    ref_dP = g.backward(dout)
    ctx, net = _ctx(2 * B, C, impl)
    net.set_params(NET_G, case["PG"])
    img = net.G_forward(noise, training=True)
    assert PU.relerr(img, ref_img) < TOL
    assert PU.relerr(net.get_bn_state(), bn) < TOL  # running statistics after one training-mode forward
    net.zero_grads(NET_G)
    net.G_backward(dout)
    errs = _layer_errs(net.get_grads(NET_G), ref_dP, OS.G_layout(C))
    assert max(errs.values()) < (TOL if init == "near" else KINK_TOL), errs
    # evaluate(): running statistics instead of batch statistics
    net.set_bn_state(bn)
    ev = net.G_forward(noise, training=False)
    ref_ev = _G_eval_reference(case["PG"], noise, C, bn)
    assert PU.relerr(ev, ref_ev) < TOL


def _G_eval_reference(P, noise, C, bn):
    """G16 in evaluate() mode from the oracle's layer ops: BatchNorm uses running_mean / running_var (eps 1e-5)."""
    t, s = O.f64, OS.f64
    L = OS.G_layout(C)
    p = {k: np.asarray(P[o:o + int(np.prod(sh))], np.float64).reshape(sh) for k, (o, sh) in L.items()}
    B = noise.shape[0]
    h = t.prelu_fwd(t.linear_fwd(noise, p["L1W"], p["L1b"]).reshape(B, 128, 4, 4), float(p["a1"][0]))

    def bn_eval(x, gm, be, rm, rv):
        return (x - rm[None, :, None, None]) / np.sqrt(rv[None, :, None, None] + 1e-5) * gm[None, :, None, None] + be[None, :, None, None]
    h = t.conv_fwd(t.up2_fwd(h), p["C1W"], p["C1b"])
    h = t.prelu_fwd(bn_eval(h, p["g1"], p["be1"], bn[0:256], bn[256:512]), float(p["a2"][0]))
    h = t.conv_fwd(t.up2_fwd(h), p["C2W"], p["C2b"])
    h = t.prelu_fwd(bn_eval(h, p["g2"], p["be2"], bn[512:640], bn[640:768]), float(p["a3"][0]))
    z = t.conv_fwd(h, p["C3W"], p["C3b"])
    return 1.0 / (1.0 + np.exp(-z))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 1])
@pytest.mark.parametrize("impl", [0, 2])
@pytest.mark.parametrize("init", ["near", "trained"])
def test_gpu_s16_D_forward_backward(C, impl, init):
    from face_generator_b200.lib import NET_D
    B = 6
    case = SU.make_case(2 * B, C, seed=950 + C, init=init)
    rng = np.random.default_rng(12)
    img = rng.random((B, C, 16, 16)).astype(np.float32)
    masks = case["masks_D"][:B]
    dout = rng.standard_normal(B).astype(np.float32)
    d = OS.f64.D()
    ref_out = d.forward(case["PD"], img, masks, True)
    ref_dP, ref_dimg = d.backward(dout)
    ctx, net = _ctx(2 * B, C, impl)
    net.set_params(NET_D, case["PD"])
    out = net.D_forward(img, masks, training=True)
    assert PU.relerr(out, ref_out) < TOL
    net.zero_grads(NET_D)
    dimg = net.D_backward(dout, want_wgrad=True, want_dimg=True)
    gtol = TOL if init == "near" else KINK_TOL
    errs = _layer_errs(net.get_grads(NET_D), ref_dP, OS.D_layout(C))
    assert max(errs.values()) < gtol, errs
    assert PU.relerr(dimg, ref_dimg) < gtol  # ConcatTable backward: conv branch + dense branch
    # evaluate(): SpatialDropout scales by 1-p, Dropout is the identity
    ev = net.D_forward(img, None, training=False)
    assert PU.relerr(ev, d.forward(case["PD"], img, None, False)) < TOL
    # the G step discards D's weight gradients: want_wgrad=0 must leave them untouched
    net.zero_grads(NET_D)
    net.D_forward(img, masks, training=True)
    net.D_backward(dout, want_wgrad=False, want_dimg=True)
    assert not net.get_grads(NET_D).any()


@pytest.mark.gpu
@pytest.mark.parametrize("C,B", [(3, 8), (1, 12)])
@pytest.mark.parametrize("impl", [0, 1, 2])
def test_gpu_s16_train_step_matches_oracle(C, B, impl):
    """fg_s16_train_step == the adversarial.lua iteration composed from the fp64 oracle: losses, confusion counts,
    both clamped gradients (recovered from Adam's first moment: m = (1-beta1) g at t = 1), parameters, BN state."""
    from face_generator_b200.lib import NET_D, NET_G, hyper_default
    case = SU.make_case(B, C, seed=1000 + C, init="near")
    ref = SU.oracle_iteration(case, B, C)
    ctx, net = _ctx(B, C, impl)
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    h = hyper_default()
    st = net.train_step(h, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
    assert abs(st["loss_D"] - ref["lossD"]) < TOL * max(1.0, abs(ref["lossD"]))
    assert abs(st["loss_G"] - ref["lossG"]) < 2e-3 * max(1.0, abs(ref["lossG"]))  # G step runs on D after an Adam step (+-lr flips)
    assert list(st["conf"]) == [int(v) for v in ref["conf"]]
    assert st["trained_D"] == 1 and st["t_D"] == 1 and st["t_G"] == 1
    mD, vD, tD = net.get_adam_state(NET_D)
    assert tD == 1
    errs = _layer_errs(mD / (1.0 - h.beta1), ref["gradD"], OS.D_layout(C))
    assert max(errs.values()) < TOL, errs
    mG, vG, tG = net.get_adam_state(NET_G)
    errs = _layer_errs(mG / (1.0 - h.beta1), ref["gradG"], OS.G_layout(C))
    assert max(errs.values()) < 5e-3, errs  # through D's post-Adam parameters, see above
    # Adam at t=1 moves every parameter by ~lr*sign(g): compare the updates where the gradient is not rounding noise
    for netid, key, g in ((NET_D, "PD", ref["gradD"]), (NET_G, "PG", ref["gradG"])):
        P0, P1, R1 = case[key].astype(np.float64), net.get_params(netid).astype(np.float64), ref[key]
        big = np.abs(g) > 1e-3 * np.abs(g).max()
        assert np.abs((P1 - P0)[big] - (R1 - P0)[big]).max() < 2e-5, key  # lr = 1e-3
    assert PU.relerr(net.get_bn_state(), ref["bn"]) < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [0, 2])
def test_gpu_s16_train_step_matches_golden(impl):
    """the same step against the committed golden vectors (no oracle run on the GPU box)"""
    import os
    from face_generator_b200.lib import NET_D, NET_G, hyper_default
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s16_train_color_b8.npz"), allow_pickle=False)
    B, C = int(g["B"]), int(g["C"])
    case = SU.make_case(B, C, seed=int(g["seed"]), init=str(g["init"]))
    ctx, net = _ctx(B, C, impl)
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    h = hyper_default()
    st = net.train_step(h, B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
    assert abs(st["loss_D"] - float(g["lossD"])) < TOL * max(1.0, abs(float(g["lossD"])))
    assert abs(st["loss_G"] - float(g["lossG"])) < 2e-3 * max(1.0, abs(float(g["lossG"])))
    assert list(st["conf"]) == [int(v) for v in g["conf"]]
    mD, _, _ = net.get_adam_state(NET_D)
    assert np.abs(mD[::1009] / (1.0 - h.beta1) - g["gradD"]).max() < TOL * float(g["gradD_absmax"])
    mG, _, _ = net.get_adam_state(NET_G)
    assert np.abs(mG[::1009] / (1.0 - h.beta1) - g["gradG"]).max() < 5e-3 * float(g["gradG_absmax"])
    assert PU.relerr(net.get_bn_state(), g["bn"]) < 1e-3


@pytest.mark.gpu
def test_gpu_s16_accuracy_gate_and_generated_masks():
    """D_maxAcc below the running accuracy closes the gate: the D update is skipped (adversarial.lua:156-178,
    interruptable_optimizers.lua:64-66) while G keeps training; masks drawn on the device when none are given."""
    from face_generator_b200.lib import NET_D, NET_G, hyper_default
    B, C = 8, 3
    case = SU.make_case(B, C, seed=1100, init="trained")
    ctx, net = _ctx(B, C, 2)
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    h = hyper_default()
    h.D_maxAcc, h.accs_interval = 0.0, 1  # any accuracy >= 0 closes the gate
    p0 = net.get_params(NET_D)
    g0 = net.get_params(NET_G)
    st = net.train_step(h, B, case["real"], case["noise_D"], case["noise_G"], None, None, seed=5)
    assert st["trained_D"] == 0 and st["t_D"] == 0 and st["t_G"] == 1
    np.testing.assert_array_equal(net.get_params(NET_D), p0)
    assert np.abs(net.get_params(NET_G) - g0).max() > 0
    h.D_maxAcc = 1.01
    st = net.train_step(h, B, case["real"], case["noise_D"], case["noise_G"], None, None, seed=6)
    assert st["trained_D"] == 1 and st["t_D"] == 1 and st["t_G"] == 2
    assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])


@pytest.mark.gpu
def test_gpu_s16_batch_256_runs_on_the_tensor_cores():
    """BASELINE batch size: finite losses, and the two stride-2 layers / Linear layers take the tensor-core path
    (their timers are only attached to tensor-core launches' names, so compare impl 0 vs 2 outputs instead)."""
    from face_generator_b200.lib import NET_D, NET_G, hyper_default
    B, C = 256, 3
    case = SU.make_case(B, C, seed=1200, init="trained")
    outs = []
    for impl in (0, 2):
        ctx, net = _ctx(B, C, impl)
        net.set_params(NET_G, case["PG"])
        net.set_params(NET_D, case["PD"])
        img = net.G_forward(case["noise_G"], training=True)
        outs.append((img, net.D_forward(img, case["masks_G"], training=True)))
        st = net.train_step(hyper_default(), B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"]) and sum(st["conf"]) == B
        net.close()
        ctx.close()
    assert PU.relerr(outs[1][0], outs[0][0]) < TOL and PU.relerr(outs[1][1], outs[0][1]) < TOL


@pytest.mark.gpu
def test_gpu_s16_epoch_loop():
    """adversarial.train (the adversarial.lua:29-334 epoch loop) drives the 16x16 nets through the same call"""
    from face_generator_b200 import adversarial
    from face_generator_b200.lib import NET_D, NET_G, hyper_default
    B, C = 8, 3
    case = SU.make_case(B, C, seed=1300, init="trained")
    ctx, net = _ctx(B, C, 2)
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    data = np.random.default_rng(3).random((40, C, 16, 16)).astype(np.float32)
    acc, conf, trained = adversarial.train(net, data, hyper_default(), B, n_epoch=16, epoch=1)
    batches = adversarial.epoch_batches(16, B)  # the tail batch shrinks (adversarial.lua:56)
    nb = len(batches)
    assert conf.sum() == sum(b for _, b in batches) and trained == nb and 0.0 <= acc <= 1.0
    assert net.get_adam_state(NET_G)[2] == nb


# ------------------------------------------------------------------------------------------ SCU factor != 1
@pytest.mark.gpu
@pytest.mark.parametrize("impl", [0, 2])
@pytest.mark.parametrize("Cin,nOut,k,factor,H", [(64, 32, 3, 2, 8), (3, 8, 5, 2, 8), (64, 16, 3, 3, 4)])
def test_gpu_scu_factor_is_a_raw_view_of_the_wide_convolution(impl, Cin, nOut, k, factor, H):
    """cudnnSpatialConvolutionUpsample.lua:14-15 builds a convolution to nOut*f*f planes; :18-30 re-VIEWS its contiguous
    output as [N][nOut][H*f][W*f]; :32-58 view gradOutput back.  Checked against the oracle's convolution with the
    views applied in numpy (reshape of a contiguous array == torch's :view)."""
    import face_generator_b200 as fg
    from face_generator_b200.lib import _ptr
    N = 4
    rng = np.random.default_rng(70 + factor + k)
    planes = nOut * factor * factor
    x = rng.standard_normal((N, Cin, H, H)).astype(np.float32)
    w = (rng.standard_normal((planes, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(planes).astype(np.float32)
    ctx = fg.Context(0, max_batch=N, channels=3)
    ctx.set_option("conv_impl", impl)
    lib, h = ctx.lib, ctx.h
    y = np.empty((N, nOut, H * factor, H * factor), np.float32)  # the module's output shape
    assert lib.fg_scu_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, H, H, nOut, k, factor) == 0, lib.fg_last_error()
    ref = O.f64.conv_fwd(x, w, b).reshape(N, nOut, H * factor, H * factor)
    assert PU.relerr(y, ref) < TOL
    dy = rng.standard_normal(y.shape).astype(np.float32)  # gradOutput arrives in the upsampled shape
    dx = np.empty_like(x)
    assert lib.fg_scu_backward_data(h, _ptr(dy), _ptr(w), _ptr(dx), N, Cin, H, H, nOut, k, factor) == 0, lib.fg_last_error()
    dw, db = np.zeros_like(w), np.zeros_like(b)
    assert lib.fg_scu_backward_filter(h, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), N, Cin, H, H, nOut, k, factor) == 0, lib.fg_last_error()
    rdx, rdw, rdb = O.f64.conv_bwd(x, w, dy.reshape(N, planes, H, H))
    assert PU.relerr(dx, rdx) < TOL and PU.relerr(dw, rdw) < TOL and PU.relerr(db, rdb) < TOL
    assert lib.fg_scu_forward(h, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, H, H, nOut, k, 0) != 0  # factor < 1 is rejected
