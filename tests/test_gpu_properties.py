"""Size-independent properties at BASELINE.json's full size (B=256 colour), where the oracle is too slow."""
import numpy as np
import pytest

import parity_utils as PU

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def big():
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    B, C = 256, 3
    case = PU.make_case(B, C, seed=1001)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_params(NET_G, case["PG"])
    ctx.set_params(NET_D, case["PD"])
    yield fg, ctx, case, B, C
    ctx.close()


def test_bn_output_statistics_and_range(big):
    fg, ctx, case, B, C = big
    out = ctx.G_forward(case["noise_G"])
    assert out.shape == (B, C, 32, 32) and np.isfinite(out).all() and out.min() >= 0 and out.max() <= 1
    # (z - mean) * istd has zero mean / unit variance per channel over (N,H,W)
    for name, Cc, m, s in (("z1", 256, "G.bn_mean1", "G.bn_istd1"), ("z2", 128, "G.bn_mean2", "G.bn_istd2")):
        z = ctx.debug_tensor("G." + name).reshape(-1, Cc).astype(np.float64)
        xh = (z - ctx.debug_tensor(m)) * ctx.debug_tensor(s)
        assert np.abs(xh.mean(0)).max() < 1e-4
        assert np.abs(xh.var(0) - 1).max() < 2e-3  # eps=1e-5 inside the sqrt


def test_batch_independence_of_D(big):
    """D has no cross-sample coupling: row i of D(x) only depends on x[i] (and its masks)."""
    fg, ctx, case, B, C = big
    rng = np.random.default_rng(5)
    x = rng.random((B, C, 32, 32)).astype(np.float32)
    full = ctx.D_forward(x, masks=case["masks_D"])
    part = ctx.D_forward(x[64:128], masks=case["masks_D"][64:128])
    np.testing.assert_allclose(part, full[64:128], rtol=2e-5, atol=1e-6)


def test_full_size_step_first_adam_update_is_lr(big):
    fg, ctx, case, B, C = big
    from face_generator_b200.lib import NET_D, NET_G
    P0D, P0G = ctx.get_params(NET_D), ctx.get_params(NET_G)
    st = ctx.train_step(fg.hyper_default(), B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"],
                        case["masks_G"])
    assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"]) and sum(st["conf"]) == B
    for net, P0 in ((NET_D, P0D), (NET_G, P0G)):
        P1, g = ctx.get_params(net), ctx.get_grads(net)
        assert np.isfinite(P1).all() and np.isfinite(g).all()
        big_g = np.abs(g) > 1e-4  # eps/(sqrt(1-b2)|g|) < 0.4% there
        # interruptable_optimizers.lua:78-90 at t=1: |dx| = lr*|g|/(|g|+eps*sqrt(1-b2)...) ~= lr
        np.testing.assert_allclose(np.abs(P1 - P0)[big_g], 1e-3, rtol=2e-2)
        assert np.all(np.sign(P0 - P1)[big_g] == np.sign(g)[big_g])
    assert np.abs(ctx.get_grads(NET_D)).max() <= 1.0 + 1e-6 and np.abs(ctx.get_grads(NET_G)).max() <= 5.0 + 1e-6


def test_step_is_deterministic_given_masks(big):
    fg, ctx, case, B, C = big
    from face_generator_b200.lib import NET_D, NET_G
    outs = []
    for _ in range(2):
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        ctx.set_adam_state(NET_G, np.zeros(ctx.nG), np.zeros(ctx.nG), 0)
        ctx.set_adam_state(NET_D, np.zeros(ctx.nD), np.zeros(ctx.nD), 0)
        st = ctx.train_step(fg.hyper_default(), B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"],
                            case["masks_G"])
        outs.append((st["loss_D"], st["loss_G"], ctx.get_grads(NET_G), ctx.get_grads(NET_D), ctx.get_params(NET_G),
                     ctx.get_params(NET_D)))
    # every cross-block sum is added in a fixed order (no float atomics), so the same step is bit-identical
    assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1]
    for a, b in zip(outs[0][2:], outs[1][2:]):
        np.testing.assert_array_equal(a, b)


def test_in_kernel_dropout_rates(big):
    fg, ctx, case, B, C = big
    x = np.random.default_rng(6).random((B, C, 32, 32)).astype(np.float32)
    ctx.D_forward(x, masks=None, seed=1234)
    m = ctx.debug_tensor("D.masks").reshape(B, -1)
    assert abs(m[:, :960].mean() - 0.8) < 0.01 and abs(m[:, 960:].mean() - 0.5) < 0.01
    assert set(np.unique(m)) <= {0.0, 1.0}


@pytest.mark.parametrize("opt,val", [("mma_f16", 0), ("use_graph", 0), ("bn_epilogue", 0), ("edge_impl", 0)])
def test_alternative_code_paths_agree_with_the_default(opt, val):
    """Every option selects another implementation of the same arithmetic: three steps at batch 64 with device-drawn
    dropout masks (the same seeds) give the default path's losses and confusion counts.  mma_f16 = 0 is the 3xTF32
    operand split instead of 3xFP16, use_graph = 0 eager launches instead of the captured step, bn_epilogue = 0 the
    separate BatchNorm statistics pass, edge_impl = 0 the round-1 kernels of the 3-channel-side convolutions."""
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    B, C = 64, 3
    case = PU.make_case(B, C, seed=2024)
    res = []
    for setting in (None, (opt, val)):
        ctx = fg.Context(0, max_batch=B, channels=C)
        if setting:
            ctx.set_option(*setting)
            assert ctx.get_option(opt) == val
        ctx.set_params(NET_G, case["PG"])
        ctx.set_params(NET_D, case["PD"])
        h = fg.hyper_default()
        sts = [ctx.train_step(h, B, case["real"], case["noise_D"], case["noise_G"], None, None, 100 + i) for i in range(3)]
        res.append((sts, ctx.get_params(NET_G)))
        ctx.close()
    for a, b in zip(res[0][0], res[1][0]):
        assert list(a["conf"]) == list(b["conf"]) and a["t_D"] == b["t_D"] and a["t_G"] == b["t_G"]
        assert abs(a["loss_D"] - b["loss_D"]) < 2e-4 * max(1.0, abs(a["loss_D"]))
        assert abs(a["loss_G"] - b["loss_G"]) < 2e-3 * max(1.0, abs(a["loss_G"]))  # behind Adam's +-lr amplification
    # parameters after three Adam steps: a PReLU pre-activation within rounding noise of 0 may take the other branch under
    # another operand rounding (section 5 of DESIGN.md), which moves G's gradient by ~1e-2 relative and an Adam update
    # by ~1e-5; noise-level gradients flip whole +-lr steps.  Bound: a few lr at most, and almost everything within 1e-4.
    # (measured for mma_f16 = 0 vs 1: max 1.0e-3, 18 % of the elements beyond 1e-5; a wrong code path moves every
    # element by ~lr per step and shows in the losses above first)
    d = np.abs(res[0][1].astype(np.float64) - res[1][1])
    assert d.max() <= 3 * 2e-3 + 1e-6 and d.mean() < 5e-4, (d.max(), d.mean())
