"""Option bwd_merge: the weight and data gradients of G's upsampled 5x5 layers in one persistent launch
(bwd_pair_tc_kernel) compute every output tile with the arithmetic of the two separate launches, so a train step
gives the same bits with the option on and off."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _state(ctx):
    from face_generator_b200.lib import NET_D, NET_G
    mG, vG, tG = ctx.get_adam_state(NET_G)
    return {"params_G": ctx.get_params(NET_G), "grads_G": ctx.get_grads(NET_G), "adam_m_G": mG, "adam_v_G": vG,
            "adam_t_G": np.array([tG]), "bn_state_G": ctx.get_bn_state(), "params_D": ctx.get_params(NET_D),
            "grads_D": ctx.get_grads(NET_D)}


def _run(B, merge, use_graph, ctas=0, steps=3):
    """`steps` train steps with device-drawn dropout masks; returns the state they leave and the launches per step."""
    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_D, NET_G
    C = 3
    rng = np.random.default_rng(7)
    ctx = fg.Context(0, max_batch=B, channels=C)
    try:
        ctx.set_option("bwd_merge", merge)
        ctx.set_option("bwd_merge_ctas", ctas)
        ctx.set_option("use_graph", use_graph)
        assert (ctx.get_option("bwd_merge"), ctx.get_option("bwd_merge_ctas")) == (merge, ctas)
        ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
        ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
        f = lambda a: np.ascontiguousarray(a, np.float32)
        real = f(rng.random((B // 2, C, 32, 32)))
        nD, nG = f(rng.uniform(-1, 1, (B // 2, 100))), f(rng.uniform(-1, 1, (B, 100)))
        h = fg.hyper_default()
        launches = []
        for i in range(steps):
            l0 = ctx.launches()
            ctx.train_step(h, B, real, nD, nG, None, None, 40 + i)
            launches.append(ctx.launches() - l0)
        ctx.sync()
        return _state(ctx), launches
    finally:
        ctx.close()


def _assert_same(a, b):
    for k in a:
        assert a[k].shape == b[k].shape, k
        assert np.array_equal(a[k], b[k]), (k, int(np.sum(a[k] != b[k])), float(np.max(np.abs(a[k] - b[k]))))


@pytest.mark.parametrize("B", [256, 130])
def test_merged_backward_is_bitwise_the_two_launches(B):
    """Eager launches, 3 steps; batch 130 leaves a ragged batch tail in every pixel tiling.  The merged step issues
    one kernel less (G.C2's weight and data gradient in one launch)."""
    ref, l_ref = _run(B, 0, 0)
    got, l_got = _run(B, 1, 0)
    _assert_same(got, ref)
    assert l_got == [n - 1 for n in l_ref], (l_got, l_ref)


def test_merged_backward_bitwise_under_graph_replay():
    """The captured step replayed on consecutive steps: the claim counter is reset inside the graph."""
    ref, _ = _run(256, 0, 1)
    got, _ = _run(256, 1, 1)
    _assert_same(got, ref)


@pytest.mark.parametrize("B,ctas", [(256, 40), (130, 1)])
def test_merged_backward_with_fewer_ctas_than_weight_gradient_items(B, ctas):
    """Fewer CTAs than the 72 weight-gradient items: a CTA runs several items of both kinds back to back on one
    stage ring (1 CTA: every item of the layer).  bwd_merge = 2, as so few CTAs make the merged launch the slower one."""
    ref, _ = _run(B, 0, 1)
    got, _ = _run(B, 2, 1, ctas=ctas)
    _assert_same(got, ref)


@pytest.mark.parametrize("B", [256, 130])
def test_merging_g_c1_as_well_is_bitwise_the_two_launches(B):
    """bwd_merge = 2 also merges G.C1, which the default leaves on two launches at these batches (its 128 dgrad tiles
    of 144 K blocks pack no better around the 72 weight-gradient items of 256)."""
    ref, l_ref = _run(B, 0, 0)
    got, l_got = _run(B, 2, 0)
    _assert_same(got, ref)
    assert l_got == [n - 2 for n in l_ref], (l_got, l_ref)


def test_bwd_merge_option_range():
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=8, channels=3)
    try:
        assert ctx.get_option("bwd_merge") == 1 and ctx.get_option("bwd_merge_ctas") == 0
        for key, bad in (("bwd_merge", 3), ("bwd_merge", -1), ("bwd_merge_ctas", -1)):
            with pytest.raises(Exception):
                ctx.set_option(key, bad)
    finally:
        ctx.close()
