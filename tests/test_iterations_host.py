"""CPU: the host side of --D_iterations / --G_iterations (train.lua:33-34, train_c2f.lua:31-32): what the epoch loop
feeds a multi-iteration call, the range check, and that the Lua shims read both flags."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _RecordingCtx:
    """stands in for face_generator_b200.Context: records what train() feeds each fused call"""

    def __init__(self):
        self.calls = []

    def train_step(self, hyper, B, real, noise_D, noise_G, masks_D, masks_G, seed):
        self.calls.append(("single", B, 1, 1, real.copy(), noise_D.copy(), noise_G.copy(), seed))
        return dict(conf=[B // 2, 0, 0, B // 2], trained_D=1)

    def train_step_iters(self, hyper, B, d, g, real, noise_D, noise_G, masks_D, masks_G, seed):
        self.calls.append(("iters", B, d, g, real.copy(), noise_D.copy(), noise_G.copy(), seed))
        return dict(conf=[d * B // 2, 0, 0, d * B // 2], trained_D=d)


def _data():
    # every image is constant and carries its index, so a real half-batch names the images it drew
    return np.arange(256, dtype=np.float32).reshape(256, 1, 1, 1) * np.ones((1, 1, 32, 32), np.float32)


def test_train_feeds_every_iteration_its_own_draws():
    from face_generator_b200 import adversarial as A
    ctx = _RecordingCtx()
    acc, conf, trained = A.train(ctx, _data(), None, 16, n_epoch=64, D_iterations=2, G_iterations=3)
    assert ctx.calls and all(c[0] == "iters" for c in ctx.calls)
    for kind, B, d, g, real, nD, nG, seed in ctx.calls:
        assert (d, g) == (2, 3)
        assert real.shape == (2, B // 2, 1, 32, 32) and nD.shape == (2, B // 2, 100) and nG.shape == (3, B, 100)
        assert not np.array_equal(real[0], real[1])                      # two real half-batches
        noises = [nD[0], nD[1], nG[0], nG[1], nG[2]]                     # 2 + 3 distinct noise tensors
        for i in range(len(noises)):
            for j in range(i):
                assert not np.array_equal(noises[i].ravel()[:100], noises[j].ravel()[:100])
    assert trained == 2 * len(ctx.calls)
    assert conf.sum() == sum(2 * c[1] for c in ctx.calls)


def test_train_with_one_iteration_each_keeps_the_single_iteration_call():
    """D_iterations = G_iterations = 1 is the existing fg_train_step path, draw for draw"""
    from face_generator_b200 import adversarial as A
    a, b = _RecordingCtx(), _RecordingCtx()
    A.train(a, _data(), None, 16, n_epoch=64)
    A.train(b, _data(), None, 16, n_epoch=64, D_iterations=1, G_iterations=1)
    assert len(a.calls) == len(b.calls) and all(c[0] == "single" for c in b.calls)
    for x, y in zip(a.calls, b.calls):
        for u, v in zip(x[4:7], y[4:7]):
            np.testing.assert_array_equal(u, v)


def test_single_iteration_draws_are_the_first_iteration_draws():
    """the host draws in the reference's order: (real, noise) per D iteration, then the G noise -- so iteration 0 of
    a (d, g) call sees exactly what a (1, 1) call would have seen"""
    from face_generator_b200 import adversarial as A
    a, b = _RecordingCtx(), _RecordingCtx()
    A.train(a, _data(), None, 16, n_epoch=16)
    A.train(b, _data(), None, 16, n_epoch=16, D_iterations=2, G_iterations=1)
    np.testing.assert_array_equal(a.calls[0][4], b.calls[0][4][0])
    np.testing.assert_array_equal(a.calls[0][5], b.calls[0][5][0])


@pytest.mark.parametrize("d,g", [(0, 1), (1, 0), (17, 1), (1, 17), (-1, 2), (1.5, 1)])
def test_out_of_range_counts_raise_before_any_call(d, g):
    from face_generator_b200 import adversarial as A
    from face_generator_b200.lib import check_iters
    ctx = _RecordingCtx()
    with pytest.raises(ValueError):
        A.train(ctx, _data(), None, 16, n_epoch=64, D_iterations=d, G_iterations=g)
    assert ctx.calls == []
    with pytest.raises(ValueError):
        check_iters(d, g)


def test_iteration_root_formula():
    from face_generator_b200.lib import iteration_root
    assert iteration_root(5, 0) == 5
    assert iteration_root(5, 3) == (1 << 60) | (5 << 8) | 3
    assert iteration_root(2 ** 64 - 1, 1) < 2 ** 64
    assert len({iteration_root(s, j) for s in range(64) for j in range(16)}) == 64 * 16


@pytest.mark.parametrize("shim,entry", [("adversarial_b200.lua", ("fg_train_step_iters", "fg_s16_train_step_iters")),
                                        ("adversarial_c2f_b200.lua", ("fg_c2f_train_step_iters",))])
def test_lua_shims_read_the_iteration_flags(shim, entry):
    src = open(os.path.join(ROOT, "face_generator_b200", "lua", shim)).read()
    assert "OPT.D_iterations" in src and "OPT.G_iterations" in src
    called = set(re.findall(r"C\.(fg_[a-zA-Z0-9_]+)", src))
    assert set(entry) <= called
