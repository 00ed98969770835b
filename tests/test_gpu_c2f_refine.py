"""The coarse-to-fine refinement on the GPU: fg_image_scale, fg_c2f_refine (sample.lua:176-214) and sample_pyramid.

 * fg_image_scale against oracle_data.scale within 1e-6: shrink, enlarge, 1-pixel sources, non-square, C = 1 and 3.
 * fg_c2f_refine against the float64 restatement (c2f_refine_ref.py) at S = 32 and 64, C = 3 and 1, N = 13 (ragged
   against the chunk), 10 tries, evaluate() and training with explicit masks.  The pick must be the oracle's wherever
   its best two predictions are more than 2e-5 apart (decided from oracle data only, like the PReLU-kink rules).
 * Bitwise: refine equals the composed path (fg_image_scale, G and D forwards, numpy pick, add); the default streams are
   fg_noise_uniform(2*seed) / fg_dropout_mask(2*seed+1); chunk 1, 7 and max_batch/tries, host and device buffers and a
   repeated seed give the same bits.  Edges, argument errors with nothing launched, the pyramid, checkpoints.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import c2f_refine_ref as RR  # noqa: E402
from face_generator_b200 import layouts as LY  # noqa: E402
from oracle import oracle_data as OD  # noqa: E402

pytestmark = pytest.mark.gpu

MAXB, T = 40, 10  # chunk = max_batch / tries = 4 images: N = 13 runs 4 + 4 + 4 + 1


def _ctx(C=3, maxB=MAXB, f16=1):
    import face_generator_b200 as fg
    ctx = fg.Context(0, max_batch=maxB, channels=C)
    ctx.set_option("mma_f16", f16)
    return ctx


def _net(ctx, S, seed=1):
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    rng = np.random.default_rng(seed + S)
    net = fg.C2f(ctx, S)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(ctx.C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(ctx.C, S), rng, 1.0))
    return net


def _inputs(net, N, in_size, seed=3, tries=T):
    rng = np.random.default_rng(seed)
    S = net.S
    images = rng.random((N, net.C, in_size, in_size)).astype(np.float32)
    noise = rng.uniform(-1, 1, (N * tries, 1, S, S)).astype(np.float32)
    masks = (rng.random((N * tries, net.mask_per_sample)) < 0.5).astype(np.float32)
    return images, noise, masks


def _composed(ctx, net, images, noise, masks, training, tries, rows):
    """fg_image_scale -> replicate -> fg_c2f_G_forward + fg_c2f_D_forward (`rows` rows per call) -> numpy pick -> add"""
    from face_generator_b200.pyramid import image_scale
    N, S = images.shape[0], net.S
    up = image_scale(ctx, images, S)
    cond = np.ascontiguousarray(np.repeat(up, tries, axis=0))
    diff = np.empty_like(cond)
    pred = np.empty(N * tries, np.float32)
    for r in range(0, N * tries, rows):
        e = min(r + rows, N * tries)
        diff[r:e] = net.G_forward(noise[r:e], cond[r:e])
        pred[r:e] = net.D_forward(diff[r:e], cond[r:e], masks[r:e] if training else None, training=bool(training))
    pred = pred.reshape(N, tries)
    pick = RR.pick_rule(pred)
    out = up + diff.reshape(N, tries, net.C, S, S)[np.arange(N), pick]
    return out, pick, pred, up, diff


def _same(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


# ============================================================================================ fg_image_scale
SCALE_CASES = [(3, 64, 64, 32, 32), (1, 64, 64, 16, 16), (3, 16, 16, 64, 64), (1, 32, 32, 64, 64), (3, 1, 1, 5, 7),
               (1, 1, 9, 4, 2), (3, 48, 20, 17, 33), (1, 7, 30, 30, 7), (3, 64, 64, 1, 1), (3, 31, 31, 31, 31)]


@pytest.mark.parametrize("C,Hs,Ws,Ho,Wo", SCALE_CASES)
def test_image_scale_matches_oracle(C, Hs, Ws, Ho, Wo):
    from face_generator_b200.lib import _check, _ptr
    ctx = _ctx(3, 8)
    x = np.random.default_rng(Hs * Ws + Ho).random((5, C, Hs, Ws)).astype(np.float32)
    out = np.empty((5, C, Ho, Wo), np.float32)
    _check(ctx.lib.fg_image_scale(ctx.h, _ptr(x), 5, C, Hs, Ws, Ho, Wo, _ptr(out)), "fg_image_scale")
    np.testing.assert_allclose(out, OD.scale(x.astype(np.float64), Wo, Ho), rtol=0, atol=1e-6)
    # device buffers give the same bits
    xd, od = ctx.dev_array(x), ctx.dev_array(np.zeros_like(out))
    _check(ctx.lib.fg_image_scale(ctx.h, xd, 5, C, Hs, Ws, Ho, Wo, od), "fg_image_scale")
    back = np.empty_like(out)
    _check(ctx.lib.fg_memcpy(ctx.h, _ptr(back), od, back.nbytes), "fg_memcpy")
    np.testing.assert_array_equal(back, out)
    ctx.dev_free(xd)
    ctx.dev_free(od)
    ctx.close()


# ============================================================================================ numerics vs fp64
NUM_PARAMS = [(S, C, tr) for S in (32, 64) for C in (3, 1) for tr in (0, 1)]
_G_ORACLE = {}  # (S, C) -> the oracle's G rows, shared by the evaluate() and training cases (same nets, same inputs)


@pytest.mark.parametrize("S,C,training", NUM_PARAMS, ids=["S%d-C%d-train%d" % p for p in NUM_PARAMS])
def test_refine_matches_fp64(S, C, training):
    from face_generator_b200.lib import NET_D, NET_G
    from face_generator_b200.pyramid import refine
    N = 13
    ctx = _ctx(C)
    net = _net(ctx, S)
    images, noise, masks = _inputs(net, N, S // 2)
    out, pick, pred = refine(net, images, T, training=training, noise=noise, masks=masks if training else None)
    ref = RR.refine(net.get_params(NET_G).astype(np.float64), net.get_params(NET_D).astype(np.float64), images, S,
                    noise.astype(np.float64), masks.astype(np.float64), training, _G_ORACLE.get((S, C)))
    _G_ORACLE[(S, C)] = ref["diff"]
    p32 = ref["pred"].astype(np.float32).astype(np.float64)
    assert np.linalg.norm(pred - p32) <= 1e-4 * np.linalg.norm(p32)
    # every G row, through the composed path (bitwise refine's, test_refine_is_the_composed_path)
    _, _, _, up, diff = _composed(ctx, net, images, noise, masks, training, T, MAXB)
    for r in range(N * T):
        assert np.linalg.norm(diff[r] - ref["diff"][r]) <= 1e-4 * np.linalg.norm(ref["diff"][r]), r
    srt = np.sort(p32, axis=1)
    clear = (srt[:, -1] - srt[:, -2] > 2e-5) if T > 1 else np.ones(N, bool)
    np.testing.assert_array_equal(pick[clear], ref["pick"][clear])
    want = ref["up"] + ref["diff"].reshape(N, T, C, S, S)[np.arange(N), pick]
    np.testing.assert_allclose(out, want, rtol=0, atol=1e-4)
    net.close()
    ctx.close()


# ============================================================================================ bitwise properties
@pytest.mark.parametrize("training", [0, 1])
def test_refine_is_the_composed_path(training):
    from face_generator_b200.pyramid import refine
    N, S = 13, 32
    ctx = _ctx()
    net = _net(ctx, S)
    images, noise, masks = _inputs(net, N, 16)
    got = refine(net, images, T, chunk=MAXB // T, training=training, noise=noise, masks=masks)
    want = _composed(ctx, net, images, noise, masks, training, T, MAXB)[:3]
    _same(got, want)
    net.close()
    ctx.close()


def test_default_streams_are_noise_uniform_and_dropout_mask():
    from face_generator_b200.lib import _check, _ptr
    from face_generator_b200.pyramid import refine
    N, S, seed = 5, 32, 21
    ctx = _ctx()
    net = _net(ctx, S)
    images = _inputs(net, N, 16)[0]
    noise = np.empty((N * T, 1, S, S), np.float32)
    _check(ctx.lib.fg_noise_uniform(ctx.h, 2 * seed, noise.size, _ptr(noise)), "fg_noise_uniform")
    masks = ctx.dropout_mask(N * T * net.mask_per_sample, 0.5, 2 * seed + 1)
    _same(refine(net, images, T, seed=seed), refine(net, images, T, seed=seed, noise=noise, masks=masks))
    net.close()
    ctx.close()


@pytest.mark.parametrize("f16", [1, 0])
def test_result_does_not_depend_on_chunk(f16):
    from face_generator_b200.pyramid import refine
    N, S, maxB = 13, 64, 80
    ctx = _ctx(maxB=maxB, f16=f16)
    net = _net(ctx, S)
    images = _inputs(net, N, 32)[0]
    runs = [refine(net, images, T, chunk=ch, seed=5) for ch in (1, 7, maxB // T)]
    for r in runs[1:]:
        _same(runs[0], r)
    _same(runs[0], refine(net, images, T, chunk=7, seed=5))  # the same seed twice
    net.close()
    ctx.close()


def test_host_and_device_buffers_give_the_same_bits():
    from face_generator_b200.lib import _check, _ptr
    from face_generator_b200.pyramid import refine
    N, S = 13, 32
    ctx = _ctx()
    net = _net(ctx, S)
    images, noise, masks = _inputs(net, N, 16)
    host = refine(net, images, T, noise=noise, masks=masks)
    dims = [ctx.dev_array(a) for a in (images, noise, masks)]
    outs = [ctx.dev_array(np.zeros(n, np.float32)) for n in (N * net.C * S * S, N, N * T)]
    _check(ctx.lib.fg_c2f_refine(net.h, dims[0], N, 16, T, 3, 1, dims[1], dims[2], 0, outs[0], outs[1], outs[2]),
           "fg_c2f_refine")
    dev = [np.empty_like(host[0]), np.empty(N, np.int32), np.empty_like(host[2])]
    for h, d in zip(dev, outs):
        _check(ctx.lib.fg_memcpy(ctx.h, h.ctypes.data_as(ctypes.c_void_p), d, h.nbytes), "fg_memcpy")
    _same(host, dev)
    for p in dims + outs:
        ctx.dev_free(p)
    net.close()
    ctx.close()


# ============================================================================================ edges
def test_one_try_is_up_plus_the_G_diff_and_equal_sizes_do_not_rescale():
    from face_generator_b200.pyramid import refine
    N, S = 9, 32
    ctx = _ctx()
    net = _net(ctx, S)
    images, noise, _ = _inputs(net, N, S, tries=1)
    out, pick, pred = refine(net, images, 1, training=0, noise=noise)
    assert (pick == 0).all()
    np.testing.assert_array_equal(out, images + net.G_forward(noise, images))  # in_size = S: up is the image itself
    net.close()
    ctx.close()


def test_four_fold_enlarge_16_to_64():
    from face_generator_b200.pyramid import refine
    N, S = 6, 64
    ctx = _ctx()
    net = _net(ctx, S)
    images, noise, masks = _inputs(net, N, 16)
    _same(refine(net, images, T, chunk=MAXB // T, noise=noise, masks=masks),
          _composed(ctx, net, images, noise, masks, 1, T, MAXB)[:3])
    net.close()
    ctx.close()


def test_bad_arguments_launch_nothing():
    from face_generator_b200.lib import _ptr
    N, S = 4, 32
    ctx = _ctx()
    net = _net(ctx, S)
    images = _inputs(net, N, 16)[0]
    out = np.empty((N, 3, S, S), np.float32)
    fn = ctx.lib.fg_c2f_refine
    before = ctx.launches()
    bad = [(_ptr(images), N, 16, 0, 1, _ptr(out)),            # tries < 1
           (_ptr(images), N, 16, T, MAXB // T + 1, _ptr(out)),  # chunk * tries > max_batch
           (_ptr(images), N, 16, T, 0, _ptr(out)),            # chunk < 1
           (_ptr(images), N, 0, T, 1, _ptr(out)),             # in_size outside 1..64
           (_ptr(images), N, 65, T, 1, _ptr(out)),
           (None, N, 16, T, 1, _ptr(out)),                    # NULL images
           (_ptr(images), N, 16, T, 1, None),                 # NULL out
           (_ptr(images), 0, 16, T, 1, _ptr(out))]            # N < 1
    for im, n, ins, tries, chunk, o in bad:
        assert fn(net.h, im, n, ins, tries, chunk, 1, None, None, 0, o, None, None) != 0
        assert ctx.lib.fg_last_error()
    assert fn(None, _ptr(images), N, 16, T, 1, 1, None, None, 0, _ptr(out), None, None) != 0
    assert ctx.launches() == before
    net.close()
    ctx.close()


# ============================================================================================ pyramid
def test_pyramid_is_the_hand_chain():
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_G, _check, _ptr
    from face_generator_b200.pyramid import refine, sample_pyramid
    from oracle import oracle_s16 as O16
    N, chunk, seed = 7, 4, 3
    ctx = _ctx()
    rng = np.random.default_rng(9)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(3), rng))
    s16 = fg.S16(ctx)
    s16.set_params(NET_G, LY.trained_like_init((O16.G_layout(3), O16.G_param_count(3)), rng))
    l32, l64 = _net(ctx, 32, 1), _net(ctx, 64, 2)
    noise = np.empty((N, 100), np.float32)
    _check(ctx.lib.fg_noise_uniform(ctx.h, 4 * seed, noise.size, _ptr(noise)), "fg_noise_uniform")
    # 32 -> 64
    got = sample_pyramid(ctx, [l64], N, T, chunk, seed)
    want = refine(l64, ctx.sample(noise, chunk), T, seed=4 * seed + 1)[0]
    np.testing.assert_array_equal(got, want)
    # 16 -> 32 -> 64
    got = sample_pyramid(s16, [l32, l64], N, T, chunk, seed)
    base = np.concatenate([s16.G_forward(noise[s:s + chunk], training=True) for s in range(0, N, chunk)])
    mid = refine(l32, base, T, seed=4 * seed + 1)[0]
    np.testing.assert_array_equal(got, refine(l64, mid, T, seed=4 * seed + 2)[0])
    for n in (l32, l64, s16):
        n.close()
    ctx.close()


# ============================================================================================ checkpoints
def test_c2f_checkpoint_loads_exactly(tmp_path):
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200.lib import NET_D, NET_G
    from test_c2f_refine_cpu import write_c2f_like
    p = tmp_path / "adversarial_c2f_32_to_64.net"
    PG, PD = write_c2f_like(p, 3, 64)
    ctx = _ctx()
    net = _net(ctx, 64)
    assert CK.load_c2f_checkpoint(net, p) == 11
    np.testing.assert_array_equal(net.get_params(NET_G), PG)
    np.testing.assert_array_equal(net.get_params(NET_D), PD)
    net.close()
    ctx.close()
