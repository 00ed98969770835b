"""sample.lua's coarse-to-fine pyramid on the GPU: a base generator's faces refined by trained c2f levels (16 -> 32 -> 64).

image_scale    image.scale(x, size, size) on float batches (fg_image_scale)
refine         sample.lua:176-214 c2f(images, G, D, fineSize) with one C2f net (fg_c2f_refine)
sample_pyramid base G, then every level in turn; intermediates stay in device memory

The executable mirror of lua/sample_b200.lua.
"""
import ctypes as C

import numpy as np

from .lib import NOISE_DIM, S16, FGError, _check, _ptr, f32


def image_scale(ctx, x, size):
    """image.scale(x, size, size) (default 'bilinear' mode) of x [N][C][H][W] -> [N][C][size][size], float32 host arrays."""
    x = f32(x)
    N, Cc, H, W = x.shape
    out = np.empty((N, Cc, size, size), np.float32)
    _check(ctx.lib.fg_image_scale(ctx.h, _ptr(x), N, Cc, H, W, size, size, _ptr(out)), "fg_image_scale")
    return out


def _refine_call(net, images, N, in_size, tries, chunk, training, seed, noise, masks, out, pick, pred):
    """fg_c2f_refine on pointers (numpy float32 arrays or raw device addresses; pick: int32 array or None)"""
    if chunk is None:
        chunk = max(1, net.ctx.max_batch // tries)
    pk = pick.ctypes.data_as(C.c_void_p) if pick is not None else None
    _check(net.lib.fg_c2f_refine(net.h, _ptr(images), N, in_size, tries, chunk, int(training), _ptr(noise), _ptr(masks),
                                 seed, _ptr(out), pk, _ptr(pred)), "fg_c2f_refine")


def refine(net, images, tries=10, chunk=None, training=True, seed=0, noise=None, masks=None):
    """sample.lua's c2f(images, G, D, fineSize) with the C2f `net` (fine size S): images [N][C][in][in], in <= 64.
    Returns (out [N][C][S][S], pick [N] int32, pred [N][tries]).  chunk: images per pass (default max_batch // tries);
    training=True keeps D's dropout live as sample.lua does; noise [N][tries][1][S][S] and masks
    [N][tries][mask_per_sample] default to the streams 2*seed and 2*seed+1 (fg_b200.h)."""
    images = f32(images)
    N, Cc, H, W = images.shape
    if H != W or Cc != net.C:
        raise FGError("refine: images must be [N][%d][in][in], got %s" % (net.C, images.shape))
    S = net.S
    noise = None if noise is None else net._sized("refine noise", noise, N * tries * S * S)
    masks = None if masks is None else net._sized("refine masks", masks, N * tries * net.mask_per_sample)
    out = np.empty((N, Cc, S, S), np.float32)
    pick = np.empty(N, np.int32)
    pred = np.empty((N, tries), np.float32)
    _refine_call(net, images, N, H, tries, chunk, training, seed, noise, masks, out, pick, pred)
    return out, pick, pred


def _dev_empty(ctx, n):
    p = ctx.lib.fg_dev_alloc(max(int(n), 1) * 4)
    if not p:
        raise FGError("fg_dev_alloc failed: " + ctx.lib.fg_last_error().decode())
    return p


def sample_pyramid(base, levels, N, tries=10, chunk=16, seed=0):
    """N faces from `base`, refined by each C2f of `levels` (increasing fine sizes, same ctx) in turn.

    base: a Context (32x32 G through fg_sample, `chunk` images per training-mode BatchNorm batch, as sample.lua) or an
    S16 (16x16 G, training-mode, `chunk` at a time).  Base noise is fg_noise_uniform(4*seed, N*100); level k refines
    with seed 4*seed+1+k (training-mode D, `tries` tries).  Only the last level's images come back to the host:
    returns [N][C][S][S] float32."""
    if not levels:
        raise FGError("sample_pyramid: no levels")
    s16 = isinstance(base, S16)
    ctx = base.ctx if s16 else base
    if any(lv.ctx is not ctx for lv in levels):
        raise FGError("sample_pyramid: every level must live on the base's ctx")
    if not 1 <= chunk <= ctx.max_batch:
        raise FGError("sample_pyramid: chunk %d outside [1, %d]" % (chunk, ctx.max_batch))
    lib, Cc = ctx.lib, ctx.C
    size = 16 if s16 else 32
    bufs = []
    try:
        noise = _dev_empty(ctx, N * NOISE_DIM)
        bufs.append(noise)
        _check(lib.fg_noise_uniform(ctx.h, 4 * seed, N * NOISE_DIM, noise), "fg_noise_uniform")
        cur = _dev_empty(ctx, N * Cc * size * size)
        bufs.append(cur)
        if s16:
            for s in range(0, N, chunk):
                b = min(chunk, N - s)
                _check(lib.fg_s16_G_forward(base.h, noise + 4 * s * NOISE_DIM, b, 1, cur + 4 * s * Cc * 256),
                       "fg_s16_G_forward")
        else:
            _check(lib.fg_sample(ctx.h, noise, N, chunk, cur), "fg_sample")
        for k, lv in enumerate(levels):
            last = k == len(levels) - 1
            out = np.empty((N, Cc, lv.S, lv.S), np.float32) if last else _dev_empty(ctx, N * Cc * lv.S * lv.S)
            if not last:
                bufs.append(out)
            _refine_call(lv, cur, N, size, tries, None, True, 4 * seed + 1 + k, None, None, out, None, None)
            cur, size = out, lv.S
        return cur
    finally:
        ctx.sync()
        for p in bufs:
            lib.fg_dev_free(p)
