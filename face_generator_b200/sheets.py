"""sample.lua's image sheets on the GPU: the JPEG files `th sample.lua` writes into --writeto.

image_grid   image.toDisplayTensor{input=images, nrow=nrow, padding=padding} + image.save's byte conversion
             (fg_image_grid): uint8 [C][Hg][Wg]
encode_jpeg  image.save's JPEG files of uint8 images, byte for byte Pillow's (fg_jpeg_encode)
save_image   one sheet (or uint8 image) written to a JPEG file
sample_run   sample.lua:main()'s loop body for one run: the five sheets, and the neighbour sheet with a dataset

The executable mirror of lua/sample_b200.lua's main().
"""
import ctypes as C
import os

import numpy as np

from .lib import NOISE_DIM, S16, FGError, _check, _ptr

_U64 = 2 ** 64 - 1


class DeviceImages:
    """float32 images [N][C][H][W] at a device address (fg_dev_alloc, fg_sample's output, ...); not owned."""

    def __init__(self, addr, shape):
        self.addr, self.shape = int(addr), tuple(int(v) for v in shape)


def _images_arg(images):
    if isinstance(images, DeviceImages):
        return C.c_void_p(images.addr), images.shape
    a = np.ascontiguousarray(images, np.float32)
    if a.ndim != 4:
        raise FGError("image_grid: images must be [N][C][H][W], got %s" % (a.shape,))
    return a, a.shape


def _order_arg(order):
    if order is None or isinstance(order, int):  # None, or a device address of int32 entries
        return order
    return np.ascontiguousarray(order, np.int32)


def grid_size(ctx, shape, nrow, padding=0, count=None):
    """(Hg, Wg) of the sheet of `count` (default N) images of shape [N][C][H][W] (fg_image_grid's size query)."""
    N, Cc, H, W = shape
    hg, wg = C.c_int(0), C.c_int(0)
    dummy = C.c_void_p(1)  # not read: a size query launches nothing
    _check(ctx.lib.fg_image_grid(ctx.h, dummy, N, Cc, H, W, None, N if count is None else count, nrow, padding, None,
                                 C.byref(hg), C.byref(wg)), "fg_image_grid")
    return hg.value, wg.value


def image_grid(ctx, images, nrow, padding=0, order=None, count=None, out=None):
    """toDisplayTensor of images[order] (all N images when order is None) -> uint8 [C][Hg][Wg].

    images: float32 [N][C][H][W] numpy array or DeviceImages; order: int32 indices (numpy, host) or a device address
    of `count` int32 entries; out: None (a new host array is returned) or a device address of C*Hg*Wg bytes (returned
    as is)."""
    img, (N, Cc, H, W) = _images_arg(images)
    order = _order_arg(order)
    if count is None:
        if isinstance(order, int):
            raise FGError("image_grid: a device order needs count")
        count = N if order is None else order.size
    Hg, Wg = grid_size(ctx, (N, Cc, H, W), nrow, padding, count)
    dst = np.empty((Cc, Hg, Wg), np.uint8) if out is None else out
    optr = None if order is None else (C.c_void_p(order) if isinstance(order, int) else order.ctypes.data_as(C.c_void_p))
    dptr = dst.ctypes.data_as(C.c_void_p) if out is None else C.c_void_p(int(out))
    _check(ctx.lib.fg_image_grid(ctx.h, _ptr(img) if isinstance(img, np.ndarray) else img, N, Cc, H, W, optr, count, nrow,
                                 padding, dptr, None, None), "fg_image_grid")
    return dst


def encode_jpeg(ctx, images_u8, quality=75, shape=None):
    """JPEG files (list of bytes) of uint8 images [C][H][W] or [count][C][H][W], C = 1 or 3: what Pillow's
    Image.save(f, "JPEG", quality=quality) writes.  images_u8 may be a device address, with `shape` given."""
    if isinstance(images_u8, int):
        ptr, shape = C.c_void_p(images_u8), tuple(shape)
    else:
        a = np.ascontiguousarray(images_u8, np.uint8)
        shape = a.shape
        ptr = a.ctypes.data_as(C.c_void_p)
    if len(shape) == 3:
        shape = (1,) + tuple(shape)
    n, Cc, H, W = shape
    offsets = np.zeros(n + 1, np.int64)
    op = offsets.ctypes.data_as(C.c_void_p)
    _check(ctx.lib.fg_jpeg_encode(ctx.h, ptr, n, Cc, H, W, quality, None, 0, op), "fg_jpeg_encode")
    out = np.empty(max(int(offsets[-1]), 1), np.uint8)
    _check(ctx.lib.fg_jpeg_encode(ctx.h, ptr, n, Cc, H, W, quality, out.ctypes.data_as(C.c_void_p), out.size, op),
           "fg_jpeg_encode")
    data = out.tobytes()
    return [data[offsets[i]:offsets[i + 1]] for i in range(n)]


def save_image(ctx, path, grid_or_images, nrow=8, padding=0, order=None, quality=75):
    """image.save(path, x) for a JPEG path: x a uint8 sheet [C][H][W] (written as is) or float images [N][C][H][W]
    (a numpy array or DeviceImages; laid out by image_grid first)."""
    x = grid_or_images
    if not isinstance(x, DeviceImages) and np.asarray(x).dtype == np.uint8:
        data = encode_jpeg(ctx, x, quality)[0]
    else:
        data = encode_jpeg(ctx, image_grid(ctx, x, nrow, padding, order), quality)[0]
    with open(path, "wb") as f:
        f.write(data)


# ---- sample.lua:main() ------------------------------------------------------------------------------------------------
def run_streams(seed, run):
    """The seeds of run `run` (sample.lua's 1-based run counter) under --seed `seed`: key = seed * 1000003 + run
    (64-bit), then 8 * key + k for k = 0 noise (fg_noise_uniform), 1 and 2 the dropout masks of the best and worst
    scoring passes, 3 and 4 the permutations of the random256 and random sheets."""
    key = (int(seed) * 1000003 + int(run)) & _U64
    return [(8 * key + k) & _U64 for k in range(5)]


def permutation(stream, n):
    """The documented stand-in for torch.randperm(n) (Torch's CPU stream cannot be reproduced): 0..n-1 sorted by the
    splitmix64 hash of stream * 2^32 + i, ties by i."""
    with np.errstate(over="ignore"):
        x = np.uint64(stream) * np.uint64(1 << 32) + np.arange(n, dtype=np.uint64)
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return np.argsort(x, kind="stable").astype(np.int32)


SHEETS = ("random256_%04d_base.jpg", "random1024_%04d_base.jpg", "best_%04d_base.jpg", "worst_%04d_base.jpg",
          "random_%04d_base.jpg")
NEIGHBOURS_SHEET = "best_%04d_neighbours_base.jpg"


def sample_run(base, run, writeto, N=1024, chunk=16, seed=0, neighbours=None, quality=75, return_images=False):
    """One pass of sample.lua:main()'s loop (run = its 1-based counter): N images from `base` (a Context: the 32x32
    G, fg_sample; or an S16: --scale 16, training-mode G forward `chunk` at a time, as createImagesFromNoise), then
    the sheets of sample.lua:81-99 written into `writeto` as quality-75 JPEG files:
      random256   256 images of permutation(streams[3]), 16 per row
      random1024  all N, 32 per row
      best        the 64 D rates most real, from a scoring pass with live dropout (seed streams[1]), 8 per row
      worst       the 64 it rates most fake, from a second pass (seed streams[2]), 8 per row
      random      64 images of permutation(streams[4]), 8 per row
      neighbours  (a DeviceDataset given) the first 16 best, each followed by its nearest training image at the
                  base's size (torch.dist), 16 per row
    The images stay in device memory; the predictions and the files come back.  Returns a dict: the file paths, the
    two passes' predictions and the best / worst / random orders, the neighbours' dataset indices, and with
    return_images the N images (downloaded for inspection)."""
    s16 = isinstance(base, S16)
    ctx = base.ctx if s16 else base
    lib, Cc, S = ctx.lib, ctx.C, (16 if s16 else 32)
    if not 1 <= chunk <= ctx.max_batch:
        raise FGError("sample_run: chunk %d outside [1, %d]" % (chunk, ctx.max_batch))
    if N < 256:
        raise FGError("sample_run: N = %d, the sheets need at least 256 images" % N)
    streams = run_streams(seed, run)
    per = Cc * S * S
    names = [os.path.join(writeto, f % run) for f in SHEETS]
    os.makedirs(writeto, exist_ok=True)
    bufs = []

    def dev(nbytes):
        p = lib.fg_dev_alloc(max(int(nbytes), 4))
        if not p:
            raise FGError("fg_dev_alloc failed: " + lib.fg_last_error().decode())
        bufs.append(p)
        return p

    try:
        noise = dev(4 * N * NOISE_DIM)
        _check(lib.fg_noise_uniform(ctx.h, streams[0], N * NOISE_DIM, noise), "fg_noise_uniform")
        imgs = dev(4 * N * per)
        if s16:
            for s in range(0, N, chunk):
                b = min(chunk, N - s)
                _check(lib.fg_s16_G_forward(base.h, noise + 4 * s * NOISE_DIM, b, 1, imgs + 4 * s * per), "fg_s16_G_forward")
        else:
            _check(lib.fg_sample(ctx.h, noise, N, chunk, imgs), "fg_sample")
        images = DeviceImages(imgs, (N, Cc, S, S))
        score = lib.fg_s16_D_score if s16 else lib.fg_D_score
        h = base.h if s16 else ctx.h
        preds = []
        for k in (1, 2):
            p = np.empty(N, np.float32)
            _check(score(h, imgs, N, chunk, 1, streams[k], p.ctypes.data_as(C.c_void_p)), score.__name__)
            preds.append(p)
        best = np.argsort(-preds[0], kind="stable")[:64].astype(np.int32)   # sortImagesByPrediction(images, false, 64)
        worst = np.argsort(preds[1], kind="stable")[:64].astype(np.int32)   # sortImagesByPrediction(images, true, 64)
        r256, r64 = permutation(streams[3], N)[:256], permutation(streams[4], N)[:64]
        sheets = [(images, r256, 16), (images, None, 32), (images, best, 8), (images, worst, 8), (images, r64, 8)]
        result = dict(files=list(names), preds_best=preds[0], preds_worst=preds[1], best=best, worst=worst,
                      random256=r256, random=r64)
        if neighbours is not None:
            # the 16 best and their nearest training images, [16 best][16 neighbours], interleaved by the order
            pairs = dev(4 * 32 * per)
            for i in range(16):
                _check(lib.fg_memcpy(ctx.h, pairs + 4 * i * per, imgs + 4 * int(best[i]) * per, 4 * per), "fg_memcpy")
            idx, dist = dev(4 * 16), dev(4 * 16)
            _check(lib.fg_dataset_nearest_sized(neighbours.h, S, pairs, 16, idx, dist), "fg_dataset_nearest_sized")
            _check(lib.fg_dataset_gather_sized(neighbours.h, idx, 16, S, pairs + 4 * 16 * per), "fg_dataset_gather_sized")
            order = np.array([v for i in range(16) for v in (i, 16 + i)], np.int32)
            sheets.append((DeviceImages(pairs, (32, Cc, S, S)), order, 16))
            names.append(os.path.join(writeto, NEIGHBOURS_SHEET % run))
            nb = np.empty(16, np.int32)
            _check(lib.fg_memcpy(ctx.h, nb.ctypes.data_as(C.c_void_p), idx, 64), "fg_memcpy")
            result["files"], result["neighbours"] = list(names), nb
        sizes = [grid_size(ctx, src.shape, nrow, 0, src.shape[0] if order is None else order.size)
                 for src, order, nrow in sheets]
        out = dev(Cc * max(hg * wg for hg, wg in sizes))
        for (src, order, nrow), (Hg, Wg), path in zip(sheets, sizes, names):
            image_grid(ctx, src, nrow, 0, order, out=out)
            data = encode_jpeg(ctx, out, quality, shape=(Cc, Hg, Wg))[0]
            with open(path, "wb") as f:
                f.write(data)
        if return_images:
            host = np.empty((N, Cc, S, S), np.float32)
            _check(lib.fg_memcpy(ctx.h, host.ctypes.data_as(C.c_void_p), imgs, host.nbytes), "fg_memcpy")
            result["images"] = host
        return result
    finally:
        ctx.sync()
        for p in bufs:
            lib.fg_dev_free(p)
