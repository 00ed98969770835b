"""numpy float32 restatement of sample.lua's sheets before the JPEG encoder, op for op as fg_image_grid (sheets.cu):
image.toDisplayTensor{input=images, nrow=nrow, padding=padding} (defaults otherwise), image.minmax over the grid, and
image.save's byte conversion (clampImage, *255, to unsigned char).

    grid(images, nrow, padding=0, order=None) -> uint8 [C][Hg][Wg]

The three rules of torch/image that no available source pins are each one function here, as in sheets.cu:
scale (minmax divides by max - min), rescales (a constant grid is not divided) and to_byte (saturate, *255,
truncate; NaN -> 0).  NaN values take no part in the minimum and maximum.
"""
import numpy as np


def ordered_keys(x):
    """float32 -> uint32 keys in the same order (-0 just below +0), as the kernel's atomicMin / atomicMax see them."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def key_value(k):
    k = np.uint32(k)
    u = k & np.uint32(0x7FFFFFFF) if k & np.uint32(0x80000000) else ~k
    return np.array([u], np.uint32).view(np.float32)[0]


def extremes(x):
    """(min, max) of the non-NaN values of x, float32; (0, 0) when every value is NaN."""
    x = np.asarray(x, np.float32).ravel()
    x = x[~np.isnan(x)]
    if not x.size:
        return np.float32(0), np.float32(0)
    k = ordered_keys(x)
    return key_value(k.min()), key_value(k.max())


def scale(shifted, rng):
    """assumption 1: minmax divides by (max - min) in float32"""
    return (shifted / np.float32(rng)).astype(np.float32)


def rescales(rng):
    """assumption 2: a constant grid (max - min == 0) is shifted by -min and not divided"""
    return rng != 0


def to_byte(x):
    """assumption 3: clampImage saturates to [0, 1], the writer multiplies by 255 in float32 and truncates; NaN -> 0"""
    x = np.asarray(x, np.float32)
    y = np.clip(np.where(np.isnan(x), np.float32(0), x), np.float32(0), np.float32(1)).astype(np.float32)
    return (y * np.float32(255)).astype(np.float32).astype(np.uint8)


def layout(images, nrow, padding, fill):
    """toDisplayTensor's grid of images [count][C][H][W]: xmaps = min(nrow, count) columns, ceil(count / xmaps) rows
    of (H+padding) x (W+padding) cells, image k in cell (k // xmaps, k % xmaps) at offset padding / 2, fill elsewhere."""
    count, C, H, W = images.shape
    xmaps = min(nrow, count)
    ymaps = -(-count // xmaps)
    ch, cw, half = H + padding, W + padding, padding // 2
    g = np.full((C, ymaps * ch, xmaps * cw), fill, np.float32)
    for k in range(count):
        y, x = divmod(k, xmaps)
        g[:, y * ch + half:y * ch + half + H, x * cw + half:x * cw + half + W] = images[k]
    return g


def grid(images, nrow, padding=0, order=None):
    images = np.asarray(images, np.float32)
    sel = images if order is None else images[np.asarray(order, np.int64)]
    mn, mx = extremes(sel)
    g = layout(sel, nrow, padding, mx)
    rng = np.float32(mx - mn)
    t = (g - mn).astype(np.float32)
    if rescales(rng):
        t = scale(t, rng)
    return to_byte(t)
