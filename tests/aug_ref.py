"""numpy restatement of the LFW augmentation (face_generator_b200/csrc/k_aug.cuh, augment.cu), float64 op for op:
the parameter draws of fg_lfw_aug_params, the flip / brightness / scikit-image warp of one descriptor, LFW-crop's box
and Pillow's fixed-point BILINEAR resize.  Every product and sum is a separate numpy operation, so nothing is fused.

The warp restates skimage.transform.warp(img, inverse_map, mode="constant", order=1): PARITY UNPINNED (no scikit-image
here).  The resize restates Pillow's Image.resize(size, BILINEAR) and is pinned against Pillow by
tests/test_augment_cpu.py."""
import math

import numpy as np

from face_generator_b200.dataset import AUG_DTYPE  # fg_aug

CROP_Y, CROP_X, CROP = 92, 83, 84
PRECISION_BITS = 22
_M64 = (1 << 64) - 1


# ---- parameter draws ---------------------------------------------------------------------------------------------
def mix64(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def draw(seed, i, a, k):
    key = mix64(mix64(mix64(seed) ^ i) ^ a)
    return (mix64((key + k) & _M64) >> 11) * 2.0 ** -53


def draw_int(seed, i, a, k, lo, hi):
    return min(hi, lo + int(draw(seed, i, a, k) * (hi - lo + 1)))


def draws(seed, i, a):
    """generate_dataset.py's distributions for augmentation a >= 1 of photo i."""
    return dict(scale=0.82 + (1.10 - 0.82) * draw(seed, i, a, 0), deg=draw_int(seed, i, a, 1, -8, 8),
                tx=draw_int(seed, i, a, 2, -5, 5), ty=draw_int(seed, i, a, 3, -5, 5),
                hflip=int(draw(seed, i, a, 4) < 0.5), brightness=0.9 + (1.1 - 0.9) * draw(seed, i, a, 5))


def forward_matrix(scale, deg, tx, ty, H, W):
    """ImageAugmenter's T(+shift) . A . T(-shift), shift = (int(H/2), int(W/2)) for (x, y): augment() passes the
    image's shape[0] as its width."""
    rho = np.deg2rad(deg)
    A = np.array([[scale * math.cos(rho), -scale * math.sin(rho), tx], [scale * math.sin(rho), scale * math.cos(rho), ty],
                  [0.0, 0.0, 1.0]])
    sx, sy = int(H / 2.0), int(W / 2.0)
    to_tl = np.array([[1.0, 0, -sx], [0, 1.0, -sy], [0, 0, 1.0]])
    to_c = np.array([[1.0, 0, sx], [0, 1.0, sy], [0, 0, 1.0]])
    return to_c @ A @ to_tl


def identity_desc(src):
    d = np.zeros((), AUG_DTYPE)
    d["src"], d["brightness"], d["m"] = src, 1.0, np.eye(3).ravel()
    return d


# ---- one output row ------------------------------------------------------------------------------------------------
def brighten(img, b):
    """np.clip(img * b, 0, 255).astype(np.uint8)"""
    return np.clip(img.astype(np.float64) * b, 0, 255).astype(np.uint8)


def warp_crop(src, desc):
    """The flipped, brightened, warped 84x84 crop [C][84][84] uint8 of one source photo [C][H][W] uint8."""
    Cs, H, W = src.shape
    img = src[:, :, ::-1] if desc["hflip"] else src
    f = brighten(img, float(desc["brightness"])) * (1.0 / 255.0)  # img_as_float
    m = np.asarray(desc["m"], np.float64)
    y, x = np.meshgrid(np.arange(CROP_Y, CROP_Y + CROP, dtype=np.float64), np.arange(CROP_X, CROP_X + CROP, dtype=np.float64),
                       indexing="ij")
    xx = (m[0] * x + m[1] * y) + m[2]
    yy = (m[3] * x + m[4] * y) + m[5]
    with np.errstate(divide="ignore", invalid="ignore"):
        if m[6] == 0.0 and m[7] == 0.0 and m[8] == 1.0:
            c, r = xx, yy
        else:
            zz = (m[6] * x + m[7] * y) + m[8]
            c, r = xx / zz, yy / zz
        finite = np.isfinite(c) & np.isfinite(r)
        c, r = np.where(finite, c, 0.0), np.where(finite, r, 0.0)
        r0, r1, c0, c1 = np.floor(r), np.ceil(r), np.floor(c), np.ceil(c)
        dr, dc = r - r0, c - c0

    def px(rr, cc):
        ok = (rr >= 0) & (rr < H) & (cc >= 0) & (cc < W)
        ri, ci = np.where(ok, rr, 0).astype(np.int64), np.where(ok, cc, 0).astype(np.int64)
        return np.where(ok[None], f[:, ri, ci], 0.0)

    top = (1 - dc) * px(r0, c0) + dc * px(r0, c1)
    bot = (1 - dc) * px(r1, c0) + dc * px(r1, c1)
    out = (1 - dr) * top + dr * bot
    out = np.where(finite[None], out, 0.0)
    lo, hi = f.min(), f.max()
    keep = out == 0.0 if lo > 0 else np.zeros(out.shape, bool)
    out = np.clip(out, lo, hi)
    out[keep] = 0.0
    return np.array(out * 255, dtype=np.uint8)


def crop(src):
    return src[:, CROP_Y:CROP_Y + CROP, CROP_X:CROP_X + CROP]


def pillow_coeffs(in_size, out_size):
    """Pillow's precompute_coeffs (triangle filter, support scaled by in/out) + normalize_coeffs_8bpc."""
    in0, in1 = 0.0, float(np.float32(in_size))
    scale = (in1 - in0) / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int64)
    kk = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = in0 + (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = []
        for x in range(xmax):
            t = abs((x + xmin - center + 0.5) * ss)
            k.append(1.0 - t if t < 1.0 else 0.0)
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        for x, w in enumerate(k):
            kk[xx, x] = int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _clip8(v):
    return np.clip(v >> PRECISION_BITS, 0, 255).astype(np.uint8)


def pillow_resize(img, Ho, Wo):
    """Image.resize((Wo, Ho), BILINEAR) of planar images [..][C][H][W] uint8: a horizontal pass into uint8, then the
    vertical pass, each with +2^21 rounding and clip."""
    H, W = img.shape[-2:]
    hb, hk = pillow_coeffs(W, Wo)
    vb, vk = pillow_coeffs(H, Ho)
    a = img.astype(np.int64)
    tmp = np.empty(img.shape[:-1] + (Wo,), np.int64)
    for xo in range(Wo):
        xmin, n = hb[xo]
        acc = np.full(img.shape[:-1], 1 << (PRECISION_BITS - 1), np.int64)
        for k in range(n):
            acc += a[..., xmin + k] * hk[xo, k]
        tmp[..., xo] = _clip8(acc)
    out = np.empty(img.shape[:-2] + (Ho, Wo), np.uint8)
    for yo in range(Ho):
        ymin, n = vb[yo]
        acc = np.full(img.shape[:-2] + (Wo,), 1 << (PRECISION_BITS - 1), np.int64)
        for k in range(n):
            acc += tmp[..., ymin + k, :] * vk[yo, k]
        out[..., yo, :] = _clip8(acc)
    return out


def augment_row(src, desc, Ho=64, Wo=64):
    """One output row [C][Ho][Wo] uint8 of fg_dataset_augment from its source photo [C][H][W] uint8."""
    return pillow_resize(warp_crop(src, desc) if desc["warp"] else crop(src), Ho, Wo)


def augment_rows(srcs, descs, Ho=64, Wo=64, batch=2048):
    """fg_dataset_augment over descriptors whose src indexes srcs [N][C][H][W] (the resize runs batched)."""
    out = []
    for b in range(0, len(descs), batch):
        crops = np.stack([warp_crop(srcs[int(d["src"])], d) if d["warp"] else crop(srcs[int(d["src"])])
                          for d in descs[b:b + batch]])
        out.append(pillow_resize(crops, Ho, Wo))
    return np.concatenate(out)
