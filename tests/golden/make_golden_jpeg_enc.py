"""Writes tests/golden/jpeg_encode.npz: what Pillow's Image.save(f, "JPEG", quality=q) writes for generated rows and
what Pillow decodes those files to, for fg_dataset_encode_jpeg / fg_dataset_jpeg_roundtrip.  Every input comes from
tests/jpeg_enc_ref.content(kind, seed, C, H, W), a counter-based integer hash, so the GPU tests regenerate it with numpy
alone; the npz keeps the SHA-256 of Pillow's bytes and of Pillow's planar decode, and the full bytes of a few cases.

    python tests/golden/make_golden_jpeg_enc.py      # rewrites the npz (Pillow with libjpeg-turbo required)

Arrays (N cases):
    kind [N] str, seed, C, H, W, quality [N] int32   the input content(kind, seed, C, H, W) and the quality
    file_sha256, decode_sha256 [N] str               SHA-256 (hex) of Pillow's file and of its [C][H][W] uint8 decode
    full_idx [K] int32, full_data uint8, full_offsets [K+1] int64   the files of K cases, back to back
"""
import hashlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_enc_ref as R  # noqa: E402

SIZES = ((1, 1), (2, 3), (2, 16), (4, 7), (6, 6), (7, 13), (8, 8), (10, 17), (14, 9), (15, 17), (16, 16), (31, 33),
         (63, 65), (64, 64), (84, 84))
QUALITIES = (1, 10, 50, 75, 90, 100)
BIG = ((250, 250), (75, 75))  # faces and noise at q75 only


def cases():
    out = []
    for (H, W) in SIZES:
        for q in QUALITIES:
            for C in (3, 1):
                for k, kind in enumerate(R.KINDS):
                    out.append((kind, 1000 * H + W + 17 * k + q, C, H, W, q))
    for (H, W) in BIG:
        for C in (3, 1):
            for kind in ("face", "noise"):
                out.append((kind, 7 * H + W, C, H, W, 75))
    return out


def pillow(img, q):
    from PIL import Image
    a = img[0] if img.shape[0] == 1 else img.transpose(1, 2, 0)
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "JPEG", quality=q)
    b = buf.getvalue()
    d = np.asarray(Image.open(io.BytesIO(b)))
    return b, (d[None] if d.ndim == 2 else d.transpose(2, 0, 1))


def build():
    import PIL.features
    assert PIL.features.check_feature("libjpeg_turbo"), "Pillow must be built with libjpeg-turbo"
    cs = cases()
    fsha, dsha, full = [], [], []
    for i, (kind, seed, C, H, W, q) in enumerate(cs):
        b, d = pillow(R.content(kind, seed, C, H, W), q)
        fsha.append(hashlib.sha256(b).hexdigest())
        dsha.append(hashlib.sha256(np.ascontiguousarray(d, np.uint8).tobytes()).hexdigest())
        if (H, W) in ((64, 64), (15, 17)) and q == 75 and kind in ("face", "noise"):
            full.append((i, b))
    i32 = lambda v: np.asarray(v, np.int32)
    off = np.zeros(len(full) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for _, b in full])
    return dict(kind=np.asarray([c[0] for c in cs]), seed=i32([c[1] for c in cs]), C=i32([c[2] for c in cs]),
                H=i32([c[3] for c in cs]), W=i32([c[4] for c in cs]), quality=i32([c[5] for c in cs]),
                file_sha256=np.asarray(fsha), decode_sha256=np.asarray(dsha), full_idx=i32([i for i, _ in full]),
                full_data=np.frombuffer(b"".join(b for _, b in full), np.uint8), full_offsets=off)


if __name__ == "__main__":
    out = os.path.join(HERE, "jpeg_encode.npz")
    arrays = build()
    np.savez_compressed(out, **arrays)
    print("%s: %d cases, %d full files, %d bytes on disk" % (out, len(arrays["kind"]), len(arrays["full_idx"]),
                                                             os.path.getsize(out)))
