"""Writes tests/golden/sheets_jpeg.npz: the SHA-256 of what Pillow's Image.save(f, "JPEG", quality=q) writes for
generated images at the sizes of sample.lua's sheets (256x256 .. 1024x1024, a 512x64 row, a gray sheet, odd sizes),
for fg_jpeg_encode.  Every input comes from tests/jpeg_enc_ref.content(kind, seed, C, H, W), a counter-based integer
hash, so the GPU tests regenerate it with numpy alone.

    python tests/golden/make_golden_sheets.py      # rewrites the npz (Pillow with libjpeg-turbo required)

Arrays (N cases):
    kind [N] str, seed, C, H, W, quality [N] int32   the input content(kind, seed, C, H, W) and the quality
    file_sha256 [N] str                              SHA-256 (hex) of Pillow's file
"""
import hashlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_enc_ref as R  # noqa: E402

SIZES = ((3, 256, 256), (3, 512, 512), (3, 1024, 1024), (3, 512, 64), (1, 128, 128), (3, 33, 97), (3, 4096, 8))
QUALITY_SIZES = ((3, 512, 512), (1, 128, 128))  # also at quality 1, 50 and 100


def cases():
    out = []
    for C, H, W in SIZES:
        for kind in ("lines", "noise"):
            out.append((kind, 3 * H + W, C, H, W, 75))
    for C, H, W in QUALITY_SIZES:
        for q in (1, 50, 100):
            for kind in ("gradient", "noise"):
                out.append((kind, 5 * H + W + q, C, H, W, q))
    return out


def pillow_bytes(img, q):
    from PIL import Image
    a = img[0] if img.shape[0] == 1 else img.transpose(1, 2, 0)
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(a)).save(buf, "JPEG", quality=q)
    return buf.getvalue()


def main():
    cs = cases()
    shas = []
    for kind, seed, C, H, W, q in cs:
        b = pillow_bytes(R.content(kind, seed, C, H, W), q)
        shas.append(hashlib.sha256(b).hexdigest())
    col = lambda i: np.array([c[i] for c in cs], np.int32)
    np.savez_compressed(os.path.join(HERE, "sheets_jpeg.npz"), kind=np.array([c[0] for c in cs]), seed=col(1), C=col(2),
                        H=col(3), W=col(4), quality=col(5), file_sha256=np.array(shas))
    print("%d cases" % len(cs))


if __name__ == "__main__":
    main()
