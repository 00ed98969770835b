"""CPU: tests/jpeg_enc_ref.py writes Pillow's bytes at the sizes of sample.lua's sheets (256x256 to 1024x1024, a 512x64
row, a gray sheet, odd sizes such as 33x97 and 4096x8), and tests/golden/sheets_jpeg.npz, which the GPU tests of
fg_jpeg_encode read, holds the SHA-256s of those bytes.  Pillow is needed only for the first test."""
import hashlib
import io
import os

import numpy as np
import pytest

import jpeg_enc_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sheets_jpeg.npz")


def golden_cases():
    with np.load(GOLDEN) as z:
        g = {k: z[k] for k in z.files}
    return [(str(g["kind"][i]), int(g["seed"][i]), int(g["C"][i]), int(g["H"][i]), int(g["W"][i]), int(g["quality"][i]),
             str(g["file_sha256"][i])) for i in range(len(g["kind"]))]


def test_golden_covers_the_sheet_sizes():
    cases = golden_cases()
    sizes = {(C, H, W) for _, _, C, H, W, q, _ in cases if q == 75}
    assert {(3, 256, 256), (3, 512, 512), (3, 1024, 1024), (3, 512, 64), (1, 128, 128), (3, 33, 97),
            (3, 4096, 8)} <= sizes
    assert {(C, H, W, q) for _, _, C, H, W, q, _ in cases if q != 75} >= {(3, 512, 512, 1), (3, 512, 512, 100),
                                                                          (1, 128, 128, 50)}


@pytest.mark.parametrize("i", range(len(golden_cases())))
def test_reference_equals_golden_sha(i):
    kind, seed, C, H, W, q, sha = golden_cases()[i]
    assert hashlib.sha256(R.encode(R.content(kind, seed, C, H, W), q)).hexdigest() == sha, (kind, C, H, W, q)


@pytest.mark.parametrize("C,H,W", [(3, 512, 512), (3, 33, 97), (3, 4096, 8), (1, 128, 128)])
def test_reference_equals_pillow(C, H, W):
    Image = pytest.importorskip("PIL.Image")
    for q in (1, 75, 100):
        img = R.content("noise", 11 * H + W, C, H, W)
        a = img[0] if C == 1 else img.transpose(1, 2, 0)
        buf = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(a)).save(buf, "JPEG", quality=q)
        assert R.encode(img, q) == buf.getvalue(), (C, H, W, q)
