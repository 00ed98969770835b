"""CPU: tests/jpeg_enc_ref.py, the restatement of the encoder that fg_dataset_encode_jpeg is held to, writes Pillow's
bytes exactly: across sizes that reach every dummy-block and edge-expansion case, qualities 1..100, RGB and L, and
content that reaches DC category 11, AC category 10, ZRL runs and 0xFF stuffing.  Without Pillow, the golden npz the
GPU tests read is checked against the reference instead."""
import hashlib
import io
import os

import numpy as np
import pytest

import jpeg_enc_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_encode.npz")
SIZES = ((1, 1), (2, 3), (7, 13), (8, 8), (15, 17), (16, 16), (31, 33), (63, 65), (64, 64), (84, 84), (250, 250))
QUALITIES = (1, 5, 10, 25, 50, 75, 90, 95, 100)
CONTENT = ("noise", "face", "flat0", "flat255", "checker", "lines")


def pillow_bytes(img, q):
    Image = pytest.importorskip("PIL.Image")
    a = img[0] if img.shape[0] == 1 else img.transpose(1, 2, 0)
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(a)).save(buf, "JPEG", quality=q)
    return buf.getvalue()


def first_difference(a, b):
    n = next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))
    return "lengths %d / %d, first difference at byte %d" % (len(a), len(b), n)


@pytest.mark.parametrize("H,W", SIZES)
def test_reference_equals_pillow(H, W):
    qs = QUALITIES if H * W <= 84 * 84 else (5, 75, 100)
    for q in qs:
        for C in (3, 1):
            for kind in CONTENT:
                img = R.content(kind, H * 31 + W + q, C, H, W)
                got, want = R.encode(img, q), pillow_bytes(img, q)
                assert got == want, (kind, C, H, W, q, first_difference(got, want))


@pytest.mark.parametrize("W", [1, 2, 5, 8, 13, 16, 21, 32])
def test_even_heights_below_16(W):
    """Chroma is padded from its last downsampled row, not from full-resolution rows replicated to 16."""
    for H in range(2, 16, 2):
        for q in (50, 95):
            for kind in ("noise", "gradient"):
                img = R.content(kind, H * 97 + W, 3, H, W)
                got, want = R.encode(img, q), pillow_bytes(img, q)
                assert got == want, (kind, H, W, q, first_difference(got, want))


def test_content_reaches_the_rare_codes():
    """The grid above codes DC differences of category 11, AC coefficients of category 10, ZRL runs and 0xFF bytes."""
    cats_dc, cats_ac, zrl, ff = set(), set(), False, 0
    for kind in CONTENT:
        for C, q in ((3, 100), (1, 100), (3, 10)):
            img = R.content(kind, 5, C, 64, 64)
            for c in R.coefficients(img, q):
                blk = c.reshape(-1, 64)[:, R.ZIGZAG]
                cats_ac |= {int(np.abs(v)).bit_length() for v in blk[:, 1:].ravel()}
                dc = blk[:, 0]
                cats_dc |= {int(abs(v)).bit_length() for v in np.diff(np.concatenate([[0], dc]))}
                for row in blk:
                    nz = np.nonzero(row[1:])[0]
                    if len(nz) and (np.diff(np.concatenate([[-1], nz])) > 16).any():
                        zrl = True
            ff += R.encode(img, q)[len(R.header(C, 64, 64, q)):].count(b"\xff\x00")
    assert 11 in cats_dc and 10 in cats_ac and zrl and ff > 100, (sorted(cats_dc), sorted(cats_ac), zrl, ff)


@pytest.mark.parametrize("C", [1, 3])
def test_header_equals_pillow(C):
    for q in (1, 25, 75, 100):
        b = pillow_bytes(np.zeros((C, 5, 7), np.uint8), q)
        assert b.startswith(R.header(C, 5, 7, q))


def test_golden_npz_equals_reference():
    """Every golden case: the reference's file has the SHA-256 of Pillow's, and the stored files are those bytes."""
    with np.load(GOLDEN) as z:
        g = {k: z[k] for k in z.files}
    assert len(g["kind"]) >= 1000
    files = {}
    for i in range(len(g["kind"])):
        img = R.content(str(g["kind"][i]), int(g["seed"][i]), int(g["C"][i]), int(g["H"][i]), int(g["W"][i]))
        files[i] = R.encode(img, int(g["quality"][i]))
        assert hashlib.sha256(files[i]).hexdigest() == str(g["file_sha256"][i]), i
    for k, i in enumerate(g["full_idx"]):
        assert g["full_data"][g["full_offsets"][k]:g["full_offsets"][k + 1]].tobytes() == files[int(i)]


def test_hash_inputs_are_fixed():
    """The golden inputs do not depend on the machine: the first words of the hash and one face are pinned."""
    assert R.hash_u32(0, 4).tolist() == [3793791033, 2433363436, 2539140574, 487265508]
    assert hashlib.sha256(R.content("face", 11, 3, 20, 24).tobytes()).hexdigest()[:16] == "432f7be302180460"
