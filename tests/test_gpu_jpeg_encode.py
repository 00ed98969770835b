"""GPU: fg_dataset_encode_jpeg writes Pillow's files byte for byte and fg_dataset_jpeg_roundtrip gives Pillow's decode
of them, on every case of tests/golden/jpeg_encode.npz; on 20 000 rows over several chunks the two paths agree
(upload_jpeg(encode_jpeg(rows)) == jpeg_roundtrip(rows)) and rows outside the span stay as they were; the size
query, a short buffer and every refusal write and launch nothing; from_lfw(jpeg_quality=75), save_jpeg and from_dirs
agree.  Reads only the npz (no Pillow)."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import jpeg_enc_ref as R

pytestmark = pytest.mark.gpu
FG_ERR_INVALID = -1
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "jpeg_encode.npz")
LFW = os.path.join(HERE, "golden", "lfw_aug.npz")


def sha(b):
    return hashlib.sha256(b).hexdigest()


@pytest.fixture(scope="module")
def ctxs():
    import face_generator_b200 as fg
    c3, c1 = fg.Context(0, max_batch=16, channels=3), fg.Context(0, max_batch=16, channels=1)
    yield {3: c3, 1: c1}
    c3.close()
    c1.close()


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def test_golden_cases_equal_pillow(ctxs, golden):
    from face_generator_b200.dataset import DeviceDataset
    g = golden
    groups = {}
    for i in range(len(g["kind"])):
        groups.setdefault((int(g["C"][i]), int(g["H"][i]), int(g["W"][i]), int(g["quality"][i])), []).append(i)
    files = {}
    for (Cs, H, W, q), idx in groups.items():
        rows = np.stack([R.content(str(g["kind"][i]), int(g["seed"][i]), Cs, H, W) for i in idx])
        ds = DeviceDataset(ctxs[Cs], rows)
        got = ds.encode_jpeg(quality=q)
        ds.jpeg_roundtrip(quality=q)
        dec = ds.download()
        ds.close()
        for k, i in enumerate(idx):
            files[i] = got[k]
            assert sha(got[k]) == str(g["file_sha256"][i]), (str(g["kind"][i]), Cs, H, W, q)
            assert sha(dec[k].tobytes()) == str(g["decode_sha256"][i]), (str(g["kind"][i]), Cs, H, W, q)
    for k, i in enumerate(g["full_idx"]):
        assert files[int(i)] == g["full_data"][g["full_offsets"][k]:g["full_offsets"][k + 1]].tobytes()


@pytest.mark.parametrize("Cs,H,W,q", [(3, 17, 4096, 90), (1, 4096, 9, 30), (3, 4096, 4, 75)])
def test_sizes_past_the_band_budget_equal_reference(ctxs, Cs, H, W, q):
    """Rows whose single MCU row needs more than 48 KB of shared memory, and the decoder's largest size."""
    from face_generator_b200.dataset import DeviceDataset
    rows = np.stack([R.content(k, 3 + H + W, Cs, H, W) for k in ("noise", "gradient")])
    ds = DeviceDataset(ctxs[Cs], rows)
    got = ds.encode_jpeg(quality=q)
    ds.close()
    for k in range(len(rows)):
        assert got[k] == R.encode(rows[k], q), k


def mixed_rows(n):
    """n 3x64x64 rows: 160 distinct hashed images of every kind, each repeated, in a hashed order."""
    base = np.stack([R.content(R.KINDS[k % len(R.KINDS)], 900 + k, 3, 64, 64) for k in range(160)])
    order = R.hash_u32(77, n) % len(base)
    return base[order]


def test_paths_agree_over_many_chunks(ctxs):
    from face_generator_b200.dataset import DeviceDataset
    n, first = 20000, 7
    rows = mixed_rows(n)
    src = DeviceDataset(ctxs[3], shape=(first + n + 3, 3, 64, 64))
    src.upload(0, np.full((first, 3, 64, 64), 11, np.uint8))
    src.upload(first, rows)
    src.upload(first + n, np.full((3, 3, 64, 64), 13, np.uint8))
    files = src.encode_jpeg(first, n, 75)
    assert len(files) == n
    for k in (0, 1, 4999, n - 1):
        assert files[k] == R.encode(rows[k], 75), k
    one_calls = R.hash_u32(78, 24) % n
    for k in one_calls:
        assert src.encode_jpeg(first + int(k), 1, 75)[0] == files[k], k
    dec = DeviceDataset(ctxs[3], shape=(n, 3, 64, 64))
    dec.upload_jpeg(0, files)
    via_files = dec.download()
    dec.close()
    src.jpeg_roundtrip(first, n, 75)
    got = src.download()
    src.close()
    assert (got[:first] == 11).all() and (got[first + n:] == 13).all()
    bad = np.nonzero((got[first:first + n] != via_files).reshape(n, -1).any(1))[0]
    assert not len(bad), "rows %s differ" % bad[:8].tolist()


def test_size_query_short_buffer_and_refusals(ctxs):
    from face_generator_b200.dataset import DeviceDataset
    ctx = ctxs[3]
    lib = ctx.lib
    rows = mixed_rows(40)
    ds = DeviceDataset(ctx, rows)
    want = ds.encode_jpeg(0, 40, 50)
    sizes = np.cumsum([0] + [len(b) for b in want])
    offsets = np.full(41, -5, np.int64)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.fg_dataset_encode_jpeg(ds.h, 0, 40, 50, None, 0, P(offsets)) == 0
    np.testing.assert_array_equal(offsets, sizes)
    out = np.full(int(sizes[-1]), 0xA5, np.uint8)
    offsets[:] = -5
    assert lib.fg_dataset_encode_jpeg(ds.h, 0, 40, 50, P(out), int(sizes[-1]) - 1, P(offsets)) == FG_ERR_INVALID
    np.testing.assert_array_equal(offsets, sizes)
    assert (out == 0xA5).all()
    before = ctx.launches()
    for args in ((0, 40, 0), (0, 40, 101), (1, 40, 75), (-1, 2, 75), (0, 0, 75), (40, 1, 75)):
        assert lib.fg_dataset_encode_jpeg(ds.h, *args, P(out), out.size, P(offsets)) == FG_ERR_INVALID, args
        assert lib.fg_dataset_jpeg_roundtrip(ds.h, *args) == FG_ERR_INVALID, args
    assert lib.fg_dataset_encode_jpeg(ds.h, 0, 40, 75, P(out), out.size, None) == FG_ERR_INVALID
    assert ctx.launches() == before
    assert (out == 0xA5).all()
    np.testing.assert_array_equal(ds.download(), rows)
    assert lib.fg_dataset_encode_jpeg(ds.h, 0, 40, 50, P(out), out.size, P(offsets)) == 0
    assert out.tobytes() == b"".join(want)
    ds.close()


def lfw_tree(tmp_path):
    g = dict(np.load(LFW))
    root = tmp_path / "lfw"
    for k, name in enumerate(g["names"]):
        (root / os.path.dirname(str(name))).mkdir(parents=True, exist_ok=True)
        (root / str(name)).write_bytes(g["jpegs"][g["offsets"][k]:g["offsets"][k + 1]].tobytes())
    return str(root)


def test_from_lfw_save_jpeg_and_read_back(ctxs, tmp_path):
    from face_generator_b200.dataset import DeviceDataset
    ctx = ctxs[3]
    root = lfw_tree(tmp_path)
    ds = DeviceDataset.from_lfw(ctx, [root], augmentations=2, jpeg_quality=75)
    rows = ds.download()
    ds.close()
    plain = DeviceDataset.from_lfw(ctx, [root], augmentations=2)
    assert (plain.download() != rows).any()
    # the files generate_dataset.py writes: named {i:06}_{a:03}.jpg, decoding to the jpeg_quality=75 rows
    out = tmp_path / "out_aug"
    plain.save_jpeg(str(out))
    P = len(rows) // 3
    assert sorted(os.listdir(out)) == ["%06d_%03d.jpg" % (i, a) for i in range(P) for a in range(3)]
    assert (out / "000001_002.jpg").read_bytes() == plain.encode_jpeg(5, 1)[0]
    back = DeviceDataset.from_dirs(ctx, [str(out)])
    np.testing.assert_array_equal(back.download(), rows)
    back.close()
    plain.jpeg_roundtrip(quality=75)
    np.testing.assert_array_equal(plain.download(), rows)
    plain.close()
