"""GPU: fg_dataset_upload_jpeg decodes the JPEG corpus bit for bit as Pillow (libjpeg-turbo, default decompression)
does, across chunks, table sets, row offsets and refusals; a cache it fills trains exactly like one filled from the
decoded arrays; DeviceDataset.from_dirs over a directory gives the same cache."""
import numpy as np
import pytest

import jpeg_utils as JU
import parity_utils as PU

pytestmark = pytest.mark.gpu
FG_ERR_INVALID, FG_ERR_UNSUPPORTED = -1, -4


@pytest.fixture(scope="module")
def ctx():
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=16, channels=3)
    yield c
    c.close()


@pytest.fixture(scope="module")
def gray_ctx():
    import face_generator_b200 as fg
    c = fg.Context(0, max_batch=16, channels=1)
    yield c
    c.close()


def cache(ctx, N, Cs, H, W):
    from face_generator_b200.dataset import DeviceDataset
    return DeviceDataset(ctx, shape=(N, Cs, H, W))


def test_every_corpus_file_equals_pillow(ctx, gray_ctx):
    corpus = [e for e in JU.load() if e.supported]
    assert len(corpus) > 60
    for e in corpus:
        for Cs in ((3, 1) if e.C == 1 else (3,)):
            ds = cache(ctx if Cs == 3 else gray_ctx, 3, Cs, e.H, e.W)
            ds.upload_jpeg(1, [e.bytes])
            bad = e.mismatch(ds.download(1, 1)[0])
            assert bad is None, "%s Cs=%d: %s" % (e.name, Cs, bad)
            ds.close()


def mixed_64(corpus, n, rng):
    """n files drawn from every 64x64 corpus file: several qualities, subsamplings, optimised tables (one table set
    per file), restart intervals, grayscale and extra segments."""
    pool = [e for e in corpus if e.supported and (e.H, e.W) == (64, 64)]
    assert len({e.name.split("_")[0] for e in pool}) >= 5
    pick = rng.integers(0, len(pool), n)
    return [pool[i] for i in pick]


def test_many_chunks_equal_per_file_calls_and_land_at_first(ctx):
    rng = np.random.default_rng(7)
    files = mixed_64(JU.load(), 20000, rng)
    first = 37
    ds = cache(ctx, first + len(files) + 5, 3, 64, 64)
    ds.upload(0, np.full((first, 3, 64, 64), 11, np.uint8))
    ds.upload(first + len(files), np.full((5, 3, 64, 64), 13, np.uint8))
    ds.upload_jpeg(first, [e.bytes for e in files])  # spans several internal chunks
    got = ds.download()
    assert (got[:first] == 11).all() and (got[first + len(files):] == 13).all()
    for i, e in enumerate(files):
        bad = e.mismatch(got[first + i])
        assert bad is None, "row %d (%s): %s" % (first + i, e.name, bad)
    # per-file calls on a sample of the same files, into a second cache
    one = cache(ctx, 1, 3, 64, 64)
    for i in rng.choice(len(files), 64, replace=False):
        one.upload_jpeg(0, [files[i].bytes])
        np.testing.assert_array_equal(one.download()[0], got[first + i])
    one.close()
    ds.close()


def test_refusals_report_the_file_and_leave_the_context_usable(ctx):
    from face_generator_b200.lib import FGError
    corpus = JU.load()
    good = [e for e in corpus if e.face]
    refusals = [e for e in corpus if not e.supported]
    assert {e.name for e in refusals} >= {"refuse_progressive", "refuse_cmyk", "refuse_truncated",
                                          "refuse_corrupt_huffman", "refuse_wrong_size"}
    for e in refusals:
        H, W = e.cache_hw
        for pos, n in ((0, 1), (5, 8)):
            files = [g.bytes for g in good[:n]]
            files[pos] = e.bytes
            ds = cache(ctx, n, 3, H, W)
            with pytest.raises(FGError) as ex:
                ds.upload_jpeg(0, files)
            assert ex.value.rc == e.upload_rc and ex.value.index == pos, (e.name, pos, str(ex.value))
            ok = [g.bytes for g in good[:n]]
            ds.upload_jpeg(0, ok)  # the context and the dataset still work
            np.testing.assert_array_equal(ds.download(), np.stack([g.expected(3) for g in good[:n]]))
            ds.close()


def test_colour_file_refused_by_a_one_channel_cache(gray_ctx):
    from face_generator_b200.lib import FGError
    corpus = JU.load()
    good = [e for e in corpus if e.face]
    ds = cache(gray_ctx, 2, 1, 64, 64)
    with pytest.raises(FGError) as ex:
        ds.upload_jpeg(0, [next(e for e in corpus if e.name == "gray_64x64").bytes, good[0].bytes])
    assert ex.value.index == 1 and ex.value.rc == FG_ERR_INVALID
    ds.close()


def test_lowest_failing_index_across_chunks(ctx):
    """Two corrupt files in different internal chunks (8192 files each): the lower index is reported."""
    from face_generator_b200.lib import FGError
    corpus = JU.load()
    good = next(e for e in corpus if e.face)
    bad = next(e for e in corpus if e.name == "refuse_corrupt_huffman")
    files = [good.bytes] * 12000
    files[11000] = bad.bytes
    files[5000] = bad.bytes
    ds = cache(ctx, len(files), 3, 64, 64)
    with pytest.raises(FGError) as ex:
        ds.upload_jpeg(0, files)
    assert ex.value.index == 5000
    ds.close()


def test_train_step_on_jpeg_cache_equals_upload_cache():
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    B, C, seed = 16, 3, 5
    faces = [e for e in JU.load() if e.face]  # the files whose decoded pixels the corpus keeps
    files = [faces[i] for i in np.random.default_rng(11).integers(0, len(faces), 300)]
    arrays = np.stack([e.expected(3) for e in files])
    case = PU.make_case(B, C, seed=31, init="smooth")
    hyper = fg.hyper_default()
    res = []
    for mode in ("jpeg", "arrays"):
        c = fg.Context(0, max_batch=B, channels=C)
        c.set_params(NET_G, case["PG"])
        c.set_params(NET_D, case["PD"])
        if mode == "jpeg":
            ds = DeviceDataset(c, shape=arrays.shape)
            ds.upload_jpeg(0, [e.bytes for e in files])
        else:
            ds = DeviceDataset(c, arrays)
        st = [ds.train_step(hyper, B, seed + k) for k in range(2)]
        res.append((st, ds.download(), c.get_params(NET_G), c.get_params(NET_D)))
        ds.close()
        c.close()
    (s1, d1, g1, D1), (s2, d2, g2, D2) = res
    np.testing.assert_array_equal(d1, d2)
    assert s1 == s2
    np.testing.assert_array_equal(g1, g2)
    np.testing.assert_array_equal(D1, D2)


def test_from_dirs_equals_per_file_path(ctx, gray_ctx, tmp_path):
    from face_generator_b200.dataset import DeviceDataset, list_image_files
    corpus = JU.load()
    files = mixed_64(corpus, 50, np.random.default_rng(3))
    for k, e in enumerate(files):
        (tmp_path / ("%s" % ("a" if k % 2 else "b"))).mkdir(exist_ok=True)
        (tmp_path / ("a" if k % 2 else "b") / ("img%03d.jpg" % k)).write_bytes(e.bytes)
    dirs = [str(tmp_path / "b"), str(tmp_path / "a")]
    ds = DeviceDataset.from_dirs(ctx, dirs, start_at=4, count=30, chunk=7)
    order = list_image_files(dirs, "jpg", 4, 30)
    assert ds.shape == (30, 3, 64, 64)
    one = cache(ctx, 1, 3, 64, 64)
    got = ds.download()
    for i, path in enumerate(order):
        with open(path, "rb") as f:
            one.upload_jpeg(0, [f.read()])
        np.testing.assert_array_equal(got[i], one.download()[0], err_msg=path)
    one.close()
    ds.close()
    # the lfwcrop_grey form: binary PGM, uploaded as decoded images; a gray context keeps one plane
    rng = np.random.default_rng(9)
    imgs = rng.integers(0, 256, (6, 1, 20, 17), dtype=np.uint8)
    (tmp_path / "pgm").mkdir()
    for k, im in enumerate(imgs):
        (tmp_path / "pgm" / ("f%d.pgm" % k)).write_bytes(b"P5\n17 20\n255\n" + im.tobytes())
    ds = DeviceDataset.from_dirs(gray_ctx, [str(tmp_path / "pgm")], ext="pgm")
    np.testing.assert_array_equal(ds.download(), imgs)
    ds.close()
