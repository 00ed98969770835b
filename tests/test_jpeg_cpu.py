"""CPU: fg_jpeg_info on the JPEG corpus (host only, no GPU), the file list of DeviceDataset.from_dirs against
dataset.lua:156-190 loadImagesFromDirs, and the binary PGM reader of the ext="pgm" path."""
import os

import numpy as np
import pytest

import jpeg_utils as JU

FG_ERR_INVALID, FG_ERR_UNSUPPORTED = -1, -4


def test_corpus_covers_the_supported_scope():
    corpus = JU.load()
    names = {e.name for e in corpus}
    for must in ("refuse_progressive", "refuse_cmyk", "refuse_truncated", "refuse_corrupt_huffman", "refuse_wrong_size",
                 "restart_blocks3_420", "restart_rows1_422", "optimize_420", "gray_64x64", "segments_exif_icc_comment",
                 "size1x1_420", "size7x13_422", "size17x33_444", "size61x47_420", "size100x75_420", "size255x255_420"):
        assert must in names, must
    for q in (10, 50, 75, 95, 100):
        assert {"q%d_face_%s" % (q, s) for s in ("444", "422", "420")} <= names
    faces = [e for e in corpus if e.face]
    assert len(faces) >= 4 and all((e.C, e.H, e.W) == (3, 64, 64) for e in faces)
    for e in corpus:
        assert (len(e.sha256) == 64) == e.supported, e.name
        if e.face:
            assert e.decoded.shape == (3, 64, 64) and e.decoded.dtype == np.uint8
            assert e.mismatch(e.decoded) is None and e.mismatch(e.decoded[::-1]) is not None
    assert os.path.getsize(JU.CORPUS) < 300 << 10


def test_jpeg_info_matches_every_corpus_file():
    import face_generator_b200.dataset as D
    from face_generator_b200.lib import FGError, load_library
    lib = load_library()
    for e in JU.load():
        if e.info_rc == 0:
            assert D.jpeg_info(e.bytes) == (e.C, e.H, e.W), e.name
        else:
            with pytest.raises(FGError) as ex:
                D.jpeg_info(e.bytes)
            assert "(%d)" % e.info_rc in str(ex.value), (e.name, str(ex.value))
            assert ("progressive" if "progressive" in e.name else "4 components") in lib.fg_last_error().decode()


def test_jpeg_info_refuses_malformed_headers():
    import face_generator_b200.dataset as D
    from face_generator_b200.lib import FGError
    good = next(e for e in JU.load() if e.face).bytes
    sos = good.index(b"\xff\xda")
    cases = {
        b"": FG_ERR_INVALID,                                 # no SOI
        b"\x89PNG\r\n\x1a\n" + b"\0" * 16: FG_ERR_INVALID,   # another format
        good[:sos]: FG_ERR_INVALID,                          # header cut before the scan
        good[:40]: FG_ERR_INVALID,                           # cut inside a segment
        good.replace(b"\xff\xc0", b"\xff\xc2", 1): FG_ERR_UNSUPPORTED,   # SOF2: progressive
        good.replace(b"\xff\xc0", b"\xff\xc9", 1): FG_ERR_UNSUPPORTED,   # SOF9: arithmetic coding
    }
    sof = good.index(b"\xff\xc0")
    twelve = bytearray(good)
    twelve[sof + 4] = 12                                     # P = 12: 12-bit samples
    cases[bytes(twelve)] = FG_ERR_UNSUPPORTED
    odd = bytearray(good)
    odd[sof + 4 + 6 + 1] = 0x12                              # luma sampling 1x2
    cases[bytes(odd)] = FG_ERR_UNSUPPORTED
    for data, rc in cases.items():
        with pytest.raises(FGError) as ex:
            D.jpeg_info(data)
        assert "(%d)" % rc in str(ex.value), (data[:8], str(ex.value))


def lua_load_images_from_dirs(dirs, ext, start_at, count):
    """A literal transcription of dataset.lua:156-190 (file list only): paths.files order is irrelevant because
    doSort is true; file:find(ext .. '$') on a plain extension is a suffix test; table.sort with a < b compares the
    full paths byte by byte; then files[startAt .. min(startAt+count-1, #files)]."""
    files = []
    for d in dirs:
        for f in os.listdir(d):
            if f.endswith(ext):
                files.append(d.rstrip("/") + "/" + f)
        if len(files) == 0:
            raise FileNotFoundError(ext)
    files.sort(key=lambda p: p.encode())
    end_at = min(start_at + count - 1, len(files))
    return [files[i - 1] for i in range(start_at, end_at + 1)]


def test_from_dirs_file_order_and_slicing(tmp_path):
    from face_generator_b200.dataset import list_image_files
    face = next(e for e in JU.load() if e.face).bytes
    d1, d2 = tmp_path / "b_dir", tmp_path / "a_dir"
    d1.mkdir()
    d2.mkdir()
    names1 = ["img10.jpg", "img2.jpg", "Img3.jpg", "_x.jpg", "z.JPG", "notes.txt", "c.jpeg", "a b.jpg", "été.jpg"]
    names2 = ["img1.jpg", "img10.jpg", "0.jpg", "jpg"]
    for d, names in ((d1, names1), (d2, names2)):
        for n in names:
            (d / n).write_bytes(face)
    dirs = [str(d1), str(d2)]
    full = lua_load_images_from_dirs(dirs, "jpg", 1, 10 ** 9)
    assert len(full) == 10  # "jpg" itself ends in jpg, as in the reference
    assert list_image_files(dirs, "jpg") == full
    for start_at, count in ((1, 3), (2, 5), (4, 100), (10, 1), (11, 4), (1, 0)):
        assert list_image_files(dirs, "jpg", start_at, count) == lua_load_images_from_dirs(dirs, "jpg", start_at, count)
    with pytest.raises(FileNotFoundError):
        list_image_files([str(tmp_path)], "jpg")


def test_pgm_reader():
    from face_generator_b200.dataset import read_pgm
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (13, 7), dtype=np.uint8)
    for header in (b"P5\n7 13\n255\n", b"P5 7 13 255 ", b"P5\n# lfwcrop\n7\t13\n# maxval\n255\n"):
        np.testing.assert_array_equal(read_pgm(header + img.tobytes()), img[None])
    with pytest.raises(ValueError):
        read_pgm(b"P2\n7 13\n255\n" + img.tobytes())      # ASCII PGM
    with pytest.raises(ValueError):
        read_pgm(b"P5\n7 13\n255\n" + img.tobytes()[:-1])  # truncated
    with pytest.raises(ValueError):
        read_pgm(b"P5\n7 13\n65535\n" + img.tobytes() * 2)  # 16-bit
