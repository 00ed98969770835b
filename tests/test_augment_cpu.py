"""CPU: the pieces of the LFW augmentation that need no GPU.  aug_ref's restatement of Pillow's BILINEAR resize equals
Pillow bit for bit; fg_lfw_aug_params draws generate_dataset.py's distributions, reproducibly and independently of
slicing, with the inverse maps np.linalg.inv gives; list_lfw_files walks like generate_dataset.py; the golden rows are
what aug_ref computes from the golden photos."""
import hashlib
import os

import numpy as np
import pytest

import aug_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lfw_aug.npz")


def images(kind, C, rng):
    if kind == "random":
        return rng.integers(0, 256, (C, 84, 84), dtype=np.uint8)
    if kind == "smooth":
        y, x = np.mgrid[0:84, 0:84]
        ph = rng.uniform(0, 6.3, (C, 1, 1))
        return (127.5 + 127.5 * np.sin(x / 9.0 + ph) * np.cos(y / 13.0 - ph)).astype(np.uint8)
    # saturated: large flat regions at 0 and 255 with hard edges, the clip of both passes
    img = np.where(rng.random((C, 12, 12)) < 0.5, 0, 255).astype(np.uint8)
    return np.repeat(np.repeat(img, 7, axis=1), 7, axis=2)


@pytest.mark.parametrize("Ho,Wo", [(64, 64), (32, 32), (32, 48), (48, 32)])
@pytest.mark.parametrize("kind", ["random", "smooth", "saturated"])
@pytest.mark.parametrize("C", [3, 1])
def test_resize_restatement_equals_pillow(Ho, Wo, kind, C):
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(Ho * 1000 + Wo + C)
    for _ in range(8):
        img = images(kind, C, rng)
        pil = Image.fromarray(img.transpose(1, 2, 0) if C == 3 else img[0], "RGB" if C == 3 else "L")
        want = np.asarray(pil.resize((Wo, Ho), Image.BILINEAR))
        want = want.transpose(2, 0, 1) if C == 3 else want[None]
        np.testing.assert_array_equal(R.pillow_resize(img, Ho, Wo), want)


def test_params_deterministic_and_slice_independent():
    from face_generator_b200.dataset import lfw_aug_params
    a = lfw_aug_params(43, 0, 40, 19, 250, 250)
    np.testing.assert_array_equal(a, lfw_aug_params(43, 0, 40, 19, 250, 250))
    for first, n in ((0, 7), (7, 13), (20, 20)):
        np.testing.assert_array_equal(lfw_aug_params(43, first, n, 19, 250, 250), a[first * 20:(first + n) * 20])
    assert not np.array_equal(lfw_aug_params(44, 0, 40, 19, 250, 250)["m"], a["m"])
    np.testing.assert_array_equal(a["src"], np.repeat(np.arange(40), 20))


def test_params_follow_generate_dataset_distributions():
    from face_generator_b200.dataset import lfw_aug_params
    n_src, n_aug, H, W = 200, 19, 250, 250
    a = lfw_aug_params(43, 1000, n_src, n_aug, H, W).reshape(n_src, 1 + n_aug)
    row0 = a[:, 0]
    assert (row0["warp"] == 0).all() and (row0["hflip"] == 0).all() and (row0["brightness"] == 1.0).all()
    np.testing.assert_array_equal(row0["m"], np.tile(np.eye(3).ravel(), (n_src, 1)))
    aug = a[:, 1:].ravel()
    assert (aug["warp"] == 1).all()
    np.testing.assert_array_equal(aug["m"][:, 6:], np.tile([0.0, 0.0, 1.0], (aug.size, 1)))  # exactly
    assert ((aug["brightness"] >= 0.9) & (aug["brightness"] < 1.1)).all()
    assert abs(aug["hflip"].mean() - 0.5) < 0.03  # 3800 draws: 0.03 is ~3.7 sigma
    degs, txs, tys = set(), set(), set()
    for k, d in enumerate(aug):
        i, j = 1000 + k // n_aug, 1 + k % n_aug
        p = R.draws(43, i, j)
        assert 0.82 <= p["scale"] < 1.10 and -8 <= p["deg"] <= 8 and -5 <= p["tx"] <= 5 and -5 <= p["ty"] <= 5
        assert d["hflip"] == p["hflip"] and d["brightness"] == p["brightness"] and d["src"] == i
        F = R.forward_matrix(p["scale"], p["deg"], p["tx"], p["ty"], H, W)
        assert np.abs(np.linalg.inv(F).ravel() - d["m"]).max() < 1e-12, (i, j)
        degs.add(p["deg"])
        txs.add(p["tx"])
        tys.add(p["ty"])
    assert degs == set(range(-8, 9)) and txs == set(range(-5, 6)) and tys == set(range(-5, 6))


def test_params_shift_follows_the_width_height_swap():
    """augment() passes shape[0] (the height) as the width: on a 200 x 250 photo the rotation centre is
    (x, y) = (100, 125), so the inverse map fixes that point when the translation is 0."""
    from face_generator_b200.dataset import lfw_aug_params
    a = lfw_aug_params(43, 0, 400, 1, 200, 250)[1::2]
    for k, d in enumerate(a):
        p = R.draws(43, k, 1)
        if p["tx"] == 0 and p["ty"] == 0:
            m = d["m"].reshape(3, 3)
            np.testing.assert_allclose(m @ [100.0, 125.0, 1.0], [100.0, 125.0, 1.0], atol=1e-9)
            return
    pytest.fail("no draw with zero translation")


def test_params_refusals():
    from face_generator_b200.lib import load_library
    lib = load_library()
    out = np.zeros(4, R.AUG_DTYPE)
    for args in ((43, -1, 1, 1, 250, 250), (43, 0, 0, 1, 250, 250), (43, 0, 1, -1, 250, 250), (43, 0, 1, 1, 0, 250)):
        assert lib.fg_lfw_aug_params(*args, out.ctypes.data) == -1
    assert b"fg_lfw_aug_params" in lib.fg_last_error()
    assert lib.fg_lfw_aug_params(43, 0, 1, 1, 250, 250, None) == -1


def test_list_lfw_files(tmp_path):
    from face_generator_b200.dataset import list_lfw_files
    root = tmp_path / "lfw"
    (root / "Bob_B" / "deeper").mkdir(parents=True)
    (root / "Al_A").mkdir()
    (root / "a_lower").mkdir()
    for p in ("top.jpg", "Bob_B/Bob_B_0002.jpg", "Bob_B/Bob_B_0001.jpg", "Al_A/Al_A_0001.jpg", "a_lower/x.jpg",
              "Bob_B/deeper/too_deep.jpg", "Bob_B/notes.txt", "Al_A/pic.JPG", "Al_A/pic.jpeg", "Al_A/pic.jpg.png"):
        (root / p).write_bytes(b"x")
    (root / "dir.jpg").mkdir()
    got = list_lfw_files([str(root)])
    want = ["Al_A/Al_A_0001.jpg", "Bob_B/Bob_B_0001.jpg", "Bob_B/Bob_B_0002.jpg", "a_lower/x.jpg", "top.jpg"]
    assert got == [os.path.join(str(root), p) for p in want]  # byte order: upper case before lower case
    assert list_lfw_files([str(root / "Al_A")]) == [os.path.join(str(root), "Al_A", "Al_A_0001.jpg")]


def pillow_photos(g):
    Image = pytest.importorskip("PIL.Image")
    import io
    return np.stack([np.asarray(Image.open(io.BytesIO(g["jpegs"][g["offsets"][k]:g["offsets"][k + 1]].tobytes()))
                                .convert("RGB")).transpose(2, 0, 1) for k in range(len(g["names"]))])


def test_golden_photos_are_pillow_decodes():
    g = np.load(GOLDEN)
    for k, p in enumerate(pillow_photos(g)):
        assert hashlib.sha256(np.ascontiguousarray(p).tobytes()).hexdigest() == str(g["photo_sha256"][k]), k


def test_golden_rows_are_aug_ref_of_the_golden_photos():
    from face_generator_b200.dataset import lfw_aug_params
    g = np.load(GOLDEN)
    photos = pillow_photos(g)
    augs = lfw_aug_params(int(g["seed"]), 0, len(photos), int(g["n_aug"]), 250, 250)
    np.testing.assert_array_equal(augs, g["augs"])
    rows = R.augment_rows(photos, augs)
    for k, r in enumerate(rows):
        assert hashlib.sha256(r.tobytes()).hexdigest() == str(g["sha256"][k]), k
    np.testing.assert_array_equal(rows[g["full_idx"]], g["full_rows"])


def test_identity_warp_loses_levels():
    """Step 3 is lossy even at the identity: (uint8)((k * (1/255)) * 255) maps 24 of the 256 levels to k - 1, so an
    augmented row never equals the unaugmented crop of the same photo."""
    ramp = np.arange(256, dtype=np.uint8)
    src = np.zeros((1, 250, 250), np.uint8)
    src[0, 92:176, 83:167] = np.resize(ramp, (84, 84))
    d = R.identity_desc(0)
    d["warp"] = 1
    got = R.warp_crop(src, d)
    lost = got[0] != R.crop(src)[0]
    lost_levels = set(R.crop(src)[0][lost].tolist())
    assert len(lost_levels) == 24
    assert all(v - 1 == int(np.uint8(v * (1.0 / 255.0) * 255)) for v in lost_levels)
