"""GPU: fg_dataset_augment builds every row bit for bit as tests/aug_ref.py does, on generated and hand-made
descriptors (cval, the keep-zero rule, large rotations and scales, a projective map, integer sample points, the lossy
identity warp, both brightness clips, flat regions at the source minimum); one large call equals the reference and
one-row calls; DeviceDataset.from_lfw over an LFW-style tree gives the golden rows whatever the chunking; a cache it
builds trains like one uploaded from the same pixels; every refusal launches nothing and leaves the context usable."""
import hashlib
import os

import numpy as np
import pytest

import aug_ref as R

pytestmark = pytest.mark.gpu
FG_ERR_INVALID = -1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lfw_aug.npz")


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


@pytest.fixture(scope="module")
def golden(ctx):
    """The golden npz and its photos decoded on the GPU, checked against the SHA-256 of Pillow's decodes."""
    from face_generator_b200.dataset import DeviceDataset
    g = dict(np.load(GOLDEN))
    blobs = [g["jpegs"][g["offsets"][k]:g["offsets"][k + 1]].tobytes() for k in range(len(g["names"]))]
    ds = DeviceDataset(ctx, shape=(len(blobs), 3, 250, 250))
    ds.upload_jpeg(0, blobs)
    photos = ds.download()
    ds.close()
    for k, p in enumerate(photos):
        assert hashlib.sha256(p.tobytes()).hexdigest() == str(g["photo_sha256"][k]), k
    g["blobs"], g["photos"] = blobs, photos
    return g


def synthetic(rng, n, C=3):
    """Sources beyond the golden faces: random noise, smooth fields with a raised minimum, saturated blocks."""
    out = []
    y, x = np.mgrid[0:250, 0:250]
    for k in range(n):
        if k % 3 == 0:
            img = rng.integers(0, 256, (C, 250, 250), dtype=np.uint8)
        elif k % 3 == 1:
            ph = rng.uniform(0, 6.3, (C, 1, 1))
            img = (140 + 100 * np.sin(x / 17.0 + ph) * np.cos(y / 11.0 - ph)).astype(np.uint8)
        else:
            img = np.repeat(np.repeat(np.where(rng.random((C, 25, 25)) < 0.5, 0, 255), 10, 1), 10, 2).astype(np.uint8)
        out.append(img)
    return np.stack(out)


def run(ctx, srcs, augs, Ho=64, Wo=64, first=0, extra=0):
    from face_generator_b200.dataset import DeviceDataset
    src = DeviceDataset(ctx, srcs)
    dst = DeviceDataset(ctx, shape=(first + len(augs) + extra, srcs.shape[1], Ho, Wo))
    dst.augment(src, first, augs)
    got = dst.download(first, len(augs))
    src.close()
    dst.close()
    return got


def mismatch(got, want):
    bad = np.nonzero((got != want).reshape(len(got), -1).any(1))[0]
    return None if not len(bad) else "rows %s differ (first: %d pixels)" % (bad[:8].tolist(), (got[bad[0]] != want[bad[0]]).sum())


@pytest.mark.parametrize("Ho,Wo", [(64, 64), (32, 48)])
def test_generated_params_equal_aug_ref(ctx, gray_ctx, golden, Ho, Wo):
    from face_generator_b200.dataset import lfw_aug_params
    srcs = np.concatenate([golden["photos"], synthetic(np.random.default_rng(5), 6)])
    augs = lfw_aug_params(43, 0, len(srcs), 5, 250, 250)
    for c, s in ((ctx, srcs), (gray_ctx, np.ascontiguousarray(srcs[:, 1:2]))):
        got = run(c, s, augs, Ho, Wo)
        assert mismatch(got, R.augment_rows(s, augs, Ho, Wo)) is None


def hand_made(n_src):
    """Descriptors that reach the paths the LFW draws never do."""
    descs = []

    def add(src, m, b=1.0, flip=0, warp=1):
        d = R.identity_desc(src)
        d["m"], d["brightness"], d["hflip"], d["warp"] = np.asarray(m, np.float64).ravel(), b, flip, warp
        descs.append(d)

    def about_centre(A, cx=125.0, cy=125.0):
        T = np.array([[1, 0, cx], [0, 1, cy], [0, 0, 1.0]])
        return np.linalg.inv(T @ A @ np.linalg.inv(T))

    def rot(deg, s=1.0):
        r = np.deg2rad(deg)
        return np.array([[s * np.cos(r), -s * np.sin(r), 0], [s * np.sin(r), s * np.cos(r), 0], [0, 0, 1.0]])

    for src in range(n_src):
        for flip in (0, 1):
            add(src, [[1, 0, -120], [0, 1, 0], [0, 0, 1]], flip=flip)       # crop half off the left edge: cval
            add(src, [[1, 0, 37.5], [0, 1, 110.25], [0, 0, 1]], flip=flip)  # off the bottom right, fractional
            add(src, about_centre(rot(45)), flip=flip)
            add(src, about_centre(rot(-30, 0.5)), b=0.95, flip=flip)
            add(src, about_centre(rot(12, 2.0)), b=1.05, flip=flip)
            add(src, [[1, 0.02, 3], [-0.01, 1, -4], [1e-4, -2e-4, 1.0]], flip=flip)  # projective
            add(src, [[1, 0, 0], [0, 1, 0], [2 ** -7, 0, -1.25]], flip=flip)  # z = 0 on column 160: not finite there
            add(src, [[1, 0, 3], [0, 1, -2], [0, 0, 1]], flip=flip)         # integer-aligned sample points
            add(src, np.eye(3), flip=flip)                                  # the identity warp
            add(src, about_centre(rot(5, 1.1)), b=0.0, flip=flip)           # brightness 0
            add(src, about_centre(rot(-7, 0.9)), b=1.1, flip=flip)          # saturates at 255
            add(src, np.eye(3), warp=0, b=0.3, flip=flip)                   # warp 0 ignores the rest
    return np.array(descs, R.AUG_DTYPE)


def flat_at_min(rng, C):
    """Large flat regions at the source minimum next to brighter texture: bilinear weights that undershoot the
    minimum by an ulp are clipped back to it."""
    img = np.full((C, 250, 250), 37, np.uint8)
    img[:, :, 125:] = rng.integers(37, 200, (C, 250, 125), dtype=np.uint8)
    img[:, 60:90, 40:200] = 250
    return img


@pytest.mark.parametrize("Ho,Wo", [(64, 64), (32, 48), (84, 84)])
def test_hand_made_descriptors_equal_aug_ref(ctx, gray_ctx, golden, Ho, Wo):
    rng = np.random.default_rng(17)
    srcs = np.concatenate([golden["photos"][[0, 5, 6]], synthetic(rng, 3), flat_at_min(rng, 3)[None]])
    augs = hand_made(len(srcs))
    for c, s in ((ctx, srcs), (gray_ctx, np.ascontiguousarray(srcs[:, :1]))):
        want = R.augment_rows(s, augs, Ho, Wo)
        got = run(c, s, augs, Ho, Wo)
        assert mismatch(got, want) is None
    # the paths these descriptors are meant to reach are reached
    full = R.augment_rows(srcs, augs, 84, 84)
    ident = [k for k, d in enumerate(augs) if d["warp"] and d["src"] < 3 and np.array_equal(d["m"], np.eye(3).ravel())]
    assert ident and all((full[k] != R.crop(srcs[augs[k]["src"]])).any() for k in ident)  # the 24 lost levels show
    assert (full[[k for k, d in enumerate(augs) if d["brightness"] == 0.0]] == 0).all()


def test_large_call_equals_reference_and_one_row_calls(ctx, golden):
    """One call of 20 000 rows at a nonzero first row: 1000 distinct descriptors, each used 20 times in a shuffled
    order, every row checked against the reference; a sample also against one-row calls."""
    from face_generator_b200.dataset import DeviceDataset, lfw_aug_params
    rng = np.random.default_rng(23)
    srcs = np.concatenate([golden["photos"], synthetic(rng, 42)])
    base = lfw_aug_params(99, 0, 50, 19, 250, 250)
    want_base = R.augment_rows(srcs, base)
    order = rng.permutation(np.tile(np.arange(len(base)), 20))
    augs = base[order]
    first = 13
    src = DeviceDataset(ctx, srcs)
    dst = DeviceDataset(ctx, shape=(first + len(augs) + 3, 3, 64, 64))
    dst.upload(0, np.full((first, 3, 64, 64), 11, np.uint8))
    dst.upload(first + len(augs), np.full((3, 3, 64, 64), 13, np.uint8))
    dst.augment(src, first, augs)
    got = dst.download()
    assert (got[:first] == 11).all() and (got[first + len(augs):] == 13).all()
    assert mismatch(got[first:first + len(augs)], want_base[order]) is None
    one = DeviceDataset(ctx, shape=(1, 3, 64, 64))
    for k in rng.choice(len(augs), 48, replace=False):
        one.augment(src, 0, augs[k:k + 1])
        np.testing.assert_array_equal(one.download()[0], got[first + k])
    one.close()
    src.close()
    dst.close()


def lfw_tree(tmp_path, golden):
    root = tmp_path / "lfw"
    for name, b in zip(golden["names"], golden["blobs"]):
        (root / os.path.dirname(str(name))).mkdir(parents=True, exist_ok=True)
        (root / str(name)).write_bytes(b)
    (root / "README.txt").write_bytes(b"not an image")
    return str(root)


def test_from_lfw_equals_golden_and_ignores_chunking(ctx, golden, tmp_path):
    from face_generator_b200.dataset import DeviceDataset
    root = lfw_tree(tmp_path, golden)
    P = len(golden["names"])
    ds = DeviceDataset.from_lfw(ctx, [root], augmentations=2)
    assert ds.shape == (P * 3, 3, 64, 64)
    rows = ds.download()
    ds.close()
    for k, r in enumerate(rows):
        assert hashlib.sha256(r.tobytes()).hexdigest() == str(golden["sha256"][k]), k
    np.testing.assert_array_equal(rows[golden["full_idx"]], golden["full_rows"])
    ds = DeviceDataset.from_lfw(ctx, [root], augmentations=2, chunk=3)
    np.testing.assert_array_equal(ds.download(), rows)
    ds.close()
    ds = DeviceDataset.from_lfw(ctx, [root], augmentations=0, chunk=5)  # out_unaug_64x64
    np.testing.assert_array_equal(ds.download(), rows[::3])
    ds.close()
    ds = DeviceDataset.from_lfw(ctx, [root], augmentations=2, seed=44)
    other = ds.download()
    ds.close()
    np.testing.assert_array_equal(other[::3], rows[::3])
    assert all((other[k] != rows[k]).any() for k in range(len(rows)) if k % 3)


def test_from_lfw_names_a_failing_file(ctx, golden, tmp_path):
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import FGError
    root = lfw_tree(tmp_path, golden)
    bad = os.path.join(root, str(golden["names"][3]))
    with open(bad, "r+b") as f:
        f.truncate(400)
    with pytest.raises(FGError) as ex:
        DeviceDataset.from_lfw(ctx, [root], augmentations=1, chunk=2)
    assert bad in str(ex.value)


def test_train_step_on_augmented_cache_equals_uploaded_cache(golden, tmp_path):
    import face_generator_b200 as fg
    import parity_utils as PU
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    B, C, seed = 16, 3, 5
    root = lfw_tree(tmp_path, golden)
    case = PU.make_case(B, C, seed=31, init="smooth")
    hyper = fg.hyper_default()
    res, pixels = [], None
    for mode in ("augment", "upload"):
        c = fg.Context(0, max_batch=B, channels=C)
        c.set_params(NET_G, case["PG"])
        c.set_params(NET_D, case["PD"])
        if mode == "augment":
            ds = DeviceDataset.from_lfw(c, [root], augmentations=4)
            pixels = ds.download()
        else:
            ds = DeviceDataset(c, pixels)
        st = [ds.train_step(hyper, B, seed + k) for k in range(2)]
        res.append((st, ds.download(), c.get_params(NET_G), c.get_params(NET_D)))
        ds.close()
        c.close()
    (s1, d1, g1, D1), (s2, d2, g2, D2) = res
    np.testing.assert_array_equal(d1, d2)
    assert s1 == s2
    np.testing.assert_array_equal(g1, g2)
    np.testing.assert_array_equal(D1, D2)


def test_refusals_launch_nothing_and_leave_the_context_usable(ctx, gray_ctx, golden):
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset, lfw_aug_params
    from face_generator_b200.lib import FGError
    srcs = golden["photos"][:2]
    src = DeviceDataset(ctx, srcs)
    dst = DeviceDataset(ctx, shape=(6, 3, 64, 64))
    dst.upload(0, np.full((6, 3, 64, 64), 7, np.uint8))
    good = lfw_aug_params(43, 0, 2, 2, 250, 250)

    def refused(d_src, d_dst, augs, first=0, what=""):
        c = d_dst.ctx
        before = c.launches()
        with pytest.raises(FGError) as ex:
            d_dst.augment(d_src, first, augs)
        assert "fg_dataset_augment" in str(ex.value) and what in str(ex.value), str(ex.value)
        assert c.launches() == before
        return ex.value

    def desc(**kw):
        a = good.copy()
        for k, v in kw.items():
            a[2][k] = v
        return a

    refused(src, dst, desc(src=2), what="source row")
    refused(src, dst, desc(src=-1), what="source row")
    refused(src, dst, desc(brightness=np.nan), what="brightness")
    refused(src, dst, desc(brightness=-0.5), what="brightness")
    refused(src, dst, desc(brightness=np.inf), what="brightness")
    m = good[2]["m"].copy()
    m[7] = np.inf
    refused(src, dst, desc(m=m), what="m[7]")
    m[7] = np.nan
    refused(src, dst, desc(m=m), what="m[7]")
    refused(src, dst, desc(warp=2), what="warp")
    refused(src, dst, good, first=1, what="outside")  # rows [1, 7) of 6
    other = fg.Context(0, max_batch=16, channels=3)
    far = DeviceDataset(other, shape=(6, 3, 64, 64))
    refused(src, far, good, what="different contexts")
    far.close()
    other.close()
    g1 = DeviceDataset(gray_ctx, shape=(6, 1, 64, 64))
    g3 = DeviceDataset(gray_ctx, srcs)
    refused(g3, g1, good, what="channels")
    g1.close()
    g3.close()
    for shape in ((2, 3, 175, 250), (2, 3, 250, 166)):
        small = DeviceDataset(ctx, shape=shape)
        refused(small, dst, good, what="crop box")
        small.close()
    for shape in ((6, 3, 85, 64), (6, 3, 64, 85)):
        big = DeviceDataset(ctx, shape=shape)
        refused(src, big, good, what="[1, 84]")
        big.close()
    np.testing.assert_array_equal(dst.download(), np.full((6, 3, 64, 64), 7, np.uint8))  # nothing was written
    dst.augment(src, 0, good)  # the context and both caches still work
    np.testing.assert_array_equal(dst.download(), R.augment_rows(srcs, good))
    src.close()
    dst.close()
