"""GPU: sample.lua's sheets.  fg_image_grid equals tests/grid_ref.py bitwise (host and device images, orders and outputs,
size queries, refusals); fg_jpeg_encode equals tests/jpeg_enc_ref.py and the SHA-256s of tests/golden/sheets_jpeg.npz,
with the one-CTA and the multi-CTA entropy coders forced on the same inputs, and equals fg_dataset_encode_jpeg on a
dataset's rows; fg_dataset_nearest_sized at 32 equals fg_dataset_nearest and at 16 a float64 brute force;
fg_s16_D_score equals a chunked fg_s16_D_forward loop and the oracle; sample_run writes sample.lua's files, each the
reference encode of the reference grid of the run's own images.  Reads only numpy inputs (no Pillow)."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import grid_ref as G
import jpeg_enc_ref as R
import parity_utils as PU

pytestmark = pytest.mark.gpu
FG_ERR_INVALID = -1
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "sheets_jpeg.npz")


def P(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def ctxs():
    import face_generator_b200 as fg
    c3, c1 = fg.Context(0, max_batch=16, channels=3), fg.Context(0, max_batch=16, channels=1)
    yield {3: c3, 1: c1}
    c3.close()
    c1.close()


def images(N, Cc, H, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-0.9, 1.2, (N, Cc, H, H)).astype(np.float32)


def dev_copy(ctx, a):
    p = ctx.lib.fg_dev_alloc(max(a.nbytes, 4))
    assert p
    assert ctx.lib.fg_memcpy(ctx.h, p, P(a), a.nbytes) == 0
    return p


def download(ctx, p, shape, dtype):
    out = np.empty(shape, dtype)
    assert ctx.lib.fg_memcpy(ctx.h, P(out), p, out.nbytes) == 0
    return out


# ---- fg_image_grid --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cc", [1, 3])
@pytest.mark.parametrize("H", [16, 32, 64])
@pytest.mark.parametrize("padding", [0, 2])
def test_grid_equals_reference(ctxs, Cc, H, padding):
    from face_generator_b200 import sheets
    ctx = ctxs[3]
    imgs = images(1024, Cc, H, 10 * H + Cc + padding)
    for N in (1, 7, 64, 1024):
        for nrow in (1, 8, 16, 32):
            xm = min(nrow, N)
            Hg, Wg = -(-N // xm) * (H + padding), xm * (H + padding)
            sub = imgs[:N]
            if Hg > 4096 or Wg > 4096:
                out = np.full(8, 7, np.uint8)
                before = ctx.launches()
                rc = ctx.lib.fg_image_grid(ctx.h, P(sub), N, Cc, H, H, None, N, nrow, padding, P(out), None, None)
                assert rc == FG_ERR_INVALID and ctx.launches() == before and (out == 7).all(), (N, nrow)
                continue
            got = sheets.image_grid(ctx, sub, nrow, padding)
            assert got.shape == (Cc, Hg, Wg)
            np.testing.assert_array_equal(got, G.grid(sub, nrow, padding), err_msg=str((N, nrow)))
            if N == 64:  # a host order: reversed, with a repeat
                order = np.concatenate([np.arange(63, 0, -1), [5]]).astype(np.int32)
                np.testing.assert_array_equal(sheets.image_grid(ctx, imgs, nrow, padding, order),
                                              G.grid(imgs, nrow, padding, order), err_msg=str(nrow))


def test_grid_device_inputs_outputs_order_and_size_queries(ctxs):
    from face_generator_b200 import sheets
    ctx = ctxs[3]
    imgs = images(300, 3, 32, 5)
    order = ((np.arange(64) * 37) % 300).astype(np.int32)
    want = G.grid(imgs, 8, 2, order)
    Hg, Wg = want.shape[1:]
    bufs = [dev_copy(ctx, imgs), dev_copy(ctx, order), ctx.lib.fg_dev_alloc(want.size)]
    try:
        di, do, dout = bufs
        dimg = sheets.DeviceImages(di, imgs.shape)
        for img_arg in (imgs, dimg):
            for ord_arg, count in ((order, None), (do, 64)):
                np.testing.assert_array_equal(sheets.image_grid(ctx, img_arg, 8, 2, ord_arg, count=count), want)
                sheets.image_grid(ctx, img_arg, 8, 2, ord_arg, count=count, out=dout)
                np.testing.assert_array_equal(download(ctx, dout, want.shape, np.uint8), want)
        # a size query launches nothing
        hg, wg = C.c_int(0), C.c_int(0)
        before = ctx.launches()
        assert ctx.lib.fg_image_grid(ctx.h, P(imgs), 300, 3, 32, 32, P(order), 64, 8, 2, None, C.byref(hg), C.byref(wg)) == 0
        assert (hg.value, wg.value) == (Hg, Wg) and ctx.launches() == before
        assert sheets.grid_size(ctx, imgs.shape, 32) == (10 * 32, 32 * 32)
    finally:
        for p in bufs:
            ctx.lib.fg_dev_free(p)


def test_grid_refusals_launch_nothing(ctxs):
    ctx = ctxs[3]
    imgs = images(8, 3, 16, 1)
    out = np.full(3 * 64 * 64, 9, np.uint8)
    bad_order = np.array([0, 8], np.int32)
    before = ctx.launches()
    for args in ((imgs, 8, 0, 16, 16, None, 8, 4, 0), (imgs, 8, 4, 16, 16, None, 8, 4, 0),
                 (imgs, 8, 3, 16, 16, None, 8, 4, 1), (imgs, 8, 3, 16, 16, None, 8, 4, -2),
                 (imgs, 8, 3, 16, 16, None, 9, 4, 0), (imgs, 8, 3, 16, 16, None, 8, 0, 0),
                 (imgs, 8, 3, 16, 16, None, 0, 4, 0), (imgs, 8, 3, 16, 16, bad_order, 2, 4, 0),
                 (imgs, 8, 3, 16, 16, None, 8, 1, 0), (None, 8, 3, 16, 16, None, 8, 4, 0)):
        im, N, Cc, H, W, order, count, nrow, pad = args
        if nrow == 1 and pad == 0:  # 8 rows of a 600-high image: above 4096
            H = W = 600
        rc = ctx.lib.fg_image_grid(ctx.h, None if im is None else P(im), N, Cc, H, W, None if order is None else P(order),
                                   count, nrow, pad, P(out), None, None)
        assert rc == FG_ERR_INVALID, args
    assert ctx.launches() == before and (out == 9).all()


def test_grid_nan_and_constant(ctxs):
    from face_generator_b200 import sheets
    ctx = ctxs[1]
    imgs = images(9, 1, 16, 3)
    imgs[2, 0, 3, 4] = np.nan
    imgs[5, 0, 0, 0] = np.nan
    np.testing.assert_array_equal(sheets.image_grid(ctx, imgs, 4, 2), G.grid(imgs, 4, 2))
    flat = np.full((5, 1, 16, 16), 0.25, np.float32)
    assert (sheets.image_grid(ctx, flat, 2) == 0).all()


# ---- fg_jpeg_encode -------------------------------------------------------------------------------------------------
def golden_cases():
    with np.load(GOLDEN) as z:
        g = {k: z[k] for k in z.files}
    return [(str(g["kind"][i]), int(g["seed"][i]), int(g["C"][i]), int(g["H"][i]), int(g["W"][i]), int(g["quality"][i]),
             str(g["file_sha256"][i])) for i in range(len(g["kind"]))]


def encode_routes(ctx, img, q):
    """fg_jpeg_encode's file under the automatic, the one-CTA and the multi-CTA routes"""
    from face_generator_b200 import sheets
    out = []
    try:
        for route in (0, 1, 2):
            ctx.set_option("jpeg_route", route)
            out.append(sheets.encode_jpeg(ctx, img, q)[0])
    finally:
        ctx.set_option("jpeg_route", 0)
    return out


def test_encode_equals_golden_on_both_routes(ctxs):
    for kind, seed, Cc, H, W, q, sha in golden_cases():
        img = R.content(kind, seed, Cc, H, W)
        files = encode_routes(ctxs[Cc], img, q)
        for f in files:
            assert hashlib.sha256(f).hexdigest() == sha, (kind, Cc, H, W, q)
        if H * W <= 512 * 512:
            assert files[0] == R.encode(img, q), (kind, Cc, H, W, q)


@pytest.mark.parametrize("Cc,H,W", [(3, 256, 256), (3, 1024, 1024), (1, 512, 512), (3, 100, 300), (3, 2048, 2048),
                                    (3, 16, 16)])
def test_routes_agree_on_noise_at_quality_100(ctxs, Cc, H, W):
    """Noise at quality 100: 0xFF bytes everywhere, so stuffed bytes fall on the multi-CTA coder's segment edges."""
    img = R.content("noise", H + 7 * W, Cc, H, W)
    files = encode_routes(ctxs[Cc], img, 100)
    assert files[0] == files[1] == files[2]
    assert files[0].count(b"\xff\x00") > H * W // 200 or H * W < 1024
    if H * W <= 300 * 300:
        assert files[0] == R.encode(img, 100)


def test_several_images_host_and_device_sizes_and_short_buffer(ctxs):
    from face_generator_b200 import sheets
    ctx = ctxs[3]
    imgs = np.stack([R.content(k, 40 + i, 3, 192, 256) for i, k in enumerate(("noise", "lines", "gradient"))])
    want = [R.encode(im, 75) for im in imgs]
    for route in (1, 2):
        ctx.set_option("jpeg_route", route)
        try:
            assert sheets.encode_jpeg(ctx, imgs, 75) == want
            p = dev_copy(ctx, imgs)
            try:
                assert sheets.encode_jpeg(ctx, p, 75, shape=imgs.shape) == want
            finally:
                ctx.lib.fg_dev_free(p)
        finally:
            ctx.set_option("jpeg_route", 0)
    sizes = np.cumsum([0] + [len(b) for b in want])
    offsets = np.full(4, -3, np.int64)
    out = np.full(int(sizes[-1]), 0xA5, np.uint8)
    assert ctx.lib.fg_jpeg_encode(ctx.h, P(imgs), 3, 3, 192, 256, 75, P(out), out.size - 1, P(offsets)) == FG_ERR_INVALID
    np.testing.assert_array_equal(offsets, sizes)
    assert (out == 0xA5).all()
    before = ctx.launches()
    for args in ((0, 3, 192, 256, 75), (3, 2, 192, 256, 75), (3, 3, 0, 256, 75), (3, 3, 192, 4097, 75),
                 (3, 3, 192, 256, 0), (3, 3, 192, 256, 101)):
        assert ctx.lib.fg_jpeg_encode(ctx.h, P(imgs), *args, P(out), out.size, P(offsets)) == FG_ERR_INVALID, args
    assert ctx.lib.fg_jpeg_encode(ctx.h, P(imgs), 3, 3, 192, 256, 75, P(out), out.size, None) == FG_ERR_INVALID
    assert ctx.lib.fg_jpeg_encode(ctx.h, None, 3, 3, 192, 256, 75, P(out), out.size, P(offsets)) == FG_ERR_INVALID
    assert ctx.launches() == before and (out == 0xA5).all()


def test_encode_equals_dataset_encode(ctxs):
    from face_generator_b200 import sheets
    from face_generator_b200.dataset import DeviceDataset
    for Cc in (3, 1):
        rows = np.stack([R.content(R.KINDS[k % len(R.KINDS)], 300 + k, Cc, 64, 64) for k in range(40)])
        ds = DeviceDataset(ctxs[Cc], rows)
        want = ds.encode_jpeg(quality=75)
        ds.close()
        assert sheets.encode_jpeg(ctxs[Cc], rows, 75) == want


# ---- --scale 16 scoring and sized neighbours ---------------------------------------------------------------------------
def test_nearest_sized(ctxs):
    from face_generator_b200.dataset import DeviceDataset
    ctx = ctxs[3]
    lib = ctx.lib
    rows = np.stack([R.content(R.KINDS[k % len(R.KINDS)], 500 + k, 3, 64, 64) for k in range(400)])
    ds = DeviceDataset(ctx, rows)
    rng = np.random.default_rng(4)
    q32 = rng.random((20, 3, 32, 32)).astype(np.float32)
    q32[:4] = ds.gather(np.array([7, 77, 154, 399], np.int32))  # exact hits on distinct (noise) rows
    i1, d1, i2, d2 = (np.empty(20, t) for t in (np.int32, np.float32, np.int32, np.float32))
    assert lib.fg_dataset_nearest(ds.h, P(q32), 20, P(i1), P(d1)) == 0
    assert lib.fg_dataset_nearest_sized(ds.h, 32, P(q32), 20, P(i2), P(d2)) == 0
    np.testing.assert_array_equal(i1, i2)
    assert d1.tobytes() == d2.tobytes()
    assert i1[:4].tolist() == [7, 77, 154, 399]
    # size 16: the float64 brute force over the 16x16 gathers
    cands = np.concatenate([ds.gather(np.arange(s, min(s + 16, 400), dtype=np.int32), size=16) for s in range(0, 400, 16)])
    q16 = rng.random((24, 3, 16, 16)).astype(np.float32)
    q16[:3] = cands[[14, 203, 308]] + np.float32(1e-3)
    idx, dist = np.empty(24, np.int32), np.empty(24, np.float32)
    assert lib.fg_dataset_nearest_sized(ds.h, 16, P(q16), 24, P(idx), P(dist)) == 0
    d64 = np.sqrt(((q16.reshape(24, 1, -1).astype(np.float64) - cands.reshape(1, 400, -1)) ** 2).sum(-1))
    for q in range(24):
        o = np.argsort(d64[q], kind="stable")
        near_tie = d64[q, o[1]] - d64[q, o[0]] <= 1e-6 * d64[q, o[0]]
        if not near_tie:
            assert idx[q] == o[0], q
        assert abs(dist[q] - d64[q, idx[q]]) <= 1e-5 * max(1.0, d64[q, idx[q]])
    assert idx[:3].tolist() == [14, 203, 308]
    before = ctx.launches()
    for size in (0, 65):
        assert lib.fg_dataset_nearest_sized(ds.h, size, P(q16), 24, P(idx), P(dist)) == FG_ERR_INVALID
    assert ctx.launches() == before
    ds.close()


def test_s16_D_score(ctxs):
    import s16_utils as SU
    from face_generator_b200.lib import NET_D, S16
    from oracle import oracle_s16 as OS
    ctx = ctxs[3]
    net = S16(ctx)
    case = SU.make_case(16, 3, seed=71, init="trained")
    net.set_params(NET_D, case["PD"])
    imgs = images(100, 3, 16, 8)
    for training in (1, 0):
        got = np.empty(100, np.float32)
        assert ctx.lib.fg_s16_D_score(net.h, P(imgs), 100, 16, training, 1234, P(got)) == 0
        loop = np.concatenate([net.D_forward(imgs[s:s + 16], None, training=bool(training), seed=1234 + s)
                               for s in range(0, 100, 16)])
        assert got.tobytes() == loop.tobytes(), training
    ref = OS.f64.D().forward(case["PD"], imgs, None, False)
    assert PU.relerr(got, ref) < 1e-4
    net.close()


# ---- sample_run ---------------------------------------------------------------------------------------------------------
def check_run(base, ctx, S, tmp_path, neighbours=None):
    from face_generator_b200 import sheets
    a = sheets.sample_run(base, 3, str(tmp_path / "a"), seed=9, neighbours=neighbours, return_images=True)
    names = sorted(os.listdir(tmp_path / "a"))
    want_names = sorted(f % 3 for f in sheets.SHEETS) + ([sheets.NEIGHBOURS_SHEET % 3] if neighbours else [])
    assert names == sorted(want_names)
    imgs = a["images"]
    assert imgs.shape == (1024, ctx.C, S, S)
    np.testing.assert_array_equal(a["best"], np.argsort(-a["preds_best"], kind="stable")[:64])
    np.testing.assert_array_equal(a["worst"], np.argsort(a["preds_worst"], kind="stable")[:64])
    assert (a["preds_best"] != a["preds_worst"]).any()  # two passes, two dropout draws
    expect = {"random256_0003_base.jpg": (imgs, a["random256"], 16), "random1024_0003_base.jpg": (imgs, None, 32),
              "best_0003_base.jpg": (imgs, a["best"], 8), "worst_0003_base.jpg": (imgs, a["worst"], 8),
              "random_0003_base.jpg": (imgs, a["random"], 8)}
    if neighbours is not None:
        nb = neighbours.gather(a["neighbours"], size=S)
        pairs = np.concatenate([imgs[a["best"][:16]], nb])
        expect["best_0003_neighbours_base.jpg"] = (pairs, [v for i in range(16) for v in (i, 16 + i)], 16)
        idx, dist = np.empty(16, np.int32), np.empty(16, np.float32)
        q = np.ascontiguousarray(imgs[a["best"][:16]])
        assert ctx.lib.fg_dataset_nearest_sized(neighbours.h, S, P(q), 16, P(idx), P(dist)) == 0
        np.testing.assert_array_equal(idx, a["neighbours"])
    for name, (src, order, nrow) in expect.items():
        data = (tmp_path / "a" / name).read_bytes()
        assert data == R.encode(G.grid(src, nrow, 0, order), 75), name
    b = sheets.sample_run(base, 3, str(tmp_path / "b"), seed=9, neighbours=neighbours)
    for name in names:
        assert (tmp_path / "a" / name).read_bytes() == (tmp_path / "b" / name).read_bytes(), name
    assert (a["best"] == b["best"]).all()


def test_sample_run_32(ctxs, tmp_path):
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    ctx = ctxs[3]
    case = PU.make_case(16, 3, seed=31, init="trained")
    ctx.set_params(NET_G, case["PG"])
    ctx.set_params(NET_D, case["PD"])
    rows = np.stack([R.content(R.KINDS[k % len(R.KINDS)], 700 + k, 3, 64, 64) for k in range(150)])
    ds = DeviceDataset(ctx, rows)
    check_run(ctx, ctx, 32, tmp_path, neighbours=ds)
    ds.close()


def test_sample_run_scale16(ctxs, tmp_path):
    import s16_utils as SU
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G, S16
    ctx = ctxs[3]
    net = S16(ctx)
    case = SU.make_case(16, 3, seed=32, init="trained")
    net.set_params(NET_G, case["PG"])
    net.set_params(NET_D, case["PD"])
    rows = np.stack([R.content(R.KINDS[k % len(R.KINDS)], 800 + k, 3, 64, 64) for k in range(120)])
    ds = DeviceDataset(ctx, rows)
    check_run(net, ctx, 16, tmp_path, neighbours=ds)
    ds.close()
    net.close()
