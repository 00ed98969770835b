"""Writes tests/golden/jpeg_corpus.npz: JPEG files made with Pillow from fixed seeds, each with Pillow's decode
(libjpeg-turbo, default decompression) or the refusal fg_jpeg_info / fg_dataset_upload_jpeg must give.  The GPU tests
read only the npz, so the machine that runs them needs no Pillow.  To keep the file small, every decode is stored as
the SHA-256 of its planar bytes, and only the eight dataset faces also keep their pixels.

    python tests/golden/make_golden_jpeg.py      # rewrites the npz (Pillow with libjpeg-turbo required)

Arrays (N files):
    names [N] str, data uint8 (all files back to back), offsets [N+1] int64
    C, H, W [N] int32            what fg_jpeg_info reports (0 where it refuses)
    info_rc, upload_rc [N] int32 0 for a supported file, else the FG_ERR_* code expected
    cache_h, cache_w [N] int32   the cache size the upload uses (a wrong-size file differs from H x W)
    sha256 [N] str               SHA-256 (hex) of Pillow's planar [C][H][W] uint8 decode (empty for refusals)
    decoded uint8 (back to back), dec_offsets [N+1] int64   that decode itself, for the dataset faces only
    faces [N] bool               the exact dataset/generate_dataset.py form: 64x64, quality 75, 4:2:0
"""
import hashlib
import io
import os

import numpy as np

FG_ERR_INVALID, FG_ERR_UNSUPPORTED = -1, -4
HERE = os.path.dirname(os.path.abspath(__file__))


def face(rng, h, w):
    """A face-like picture: lit background gradient, a skin ellipse, eyes, mouth, hair and a little sensor noise."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    yy, xx = (y + 0.5) / h, (x + 0.5) / w
    bg = rng.uniform(40, 200, 3)
    tilt = rng.uniform(-60, 60, 3)
    img = bg[None, None, :] + tilt[None, None, :] * (xx[..., None] - 0.5) + 30 * (yy[..., None] - 0.5)
    cy, cx = rng.uniform(0.45, 0.55), rng.uniform(0.45, 0.55)
    ry, rx = rng.uniform(0.32, 0.42), rng.uniform(0.25, 0.33)
    skin = np.array([rng.uniform(150, 235), rng.uniform(110, 180), rng.uniform(90, 150)])
    d = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
    shade = np.clip(1.0 - 0.35 * d, 0.5, 1.0)
    img = np.where((d < 1)[..., None], skin[None, None, :] * shade[..., None], img)
    hair = rng.uniform(10, 90, 3)
    img = np.where(((d < 1.15) & (yy < cy - 0.55 * ry))[..., None], hair[None, None, :], img)
    for ex in (cx - 0.4 * rx, cx + 0.4 * rx):
        e = ((yy - (cy - 0.15 * ry)) / 0.05) ** 2 + ((xx - ex) / 0.07) ** 2
        img = np.where((e < 1)[..., None], np.array([30.0, 25.0, 20.0])[None, None, :], img)
    m = ((yy - (cy + 0.45 * ry)) / 0.035) ** 2 + ((xx - cx) / 0.16) ** 2
    img = np.where((m < 1)[..., None], np.array([160.0, 60.0, 60.0])[None, None, :], img)
    img = img + rng.normal(0, 4, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def noise(rng, h, w):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def encode(arr, mode="RGB", **kw):
    from PIL import Image
    im = Image.fromarray(arr) if mode in ("RGB", "L") else Image.fromarray(arr).convert(mode)
    buf = io.BytesIO()
    im.save(buf, "JPEG", **kw)
    return buf.getvalue()


def pillow_decode(b):
    from PIL import Image
    im = Image.open(io.BytesIO(b))
    im.load()
    a = np.asarray(im)
    return a[None] if a.ndim == 2 else np.ascontiguousarray(a.transpose(2, 0, 1))


def build():
    import PIL.features
    assert PIL.features.check_feature("libjpeg_turbo"), "Pillow must be built with libjpeg-turbo"
    rng = np.random.default_rng(20261017)
    entries = []  # (name, bytes, refusal or None, cache size or None, is_face)

    def ok(name, b, is_face=False):
        entries.append((name, b, None, None, is_face))

    sub = {"444": 0, "422": 1, "420": 2}
    # the generate_dataset.py form: scipy.misc.imsave -> Pillow defaults (quality 75, 4:2:0), 64x64
    for i in range(8):
        ok("dataset_face_%d" % i, encode(face(rng, 64, 64), quality=75), True)
    # qualities x content x subsampling at 64x64
    for q in (10, 50, 75, 95, 100):
        for kind, fn in (("face", face), ("noise", noise)):
            for s in ("444", "422", "420"):
                ok("q%d_%s_%s" % (q, kind, s), encode(fn(rng, 64, 64), quality=q, subsampling=sub[s]))
    # sizes x subsampling; the narrow ones take the replicating path of chroma with fewer than 3 columns
    for (h, w) in ((1, 1), (7, 13), (17, 33), (61, 47), (100, 75), (255, 255), (5, 3), (4, 4), (9, 2), (3, 6)):
        for s in ("444", "422", "420"):
            ok("size%dx%d_%s" % (h, w, s), encode(face(rng, h, w), quality=85, subsampling=sub[s]))
    # optimised Huffman tables (one table set per file)
    for s in ("444", "420"):
        ok("optimize_%s" % s, encode(face(rng, 64, 64), quality=75, subsampling=sub[s], optimize=True))
        ok("optimize_noise_%s" % s, encode(noise(rng, 40, 56), quality=90, subsampling=sub[s], optimize=True))
    # restart intervals
    ok("restart_blocks3_420", encode(face(rng, 64, 64), quality=75, restart_marker_blocks=3))
    ok("restart_blocks1_444", encode(noise(rng, 61, 47), quality=80, subsampling=0, restart_marker_blocks=1))
    ok("restart_rows1_422", encode(face(rng, 61, 47), quality=75, subsampling=1, restart_marker_rows=1))
    ok("restart_rows2_420", encode(face(rng, 100, 75), quality=60, restart_marker_rows=2))
    # grayscale
    for (h, w) in ((64, 64), (17, 33), (1, 1), (61, 47)):
        g = face(rng, h, w)[..., 1]
        ok("gray_%dx%d" % (h, w), encode(g, "L", quality=75))
    ok("gray_restart_blocks5", encode(face(rng, 64, 64)[..., 0], "L", quality=90, restart_marker_blocks=5))
    ok("gray_optimize_q100", encode(noise(rng, 33, 17)[..., 2], "L", quality=100, optimize=True))
    # EXIF, ICC and comment segments are skipped
    from PIL import Image
    exif = Image.Exif()
    exif[0x010F] = "face-generator test"
    exif[0x0110] = "seeded"
    icc = bytes(rng.integers(0, 256, 3000, dtype=np.uint8))
    ok("segments_exif_icc_comment", encode(face(rng, 64, 64), quality=75, exif=exif.tobytes(), icc_profile=icc,
                                           comment="face-like test image"))
    # refusals
    base = encode(face(rng, 64, 64), quality=75)
    entries.append(("refuse_progressive", encode(face(rng, 64, 64), quality=75, progressive=True),
                    (FG_ERR_UNSUPPORTED, FG_ERR_UNSUPPORTED), None, False))
    entries.append(("refuse_cmyk", encode(face(rng, 64, 64), "CMYK", quality=75),
                    (FG_ERR_UNSUPPORTED, FG_ERR_UNSUPPORTED), None, False))
    entries.append(("refuse_truncated", base[:len(base) * 3 // 5], (0, FG_ERR_INVALID), None, False))
    sos = base.index(b"\xff\xda")
    at = sos + 2 + int.from_bytes(base[sos + 2:sos + 4], "big") + 200
    corrupt = base[:at] + b"\xff\x00" * 6 + base[at + 12:]
    entries.append(("refuse_corrupt_huffman", corrupt, (0, FG_ERR_INVALID), None, False))
    entries.append(("refuse_wrong_size", encode(face(rng, 32, 32), quality=75), (0, FG_ERR_INVALID), (64, 64), False))

    names, blobs, dec, sha, Cs, Hs, Ws, info_rc, up_rc, ch, cw, faces = [], [], [], [], [], [], [], [], [], [], [], []
    for name, b, refusal, cache, is_face in entries:
        names.append(name)
        blobs.append(np.frombuffer(b, np.uint8))
        faces.append(is_face)
        if refusal is None or refusal[0] == 0:
            from PIL import Image
            im = Image.open(io.BytesIO(b))
            c = 1 if im.mode == "L" else 3
            Cs.append(c), Hs.append(im.height), Ws.append(im.width)
        else:
            Cs.append(0), Hs.append(0), Ws.append(0)
        if refusal is None:
            d = pillow_decode(b)
            assert d.shape == (Cs[-1], Hs[-1], Ws[-1]), (name, d.shape)
            sha.append(hashlib.sha256(np.ascontiguousarray(d).tobytes()).hexdigest())
            dec.append(d.reshape(-1) if is_face else np.zeros(0, np.uint8))
            info_rc.append(0), up_rc.append(0)
        else:
            sha.append("")
            dec.append(np.zeros(0, np.uint8))
            info_rc.append(refusal[0]), up_rc.append(refusal[1])
        h, w = cache if cache else (Hs[-1] or 64, Ws[-1] or 64)
        ch.append(h), cw.append(w)
    off = np.zeros(len(blobs) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in blobs])
    doff = np.zeros(len(dec) + 1, np.int64)
    doff[1:] = np.cumsum([len(d) for d in dec])
    i32 = lambda v: np.asarray(v, np.int32)
    return dict(names=np.asarray(names), data=np.concatenate(blobs), offsets=off, C=i32(Cs), H=i32(Hs), W=i32(Ws),
                info_rc=i32(info_rc), upload_rc=i32(up_rc), cache_h=i32(ch), cache_w=i32(cw),
                sha256=np.asarray(sha), decoded=np.concatenate(dec), dec_offsets=doff, faces=np.asarray(faces))


if __name__ == "__main__":
    out = os.path.join(HERE, "jpeg_corpus.npz")
    arrays = build()
    np.savez_compressed(out, **arrays)
    print("%s: %d files, %d bytes of JPEG, %d bytes on disk" % (out, len(arrays["names"]), arrays["data"].size,
                                                                os.path.getsize(out)))
