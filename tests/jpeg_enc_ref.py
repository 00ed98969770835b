"""numpy restatement of the baseline JPEG encoder that Pillow's Image.save(f, "JPEG", quality=q) runs at its defaults
(libjpeg-turbo: JFIF 1.01, islow forward DCT, 4:2:0 for colour, standard Huffman tables, no restart markers).
face_generator_b200's jpeg_enc.cu is held to these rules bit for bit; tests/test_jpeg_encode_cpu.py holds these rules
to Pillow's bytes.

    encode(img, q)          img [C][H][W] uint8, C = 1 (grayscale) or 3 (YCbCr 4:2:0) -> the JFIF file
    coefficients(img, q)    the quantised coefficients, natural order, per component on its MCU-padded block grid
    header(C, H, W, q)      everything before the entropy-coded segment

The inputs of the golden cases come from hash_u32, a counter-based integer hash, so that they can be regenerated on
any machine without a random generator whose stream might change.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# T.81 Annex K.1, natural order
BASE_Q = (np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99]),
          np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32))


def _ac_vals(prefix):
    """The AC symbols of a K.3 table: its irregular head, then every other run/size symbol in increasing order."""
    rest = sorted(set([r << 4 | s for r in range(16) for s in range(1, 11)] + [0x00, 0xF0]) - set(prefix))
    return list(prefix) + rest


# T.81 Annex K.3: BITS[1..16] (number of codes of each length) and HUFFVAL; [0] DC luma, [1] AC luma, [2] DC chroma,
# [3] AC chroma
HUFF = (
    ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D],
     _ac_vals([0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22,
               0x71, 0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33,
               0x62, 0x72, 0x82, 0x09, 0x0A, 0x16])),
    ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77],
     _ac_vals([0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13,
               0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62,
               0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1])),
)


def huff_codes(t):
    """symbol -> (code, length) of a BITS / HUFFVAL table (T.81 C.2)."""
    bits, vals = HUFF[t]
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


def quant_tables(q):
    """jpeg_set_quality(q, force_baseline = TRUE): (luma, chroma), natural order."""
    assert 1 <= q <= 100
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return tuple(np.clip((b * scale + 50) // 100, 1, 255).astype(np.int64) for b in BASE_Q)


def _fix(x):
    return int(x * 65536 + 0.5)


def ycbcr(img):
    """jccolor.c rgb_ycc_convert: [3][H][W] uint8 -> Y, Cb, Cr int64 planes."""
    r, g, b = (img[c].astype(np.int64) for c in range(3))
    half = 1 << 15
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + (128 << 16) + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + (128 << 16) + half - 1) >> 16
    return y, cb, cr


def _cdiv(a, b):
    return -(-a // b)


def _pad(p, h, w):
    """p padded to h x w by replicating its last row and column."""
    return np.pad(p, ((0, h - p.shape[0]), (0, w - p.shape[1])), mode="edge")


def component_planes(img):
    """The sample planes the forward DCT reads, each padded to its component's block grid ceil(w/8) x ceil(h/8)."""
    C, H, W = img.shape
    if C == 1:
        return [_pad(img[0].astype(np.int64), 8 * _cdiv(H, 8), 8 * _cdiv(W, 8))]
    y, cb, cr = ycbcr(img)
    out = [_pad(y, 8 * _cdiv(H, 8), 8 * _cdiv(W, 8))]
    He, We = H + (H & 1), 16 * _cdiv(W, 16)  # one replicated row up to an even height; columns to the MCU width
    bias = np.tile([1, 2], We // 4)
    for p in (cb, cr):
        p = _pad(p, He, We)
        d = (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + bias[None, :]) >> 2  # h2v2_downsample
        out.append(_pad(d, 8 * _cdiv(H, 16), d.shape[1]))  # then to the iMCU height from the last downsampled row
    return out


CONST_BITS, PASS1_BITS = 13, 2
F0_298, F0_390, F0_541, F0_765, F0_899, F1_175 = 2446, 3196, 4433, 6270, 7373, 9633
F1_501, F1_847, F1_961, F2_053, F2_562, F3_072 = 12299, 15137, 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, first):
    """one jfdctint.c pass along the last axis of d [..., 8]."""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = np.empty_like(d)
    sh = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS
    if first:
        o[..., 0], o[..., 4] = (t10 + t11) << PASS1_BITS, (t10 - t11) << PASS1_BITS
    else:
        o[..., 0], o[..., 4] = _descale(t10 + t11, PASS1_BITS), _descale(t10 - t11, PASS1_BITS)
    z1 = (t12 + t13) * F0_541
    o[..., 2] = _descale(z1 + t13 * F0_765, sh)
    o[..., 6] = _descale(z1 - t12 * F1_847, sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F1_175
    t4, t5, t6, t7 = t4 * F0_298, t5 * F2_053, t6 * F3_072, t7 * F1_501
    z1, z2 = z1 * -F0_899, z2 * -F2_562
    z3, z4 = z3 * -F1_961 + z5, z4 * -F0_390 + z5
    o[..., 7] = _descale(t4 + z1 + z3, sh)
    o[..., 5] = _descale(t5 + z2 + z4, sh)
    o[..., 3] = _descale(t6 + z2 + z3, sh)
    o[..., 1] = _descale(t7 + z1 + z4, sh)
    return o


def fdct_quant(blocks, qt):
    """blocks [n][8][8] samples 0..255 -> quantised coefficients [n][64], natural order."""
    d = _fdct_1d(blocks.astype(np.int64) - 128, True)
    d = _fdct_1d(d.swapaxes(-1, -2), False).swapaxes(-1, -2).reshape(-1, 64)
    q8 = 8 * qt[None, :]
    return (np.sign(d) * ((np.abs(d) + q8 // 2) // q8)).astype(np.int64)


def mcu_grid(C, H, W):
    return (_cdiv(W, 16), _cdiv(H, 16)) if C == 3 else (_cdiv(W, 8), _cdiv(H, 8))


def coefficients(img, q):
    """[component] -> [bh][bw][64] quantised coefficients on the MCU-padded grid (the layout the decoder's scratch
    uses), with jccoefct.c's dummy blocks: zero AC, the DC of the previous block of the MCU."""
    C, H, W = img.shape
    qts = quant_tables(q)
    mcux, mcuy = mcu_grid(C, H, W)
    out = []
    for c, p in enumerate(component_planes(img)):
        bh, bw = p.shape[0] // 8, p.shape[1] // 8
        blocks = p.reshape(bh, 8, bw, 8).swapaxes(1, 2).reshape(-1, 8, 8)
        real = fdct_quant(blocks, qts[min(c, 1)]).reshape(bh, bw, 64)
        f = 2 if (C == 3 and c == 0) else 1
        full = np.zeros((mcuy * f, mcux * f, 64), np.int64)
        full[:bh, :bw] = real
        if bw < full.shape[1]:  # right dummy column of the last MCU column: the DC of its left neighbour
            full[:bh, bw, 0] = full[:bh, bw - 1, 0]
        if bh < full.shape[0]:  # bottom dummy row: the DC of the MCU's last block of the row above
            for mx in range(mcux):
                full[bh, mx * f:(mx + 1) * f, 0] = full[bh - 1, mx * f + f - 1, 0]
        out.append(full)
    return out


def _category(v):
    v = abs(int(v))
    return v.bit_length()


def _bits_of(v, s):
    return (v if v >= 0 else v + (1 << s) - 1) & ((1 << s) - 1)


def entropy_bits(coefs, C):
    """The scan as a string of '0' / '1' before byte stuffing and padding."""
    tabs = [huff_codes(t) for t in range(4)]
    mcuy, mcux = coefs[-1].shape[:2]
    f = 2 if C == 3 else 1
    parts, pred = [], [0] * C

    def block(blk, c):
        dc_t, ac_t = tabs[0 if c == 0 else 2], tabs[1 if c == 0 else 3]
        zz = blk[ZIGZAG]
        diff = int(zz[0]) - pred[c]
        pred[c] = int(zz[0])
        s = _category(diff)
        code, n = dc_t[s]
        parts.append(format(code, "0%db" % n))
        if s:
            parts.append(format(_bits_of(diff, s), "0%db" % s))
        nz = np.nonzero(zz[1:])[0] + 1
        k = 1
        for pos in nz:
            r = pos - k
            while r > 15:
                code, n = ac_t[0xF0]
                parts.append(format(code, "0%db" % n))
                r -= 16
            v = int(zz[pos])
            s = _category(v)
            code, n = ac_t[r << 4 | s]
            parts.append(format(code, "0%db" % n) + format(_bits_of(v, s), "0%db" % s))
            k = pos + 1
        if k < 64:
            code, n = ac_t[0x00]
            parts.append(format(code, "0%db" % n))

    for my in range(mcuy):
        for mx in range(mcux):
            for by in range(f):
                for bx in range(f):
                    block(coefs[0][my * f + by, mx * f + bx], 0)
            for c in range(1, C):
                block(coefs[c][my, mx], c)
    return "".join(parts)


def stuff(bits):
    """Bits -> bytes: padded with 1-bits to a whole byte, a 0x00 after every 0xFF."""
    bits += "1" * (-len(bits) % 8)
    raw = int(bits, 2).to_bytes(len(bits) // 8, "big") if bits else b""
    return raw.replace(b"\xff", b"\xff\x00")


def _seg(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + bytes(body)


def header(C, H, W, q):
    """SOI, APP0 (JFIF 1.01, density 1:1, unit 0), DQT per table, SOF0, DHT per table, SOS: Pillow's bytes."""
    qts = quant_tables(q)
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    nt = 2 if C == 3 else 1
    for t in range(nt):
        out += _seg(0xDB, [t] + [int(v) for v in qts[t][ZIGZAG]])
    comps = [(1, 0x22 if C == 3 else 0x11, 0)] + [(2, 0x11, 1), (3, 0x11, 1)][:C - 1]
    sof = [8, H >> 8, H & 255, W >> 8, W & 255, C]
    for cid, hv, tq in comps:
        sof += [cid, hv, tq]
    out += _seg(0xC0, sof)
    for t in range(2 * nt):
        bits, vals = HUFF[t]
        out += _seg(0xC4, [((t & 1) << 4) | (t >> 1)] + list(bits) + list(vals))
    sos = [C]
    for cid, _, tq in comps:
        sos += [cid, 0x00 if tq == 0 else 0x11]
    out += _seg(0xDA, sos + [0, 63, 0])
    return out


def encode(img, q=75):
    """img [C][H][W] uint8 -> the bytes Pillow's Image.save(f, "JPEG", quality=q) writes for it."""
    img = np.asarray(img, np.uint8)
    C, H, W = img.shape
    assert C in (1, 3)
    return header(C, H, W, q) + stuff(entropy_bits(coefficients(img, q), C)) + b"\xff\xd9"


# ---- inputs of the golden cases --------------------------------------------------------------------------------------
def hash_u32(seed, n):
    """n 32-bit words of a counter-based hash (the splitmix64 finaliser of seed * 2^32 + i)."""
    with np.errstate(over="ignore"):
        x = (np.uint64(seed) << np.uint64(32)) + np.arange(n, dtype=np.uint64)
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return (x >> np.uint64(32)).astype(np.uint32)


class HashRng:
    """The two numpy Generator calls make_golden_jpeg.face draws from, on hash_u32: uniform, and a normal
    approximated by the sum of four uniforms (basic float arithmetic only, so bitwise the same everywhere)."""

    def __init__(self, seed):
        self.seed, self.n = seed, 0

    def _u(self, size):
        k = int(np.prod(size)) if size is not None else 1
        u = hash_u32(self.seed, self.n + k)[self.n:].astype(np.float64) / 2.0 ** 32
        self.n += k
        return u.reshape(size) if size is not None else float(u[0])

    def uniform(self, lo, hi, size=None):
        return lo + (hi - lo) * self._u(size)

    def normal(self, mu, sigma, size):
        s = self._u((4,) + tuple(size)).sum(0) - 2.0
        return mu + sigma * s * np.sqrt(3.0)


KINDS = ("noise", "face", "flat0", "flat255", "checker", "lines", "gradient")


def content(kind, seed, C, H, W):
    """A [C][H][W] uint8 test image of one kind, from hash_u32(seed)."""
    if kind == "noise":
        return (hash_u32(seed, C * H * W) & 255).astype(np.uint8).reshape(C, H, W)
    if kind == "face":
        import os
        import sys
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
        from make_golden_jpeg import face
        f = face(HashRng(seed), H, W).transpose(2, 0, 1)
        return np.ascontiguousarray(f if C == 3 else f[1:2])
    if kind in ("flat0", "flat255"):
        return np.full((C, H, W), 0 if kind == "flat0" else 255, np.uint8)
    y, x = np.mgrid[0:H, 0:W]
    if kind == "checker":  # saturated 1-pixel checkerboard, a different phase per plane
        return np.stack([((x + y + c) & 1) * 255 for c in range(C)]).astype(np.uint8)
    if kind == "lines":  # 1-pixel lines on a hashed background
        bg = (hash_u32(seed, C * H * W) & 63).astype(np.uint8).reshape(C, H, W) + 96
        bg[:, ::5, :] = 255
        bg[:, :, 3::7] = 0
        return bg
    if kind == "gradient":
        return np.stack([((x * 255) // max(W - 1, 1) + c * 40 + (y * 3)) & 255 for c in range(C)]).astype(np.uint8)
    raise ValueError(kind)
