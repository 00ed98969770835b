// Per-symbol, per-block and per-pixel arithmetic of the baseline JPEG decoder (jpeg.cu), written from ITU-T T.81
// (Annex C Huffman tables, F.2.2 decoding, F.2.2.5 receive/extend, B.2.4.4 restart markers) and the
// Loeffler-Ligtenberg-Moschytz integer IDCT in its published 13-bit fixed-point form (the JDCT_ISLOW method), the
// triangle-filter chroma upsampling and the 16-bit fixed-point YCbCr -> RGB of the JFIF decoder everyone ships.
// Everything is integer arithmetic, so the device decode is bitwise reproducible and can be held bit for bit to
// libjpeg-turbo's default decompression (tests/test_gpu_jpeg.py).
//
// All functions are __host__ __device__ so that a host harness can hold them to the oracle before any GPU run.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define JPG_HD __host__ __device__ __forceinline__
#else
#define JPG_HD inline
#endif

namespace jpg {

// zig-zag scan position k -> natural (row-major) index (T.81 Figure A.6)
#define JPG_ZIGZAG                                                                                                    \
  {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, \
   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}
#ifdef __CUDACC__
__constant__ unsigned char kZigzagDev[64] = JPG_ZIGZAG;
#endif
static const unsigned char kZigzagHost[64] = JPG_ZIGZAG;
JPG_HD int natural_of(int k) {
#ifdef __CUDA_ARCH__
  return kZigzagDev[k];
#else
  return kZigzagHost[k];
#endif
}

// One Huffman table, decoded with a 9-bit lookahead: lut[peek9] = (code length << 8) | symbol, or 0 when the code is
// longer than 9 bits; then the canonical-code walk of T.81 F.2.2.3 over lengths 10..16 (maxcode / valoff).
constexpr int kLookBits = 9;
struct HuffTab {
  uint16_t lut[1 << kLookBits];
  int32_t maxcode[18];  // largest code of length l, -1 when none; [17] = sentinel
  int32_t valoff[17];   // index into vals of the first code of length l, minus that code
  uint8_t vals[256];
};

// Builds a table from the DHT counts bits[1..16] (bits[0] unused) and values.  Returns false for a table no
// conforming encoder writes (more codes than fit in a length, or more than 256 values).
inline bool build_huff(const uint8_t bits[17], const uint8_t* vals, HuffTab* t) {
  int n = 0;
  for (int l = 1; l <= 16; ++l) n += bits[l];
  if (n > 256) return false;
  for (int i = 0; i < (1 << kLookBits); ++i) t->lut[i] = 0;
  for (int i = 0; i < 256; ++i) t->vals[i] = i < n ? vals[i] : 0;
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t->valoff[l] = k - code;
    for (int i = 0; i < bits[l]; ++i, ++code, ++k) {
      if (l <= kLookBits) {
        const int shift = kLookBits - l;
        for (int j = 0; j < (1 << shift); ++j) t->lut[(code << shift) | j] = (uint16_t)((l << 8) | vals[k]);
      }
    }
    t->maxcode[l] = bits[l] ? code - 1 : -1;
    if (code > (1 << l)) return false;
    code <<= 1;
  }
  t->maxcode[0] = -1;
  t->maxcode[17] = 0x7fffffff;
  t->valoff[0] = 0;
  return true;
}

// MSB-first bit reader over one restart interval's entropy-coded bytes [p, end): 0xFF 0x00 is a stuffed 0xFF, any
// other 0xFF xx inside the interval is a stray marker (corrupt).  Past the end it feeds zero bits, as decoders do
// for a short final byte, and counts them so that the caller can tell whether real data ran out.
struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc = 0;  // next bits, left-aligned
  int nbits = 0;
  int padded = 0;    // zero bits fed past the end
  bool bad = false;  // a marker inside the interval
  JPG_HD void refill() {
    while (nbits <= 56) {
      uint32_t b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF) {
          if (p < end && *p == 0x00) {
            ++p;
          } else {
            bad = true;
            p = end;
            b = 0;
          }
        }
      } else {
        padded += 8;
      }
      acc |= (uint64_t)b << (56 - nbits);
      nbits += 8;
    }
  }
  JPG_HD uint32_t peek(int n) const { return (uint32_t)(acc >> (64 - n)); }
  JPG_HD void skip(int n) {
    acc <<= n;
    nbits -= n;
  }
  JPG_HD uint32_t get(int n) {
    if (n == 0) return 0;
    const uint32_t v = peek(n);
    skip(n);
    return v;
  }
  // real data was consumed past the interval's end (truncated or corrupt stream)
  JPG_HD bool overrun() const { return bad || nbits < padded; }
};

// one Huffman symbol (needs >= 16 bits in the reader); -1 for a bit pattern that is no code of the table
JPG_HD int decode_sym(BitReader& br, const HuffTab& t) {
  const uint32_t e = t.lut[br.peek(kLookBits)];
  if (e) {
    br.skip((int)(e >> 8));
    return (int)(e & 0xFF);
  }
  const uint32_t code16 = br.peek(16);
  for (int l = kLookBits + 1; l <= 16; ++l) {
    const int32_t c = (int32_t)(code16 >> (16 - l));
    if (c <= t.maxcode[l]) {
      br.skip(l);
      return t.vals[(c + t.valoff[l]) & 0xFF];
    }
  }
  return -1;
}

// T.81 F.2.2.1 EXTEND of an s-bit magnitude category
JPG_HD int extend(uint32_t v, int s) { return s == 0 ? 0 : ((int)v < (1 << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v); }

// Decodes one 8x8 block (T.81 F.2.2): the DC difference is added to *dc_pred, coefficients are written in natural
// order into out[64], which must be zero on entry (only non-zero ones are stored).  Returns false on an invalid
// code or a coefficient past position 63.
template <typename Coef>
JPG_HD bool decode_block(BitReader& br, const HuffTab& dc, const HuffTab& ac, int* dc_pred, Coef* out) {
  br.refill();
  const int s = decode_sym(br, dc);
  if (s < 0 || s > 11) return false;
  *dc_pred += extend(br.get(s), s);
  out[0] = (Coef)*dc_pred;
  for (int k = 1; k < 64;) {
    br.refill();
    const int rs = decode_sym(br, ac);
    if (rs < 0) return false;
    const int r = rs >> 4, sz = rs & 15;
    if (sz == 0) {
      if (r != 15) break;  // EOB
      k += 16;             // ZRL
      continue;
    }
    k += r;
    if (k > 63) return false;
    out[natural_of(k)] = (Coef)extend(br.get(sz), sz);
    ++k;
  }
  return true;
}

// ---- inverse DCT: LL&M, 13-bit constants, 2 extra bits of precision between the passes -------------------------
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int32_t c0_298631336 = 2446, c0_390180644 = 3196, c0_541196100 = 4433, c0_765366865 = 6270,
                  c0_899976223 = 7373, c1_175875602 = 9633, c1_501321110 = 12299, c1_847759065 = 15137,
                  c1_961570560 = 16069, c2_053119869 = 16819, c2_562915447 = 20995, c3_072711026 = 25172;

// the 1-D LL&M butterfly on x[0..7], results scaled by 2^13: out[i] for i = 0..7
JPG_HD void llm_1d(const int32_t* x, int32_t out[8]) {
  // even part: rotation of x2, x6 and the sum / difference of x0, x4
  const int32_t z1 = (x[2] + x[6]) * c0_541196100;
  const int32_t e2 = z1 - x[6] * c1_847759065;
  const int32_t e3 = z1 + x[2] * c0_765366865;
  const int32_t e0 = (x[0] + x[4]) * (1 << kConstBits);
  const int32_t e1 = (x[0] - x[4]) * (1 << kConstBits);
  const int32_t a0 = e0 + e3, a3 = e0 - e3, a1 = e1 + e2, a2 = e1 - e2;
  // odd part on x7, x5, x3, x1
  int32_t o0 = x[7], o1 = x[5], o2 = x[3], o3 = x[1];
  int32_t p1 = o0 + o3, p2 = o1 + o2, p3 = o0 + o2, p4 = o1 + o3;
  const int32_t p5 = (p3 + p4) * c1_175875602;
  o0 *= c0_298631336;
  o1 *= c2_053119869;
  o2 *= c3_072711026;
  o3 *= c1_501321110;
  p1 *= -c0_899976223;
  p2 *= -c2_562915447;
  p3 = p3 * -c1_961570560 + p5;
  p4 = p4 * -c0_390180644 + p5;
  o0 += p1 + p3;
  o1 += p2 + p4;
  o2 += p2 + p3;
  o3 += p1 + p4;
  out[0] = a0 + o3;
  out[7] = a0 - o3;
  out[1] = a1 + o2;
  out[6] = a1 - o2;
  out[2] = a2 + o1;
  out[5] = a2 - o1;
  out[3] = a3 + o0;
  out[4] = a3 - o0;
}
JPG_HD int32_t descale(int32_t x, int n) { return (x + (1 << (n - 1))) >> n; }
JPG_HD uint8_t clamp_u8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// coef[64] natural order, q[64] natural order -> 8x8 samples at out[y * ostride + x], level-shifted and clamped
template <typename Coef>
JPG_HD void idct_islow(const Coef* coef, const uint16_t* q, uint8_t* out, int ostride) {
  int32_t ws[64];
  for (int col = 0; col < 8; ++col) {
    int32_t x[8], r[8];
    for (int i = 0; i < 8; ++i) x[i] = (int32_t)coef[i * 8 + col] * (int32_t)q[i * 8 + col];
    llm_1d(x, r);
    for (int i = 0; i < 8; ++i) ws[i * 8 + col] = descale(r[i], kConstBits - kPass1Bits);
  }
  for (int row = 0; row < 8; ++row) {
    int32_t r[8];
    llm_1d(ws + row * 8, r);
    for (int i = 0; i < 8; ++i) out[row * ostride + i] = clamp_u8(descale(r[i], kConstBits + kPass1Bits + 3) + 128);
  }
}

// ---- chroma upsampling by 2 (triangle filter), edges replicated at the component's downsampled size -------------
// Horizontal output sample ox of one row in[0..w) at 2x: 3/4 of the nearer input sample + 1/4 of the farther one,
// rounding alternately up and down (bias 1 / 2).  Fewer than 3 input columns upsample by replication.
JPG_HD int up_h2(const uint8_t* in, int w, int ox) {
  const int i = ox >> 1;
  if (w <= 2) return in[i < w ? i : w - 1];
  const int v = in[i];
  if (ox & 1) {
    const int n = in[i + 1 < w ? i + 1 : w - 1];
    return (3 * v + n + 2) >> 2;
  }
  const int n = in[i > 0 ? i - 1 : 0];
  return (3 * v + n + 1) >> 2;
}
// h2v2: vertical 3:1 column sums of the nearer and the farther input row (the caller clamps rows to [0, h)), then
// the horizontal 3:1 of those sums with bias 8 / 7.
JPG_HD int up_h2v2(const uint8_t* near_row, const uint8_t* far_row, int w, int ox) {
  const int i = ox >> 1;
  if (w <= 2) return near_row[i < w ? i : w - 1];
  const int c = 3 * near_row[i] + far_row[i];
  if (ox & 1) {
    const int j = i + 1 < w ? i + 1 : w - 1;
    const int n = 3 * near_row[j] + far_row[j];
    return (3 * c + n + 7) >> 4;
  }
  const int j = i > 0 ? i - 1 : 0;
  const int n = 3 * near_row[j] + far_row[j];
  return (3 * c + n + 8) >> 4;
}

// ---- YCbCr -> RGB, 16-bit fixed point (JFIF) ----------------------------------------------------------------------
JPG_HD void ycc_to_rgb(int y, int cb, int cr, uint8_t* r, uint8_t* g, uint8_t* b) {
  constexpr int kHalf = 1 << 15;
  const int xcb = cb - 128, xcr = cr - 128;
  const int rr = (91881 * xcr + kHalf) >> 16;           // 1.40200 Cr
  const int bb = (116130 * xcb + kHalf) >> 16;          // 1.77200 Cb
  const int gg = (-22554 * xcb - 46802 * xcr + kHalf) >> 16;  // -0.34414 Cb - 0.71414 Cr
  *r = clamp_u8(y + rr);
  *g = clamp_u8(y + gg);
  *b = clamp_u8(y + bb);
}

// ---- chunk descriptors shared by the host packer (jpeg.cu) and both kernels ------------------------------------------
// One table set: the Huffman and quantisation tables a file's scan uses.  tab[0..1] are DC slots 0 / 1, tab[2..3] AC
// slots 0 / 1; q[c] is component c's table in natural order.
struct alignas(16) TableSet {
  HuffTab tab[4];
  uint16_t q[3][64];
  uint8_t dc[3], ac[3];  // per component: index into tab
};
// One file of a chunk.  Component 0 has hs x vs blocks per MCU (1x1, 2x1, 2x2), components 1, 2 one; a 1-component
// file is coded one block per MCU, so it has hs = vs = 1 and an MCU grid of ceil(W/8) x ceil(H/8).
struct ImageDesc {
  int64_t coef;    // offset of component 0's coefficients in the chunk's int16 scratch; components follow
  int64_t out;     // offset of the cache row in the dataset
  int set;         // table set
  int C, H, W;     // components and size of the file
  int Cs;          // planes of the cache row: 3 replicates a 1-component file
  int hs, vs;      // component 0's sampling factors
  int mcux, mcuy;  // MCU grid
};
// One restart interval: MCUs [mcu0, mcu0 + n) of image `img`, entropy bytes [off, off + len) of the chunk buffer.
struct IntervalDesc {
  int64_t off;
  int len, img, mcu0, n;
};
// One band of MCU rows [mr0, mr1) of image `img` for the IDCT / upsampling / colour kernel.
struct BandDesc {
  int img, mr0, mr1;
};

// blocks of component c: width and height of its block grid; offset of its coefficients relative to ImageDesc::coef
JPG_HD int comp_bw(const ImageDesc& m, int c) { return m.mcux * (c == 0 ? m.hs : 1); }
JPG_HD int comp_bh(const ImageDesc& m, int c) { return m.mcuy * (c == 0 ? m.vs : 1); }
JPG_HD int64_t comp_coef(const ImageDesc& m, int c) {
  const int64_t n0 = (int64_t)comp_bw(m, 0) * comp_bh(m, 0) * 64, n1 = (int64_t)m.mcux * m.mcuy * 64;
  return c == 0 ? 0 : n0 + (c - 1) * n1;
}
JPG_HD int64_t image_coefs(int C, int hs, int vs, int mcux, int mcuy) { return (int64_t)mcux * mcuy * 64 * (hs * vs + (C - 1)); }

// Entropy-decodes one restart interval into coef (the image's int16 scratch, zeroed beforehand).  DC prediction
// starts at 0 for every component (T.81 F.2.1.3.1: at the scan start and after each restart).  Returns false when
// the data is corrupt or ends early.
JPG_HD bool decode_interval(const uint8_t* bytes, const IntervalDesc& iv, const ImageDesc& m, const TableSet& ts, int16_t* coef) {
  BitReader br{bytes + iv.off, bytes + iv.off + iv.len};
  int pred[3] = {0, 0, 0};
  for (int u = iv.mcu0; u < iv.mcu0 + iv.n; ++u) {
    const int mx = u % m.mcux, my = u / m.mcux;
    for (int c = 0; c < m.C; ++c) {
      const int h = c == 0 ? m.hs : 1, v = c == 0 ? m.vs : 1, bw = comp_bw(m, c);
      int16_t* base = coef + comp_coef(m, c);
      for (int by = 0; by < v; ++by)
        for (int bx = 0; bx < h; ++bx) {
          int16_t* blk = base + ((int64_t)(my * v + by) * bw + (mx * h + bx)) * 64;
          if (!decode_block(br, ts.tab[ts.dc[c]], ts.tab[ts.ac[c]], &pred[c], blk)) return false;
        }
    }
  }
  return !br.overrun();
}

// Band geometry: the band holds component 0's sample rows [mr0*8*vs, mr1*8*vs) and chroma block rows [cb0, cb1),
// one more on each side when chroma is subsampled vertically (the triangle filter reads the neighbouring row).
struct BandGeom {
  int y0, y1;     // component 0 sample rows held
  int cb0, cb1;   // chroma block rows held
  int w0, wc;     // plane widths in samples (component 0, chroma)
};
JPG_HD BandGeom band_geom(const ImageDesc& m, int mr0, int mr1) {
  BandGeom g;
  g.y0 = mr0 * 8 * m.vs;
  g.y1 = mr1 * 8 * m.vs;
  g.cb0 = m.vs == 2 && mr0 > 0 ? mr0 - 1 : mr0;
  g.cb1 = m.vs == 2 && mr1 < m.mcuy ? mr1 + 1 : mr1;
  g.w0 = comp_bw(m, 0) * 8;
  g.wc = m.mcux * 8;
  return g;
}
JPG_HD int band_bytes(const ImageDesc& m, int mr0, int mr1) {
  const BandGeom g = band_geom(m, mr0, mr1);
  return (g.y1 - g.y0) * g.w0 + (m.C == 3 ? 2 * (g.cb1 - g.cb0) * 8 * g.wc : 0);
}
// the k-th block of a band: its coefficients and where its 8x8 samples go in the band's planes (plane 0 of
// (y1-y0) x w0 samples, then chroma planes of (cb1-cb0)*8 x wc).  Returns the number of blocks when k is out of range.
JPG_HD int band_blocks(const ImageDesc& m, const BandGeom& g) {
  const int b0 = (g.y1 - g.y0) / 8 * comp_bw(m, 0);
  return m.C == 3 ? b0 + 2 * (g.cb1 - g.cb0) * m.mcux : b0;
}
JPG_HD void band_block(const ImageDesc& m, const BandGeom& g, int k, int* comp, int64_t* coef_off, int* smem_off, int* stride) {
  const int bw0 = comp_bw(m, 0), n0 = (g.y1 - g.y0) / 8 * bw0;
  if (k < n0) {
    const int by = k / bw0, bx = k - by * bw0;
    *comp = 0;
    *coef_off = ((int64_t)(g.y0 / 8 + by) * bw0 + bx) * 64;
    *smem_off = by * 8 * g.w0 + bx * 8;
    *stride = g.w0;
    return;
  }
  k -= n0;
  const int nc = (g.cb1 - g.cb0) * m.mcux, c = 1 + k / nc;
  k -= (c - 1) * nc;
  const int by = k / m.mcux, bx = k - by * m.mcux;
  *comp = c;
  *coef_off = comp_coef(m, c) + ((int64_t)(g.cb0 + by) * m.mcux + bx) * 64;
  *smem_off = (g.y1 - g.y0) * g.w0 + (c - 1) * (g.cb1 - g.cb0) * 8 * g.wc + by * 8 * g.wc + bx * 8;
  *stride = g.wc;
}
// Output sample (y, x) of the image (y inside the band) from the band's planes: Y, or R, G, B of the upsampled,
// colour-converted chroma.  Chroma rows and columns are clamped to the component's downsampled size.
JPG_HD void band_pixel(const ImageDesc& m, const BandGeom& g, const uint8_t* planes, int y, int x, uint8_t* rgb) {
  const int yy = planes[(y - g.y0) * g.w0 + x];
  if (m.C == 1) {
    rgb[0] = rgb[1] = rgb[2] = (uint8_t)yy;
    return;
  }
  const int dsw = (m.W + m.hs - 1) / m.hs, dsh = (m.H + m.vs - 1) / m.vs, pc = (g.cb1 - g.cb0) * 8 * g.wc;
  const uint8_t* cp = planes + (g.y1 - g.y0) * g.w0;
  int ch[2];
  for (int c = 0; c < 2; ++c) {
    const uint8_t* pl = cp + c * pc;
    if (m.vs == 2) {
      const int i = y >> 1;
      int f = (y & 1) ? i + 1 : i - 1;
      f = f < 0 ? 0 : (f >= dsh ? dsh - 1 : f);
      ch[c] = up_h2v2(pl + (i - g.cb0 * 8) * g.wc, pl + (f - g.cb0 * 8) * g.wc, dsw, x);
    } else if (m.hs == 2) {
      ch[c] = up_h2(pl + (y - g.cb0 * 8) * g.wc, dsw, x);
    } else {
      ch[c] = pl[(y - g.cb0 * 8) * g.wc + x];
    }
  }
  ycc_to_rgb(yy, ch[0], ch[1], rgb, rgb + 1, rgb + 2);
}

}  // namespace jpg
