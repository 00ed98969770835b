// Per-pixel, per-block and per-symbol arithmetic of the baseline JPEG encoder (jpeg_enc.cu): what Pillow's
// Image.save(f, "JPEG", quality=q) computes at its defaults through libjpeg-turbo, written from ITU-T T.81 (Annex K
// tables, F.1.2 Huffman encoding) and the published 13-bit fixed-point forward DCT (the JDCT_ISLOW method).
//   colour       16-bit fixed-point RGB -> YCbCr (JFIF), rounding Y up at one half and Cb / Cr just below it
//   edges        columns replicated to the MCU width; rows replicated to an even height, downsampled 2x2 with the
//                alternating bias 1, 2, 1, 2, ..., then each plane replicated to its iMCU height from its own last row
//   DCT          islow forward DCT of samples - 128 (8x the true DCT), quantised as sign(x) ((|x| + 4q) / (8q))
//   dummy blocks the blocks of a luma MCU past the image: zero AC, the DC of the previous block of the MCU
// Everything is integer arithmetic, so the device encoder is bitwise reproducible; tests/jpeg_enc_ref.py restates
// these rules and is held to Pillow's bytes.  __host__ __device__ throughout, as k_jpeg.cuh.
#pragma once
#include <cstdint>

#include "fg_internal.h"
#include "k_jpeg.cuh"

namespace jpg {

// ---- T.81 Annex K tables -----------------------------------------------------------------------------------------
// K.1 quantisation bases, natural order: [0] luma, [1] chroma
static const uint8_t kBaseQ[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
     14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
     47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
// K.3 Huffman tables: BITS[1..16] and HUFFVAL of [0] DC luma, [1] AC luma, [2] DC chroma, [3] AC chroma (the DHT
// order Pillow writes)
static const uint8_t kStdBits[4][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                        {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                        {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},
                                        {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t kStdValsDC[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kStdValsACLuma[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t kStdValsACChroma[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
    0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
    0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
    0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
inline const uint8_t* std_vals(int t) { return t == 1 ? kStdValsACLuma : t == 3 ? kStdValsACChroma : kStdValsDC; }

// jpeg_set_quality(q, force_baseline = TRUE): table t (0 luma, 1 chroma) in natural order
inline void quant_table(int quality, int t, uint16_t out[64]) {
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int i = 0; i < 64; ++i) {
    int v = (kBaseQ[t][i] * scale + 50) / 100;
    out[i] = (uint16_t)(v < 1 ? 1 : (v > 255 ? 255 : v));
  }
}
// the canonical codes of table t (T.81 C.2): code[sym] = (length << 16) | code, 0 for a symbol the table lacks
inline void huff_codes(int t, uint32_t code_of[256]) {
  for (int i = 0; i < 256; ++i) code_of[i] = 0;
  const uint8_t* vals = std_vals(t);
  uint32_t code = 0;
  int k = 0;
  for (int l = 1; l <= 16; ++l) {
    for (int i = 0; i < kStdBits[t][l - 1]; ++i) code_of[vals[k++]] = ((uint32_t)l << 16) | code++;
    code <<= 1;
  }
}

// ---- geometry of one encode call: every row of the cache has the same size ----------------------------------------
// Cs = 3: one YCbCr scan, luma 2x2 blocks per MCU, chroma 1x1 (4:2:0); Cs = 1: one grayscale block per MCU.  The
// coefficients of a row follow the decoder's scratch layout (ImageDesc::coef, comp_coef): component 0 on its
// MCU-padded grid of mcux*hs x mcuy*vs blocks, then each chroma component on mcux x mcuy blocks.
struct EncGeom {
  int Cs, H, W;
  int hs, vs;          // luma blocks per MCU
  int mcux, mcuy;      // MCU grid
  int bwr, bhr;        // luma blocks inside the image: ceil(W/8) x ceil(H/8); the rest of the grid are dummies
  int rows, bands;     // MCU rows per band of the forward kernel, bands per row of the cache
  int nblk;            // blocks per row of the cache (= image_coefs / 64)
  uint16_t q[2][64];   // quantisation tables, natural order: luma, chroma
};

// ---- colour and sampling -----------------------------------------------------------------------------------------
JPG_HD void rgb_to_ycc(int r, int g, int b, uint8_t* y, uint8_t* cb, uint8_t* cr) {
  constexpr int kHalf = 1 << 15, kCbCrOff = (128 << 16) + kHalf - 1;
  *y = (uint8_t)((19595 * r + 38470 * g + 7471 * b + kHalf) >> 16);            // 0.29900, 0.58700, 0.11400
  *cb = (uint8_t)((-11059 * r - 21709 * g + 32768 * b + kCbCrOff) >> 16);      // -0.16874, -0.33126, 0.5
  *cr = (uint8_t)((32768 * r - 27439 * g - 5329 * b + kCbCrOff) >> 16);        // 0.5, -0.41869, -0.08131
}

// ---- forward DCT: LL&M, 13-bit constants, 2 extra bits of precision between the passes -----------------------------
// one pass on d[0], d[step], ..., d[7 step]: the first keeps PASS1_BITS of extra precision, the second removes them
template <bool kFirst>
JPG_HD void fdct_1d(int32_t* d, int step) {
  const int32_t t0 = d[0] + d[7 * step], t7 = d[0] - d[7 * step];
  const int32_t t1 = d[step] + d[6 * step], t6 = d[step] - d[6 * step];
  const int32_t t2 = d[2 * step] + d[5 * step], t5 = d[2 * step] - d[5 * step];
  const int32_t t3 = d[3 * step] + d[4 * step], t4 = d[3 * step] - d[4 * step];
  const int32_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int sh = kFirst ? kConstBits - kPass1Bits : kConstBits + kPass1Bits;
  if (kFirst) {
    d[0] = (t10 + t11) * (1 << kPass1Bits);
    d[4 * step] = (t10 - t11) * (1 << kPass1Bits);
  } else {
    d[0] = descale(t10 + t11, kPass1Bits);
    d[4 * step] = descale(t10 - t11, kPass1Bits);
  }
  const int32_t z1 = (t12 + t13) * c0_541196100;
  d[2 * step] = descale(z1 + t13 * c0_765366865, sh);
  d[6 * step] = descale(z1 - t12 * c1_847759065, sh);
  int32_t y1 = t4 + t7, y2 = t5 + t6, y3 = t4 + t6, y4 = t5 + t7;
  const int32_t z5 = (y3 + y4) * c1_175875602;
  const int32_t u4 = t4 * c0_298631336, u5 = t5 * c2_053119869, u6 = t6 * c3_072711026, u7 = t7 * c1_501321110;
  y1 *= -c0_899976223;
  y2 *= -c2_562915447;
  y3 = y3 * -c1_961570560 + z5;
  y4 = y4 * -c0_390180644 + z5;
  d[7 * step] = descale(u4 + y1 + y3, sh);
  d[5 * step] = descale(u5 + y2 + y4, sh);
  d[3 * step] = descale(u6 + y2 + y3, sh);
  d[step] = descale(u7 + y1 + y4, sh);
}
// d[64] row-major samples - 128 -> 8x the DCT coefficients, in place
JPG_HD void fdct_islow(int32_t* d) {
  for (int r = 0; r < 8; ++r) fdct_1d<true>(d + 8 * r, 1);
  for (int c = 0; c < 8; ++c) fdct_1d<false>(d + c, 8);
}
JPG_HD int quantize(int32_t x, int q) {
  const int32_t q8 = 8 * q, a = ((x < 0 ? -x : x) + 4 * q) / q8;
  return x < 0 ? -a : a;
}

// ---- entropy coding --------------------------------------------------------------------------------------------
JPG_HD int magnitude_bits(int v) {  // T.81 F.1.2.1: the size category of v
  const unsigned a = (unsigned)(v < 0 ? -v : v);
#ifdef __CUDA_ARCH__
  return 32 - __clz((int)a);
#else
  return a ? 32 - __builtin_clz(a) : 0;
#endif
}
// Block s of a row in scan order (interleaved MCUs: the hs*vs luma blocks row by row, then Cb, Cr): its component,
// the offset of its coefficients, and that of the previous block of the same component in scan order (-1: the
// first, predicted from 0)
JPG_HD int scan_block(const EncGeom& g, int s, int64_t* off, int64_t* prev) {
  const int per = g.hs * g.vs + g.Cs - 1, u = s / per, j = s - u * per;
  const int bw0 = g.mcux * g.hs;
  auto at = [&](int uu, int jj) -> int64_t {
    const int x = uu % g.mcux, y = uu / g.mcux;
    if (jj < g.hs * g.vs) return ((int64_t)(y * g.vs + jj / g.hs) * bw0 + x * g.hs + jj % g.hs) * 64;
    return (int64_t)bw0 * g.mcuy * g.vs * 64 + (int64_t)(jj - g.hs * g.vs) * g.mcux * g.mcuy * 64 +
           ((int64_t)y * g.mcux + x) * 64;
  };
  *off = at(u, j);
  if (j > 0 && j < g.hs * g.vs) *prev = at(u, j - 1);
  else if (u > 0) *prev = at(u - 1, j < g.hs * g.vs ? g.hs * g.vs - 1 : j);
  else *prev = -1;
  return j < g.hs * g.vs ? 0 : j - g.hs * g.vs + 1;
}
// Huffman-codes one block (coefficients in natural order, DC predicted from `pred`) into sink.put(bits, n), n <= 16
template <typename Sink>
JPG_HD void huff_block(const int16_t* blk, int pred, const uint32_t* dc, const uint32_t* ac, Sink& sink) {
  const int diff = blk[0] - pred;
  int s = magnitude_bits(diff);
  sink.put(dc[s] & 0xffff, (int)(dc[s] >> 16));
  if (s) sink.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1), s);
  int run = 0;
  for (int k = 1; k < 64; ++k) {
    const int v = blk[natural_of(k)];
    if (!v) {
      ++run;
      continue;
    }
    for (; run > 15; run -= 16) sink.put(ac[0xf0] & 0xffff, (int)(ac[0xf0] >> 16));
    s = magnitude_bits(v);
    const uint32_t c = ac[(run << 4) | s];
    sink.put(c & 0xffff, (int)(c >> 16));
    sink.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1), s);
    run = 0;
  }
  if (run) sink.put(ac[0] & 0xffff, (int)(ac[0] >> 16));
}
// the most bits one block can take: DC code + 11 bits, then 63 AC codes of at most 16 + 10 bits
constexpr int kMaxBlockBits = 11 + 11 + 63 * 26;
struct BitCount {
  int n = 0;
  JPG_HD void put(uint32_t, int k) { n += k; }
};

}  // namespace jpg

// The decoder's IDCT / colour kernel over descriptors already on the device (jpeg.cu), for the encoder's round trip
int jpeg_idct_launch(fg_ctx* c, const jpg::TableSet* sets, const jpg::ImageDesc* imgs, const jpg::BandDesc* bands, int n_bands,
                     int smem, const int16_t* coef, uint8_t* data);
// MCU rows per band of that kernel for an image of this shape (the decoder's budget), and the band's shared memory
int jpeg_idct_band_rows(const jpg::ImageDesc& m, int* smem);
