// Per-pixel arithmetic of the LFW augmentation (augment.cu), restated from dataset/generate_dataset.py and
// ImageAugmenter.py: the parameter draws, the scikit-image warp of one output pixel and Pillow's fixed-point BILINEAR
// resample.  tests/aug_ref.py restates every step in numpy, op for op.
//
// The warp follows skimage.transform.warp(img, inverse_map, mode="constant") at order 1 (cval 0, clip on), evaluated
// in float64 with every product and sum rounded on its own (no FMA contraction), as the compiled Cython loop does.
// PARITY UNPINNED (no scikit-image here).  The resample follows Pillow's Image.resize(size, BILINEAR) (what
// scipy.misc.imresize called) and is pinned against Pillow by tests/test_augment_cpu.py.
#pragma once
#include <cmath>
#include <cstdint>

#include "fg_b200.h"

namespace aug {

// LFW-crop's box (http://conradsanderson.id.au/lfwcrop/): rows 92..175, cols 83..166 of the 250x250 photo
constexpr int kCropY = 92, kCropX = 83, kCrop = 84;
constexpr int kPrecisionBits = 22;  // Pillow's PRECISION_BITS for 8-bit images (32 - 8 - 2)

#ifdef __CUDACC__
#define AUG_HD __host__ __device__ __forceinline__
#else
#define AUG_HD inline
#endif

AUG_HD double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
AUG_HD double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
AUG_HD double dsub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

// np.clip(v * b, 0, 255).astype(np.uint8)
AUG_HD uint8_t brighten(int v, double b) {
  const double x = dmul((double)v, b);
  return (uint8_t)(x < 0.0 ? 0.0 : (x > 255.0 ? 255.0 : x));
}
// img_as_float: a multiply by the reciprocal, not a division
AUG_HD double as_float(int u) { return dmul((double)u, 1.0 / 255.0); }

// The sample point (c, r) of output pixel (x, y) under the inverse map m (row-major 3x3), or false when it is not
// finite (a projective map whose z reaches 0 there: the pixel is cval)
AUG_HD bool sample_point(const double* m, int x, int y, double* c, double* r) {
  const double xx = dadd(dadd(dmul(m[0], x), dmul(m[1], y)), m[2]);
  const double yy = dadd(dadd(dmul(m[3], x), dmul(m[4], y)), m[5]);
  if (m[6] == 0.0 && m[7] == 0.0 && m[8] == 1.0) {
    *c = xx;
    *r = yy;
  } else {
    const double zz = dadd(dadd(dmul(m[6], x), dmul(m[7], y)), m[8]);
    *c = xx / zz;
    *r = yy / zz;
  }
  return std::isfinite(*c) && std::isfinite(*r);
}

// The bilinear taps of a finite sample point: rows r0, r1 and cols c0, c1 (-1 when outside the H x W image, i.e.
// cval) and the weights dr, dc
struct Taps {
  int r0, r1, c0, c1;
  double dr, dc;
};
AUG_HD int tap(double v, int n) { return (v >= 0.0 && v < (double)n) ? (int)v : -1; }
AUG_HD Taps taps(double c, double r, int H, int W) {
  Taps t;
  const double fr = floor(r), fc = floor(c);
  t.dr = dsub(r, fr);
  t.dc = dsub(c, fc);
  t.r0 = tap(fr, H);
  t.r1 = tap(ceil(r), H);
  t.c0 = tap(fc, W);
  t.c1 = tap(ceil(c), W);
  return t;
}
// out = (1-dr)*((1-dc)*tl + dc*tr) + dr*((1-dc)*bl + dc*br), each operation rounded
AUG_HD double bilinear(const Taps& t, double tl, double tr, double bl, double br) {
  const double ec = dsub(1.0, t.dc), er = dsub(1.0, t.dr);
  const double top = dadd(dmul(ec, tl), dmul(t.dc, tr));
  const double bot = dadd(dmul(ec, bl), dmul(t.dc, br));
  return dadd(dmul(er, top), dmul(t.dr, bot));
}
// skimage's output clip to the input's [lo, hi]; when cval 0 lies outside it (lo > 0) exact zeros stay 0.  Then
// np.array(out * 255, dtype=np.uint8).
AUG_HD uint8_t clip_store(double out, double lo, double hi) {
  if (!(out == 0.0 && lo > 0.0)) out = out < lo ? lo : (out > hi ? hi : out);
  return (uint8_t)dmul(out, 255.0);
}

// Pillow's clip8 of a fixed-point accumulator
AUG_HD uint8_t clip8(int v) {
  v >>= kPrecisionBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// ---- parameter draws (host) --------------------------------------------------------------------------------------
AUG_HD uint64_t mix64(uint64_t x) {  // splitmix64's finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// draw k of augmentation a of source photo i: uniform in [0, 1) with 53 bits
AUG_HD double draw(uint64_t seed, int64_t i, int a, int k) {
  const uint64_t key = mix64(mix64(mix64(seed) ^ (uint64_t)i) ^ (uint64_t)a);
  return (double)(mix64(key + (uint64_t)k) >> 11) * 0x1.0p-53;
}
// random.randint(lo, hi)
AUG_HD int draw_int(uint64_t seed, int64_t i, int a, int k, int lo, int hi) {
  const int v = lo + (int)(draw(seed, i, a, k) * (double)(hi - lo + 1));
  return v > hi ? hi : v;
}

}  // namespace aug
