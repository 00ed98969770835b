// The augmented LFW training set built on the GPU (fg_lfw_aug_params, fg_dataset_augment): dataset/generate_dataset.py's
// flip, brightness and affine warp of each 250x250 photo, LFW-crop's 84x84 box and scipy.misc.imresize's Pillow
// BILINEAR resize, from a cache of decoded photos straight into the rows of the training cache.
//
// Row r = i * (1 + n_aug) + a of the output comes from photo i: a = 0 is the photo itself (crop and resize only),
// a = 1..n_aug its augmentations.  The per-pixel arithmetic is k_aug.cuh.  A call:
//   host    validates every descriptor, collects the distinct source rows the warped descriptors read and Pillow's
//           resample coefficients of the destination size (they depend on geometry only), and uploads them with the
//           descriptors in one copy;
//   device  aug_minmax_kernel: min and max of each distinct source row (skimage clips the warp to the input's range);
//           aug_crop_kernel: one CTA per output row.  It warps (or copies) the 84x84xC crop into shared memory as
//           uint8, runs Pillow's horizontal pass into a second shared buffer, and the vertical pass straight into
//           the destination row.  21 KB + at most 21 KB of static shared memory.
#include <algorithm>
#include <cmath>
#include <vector>

#include "fg_internal.h"
#include "k_aug.cuh"

namespace {

constexpr int kMinmaxThreads = 256, kCropThreads = 256;
constexpr int kPlane = aug::kCrop * aug::kCrop;

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the BILINEAR (triangle) filter: output xx reads inputs
// [bounds[2xx], bounds[2xx] + bounds[2xx+1]) with the int32 weights kk[xx * ksize ..]
struct Coeffs {
  int ksize = 0;
  std::vector<int> bounds, kk;
};
Coeffs pillow_coeffs(int in_size, int out_size) {
  Coeffs r;
  const float in0 = 0.f, in1 = (float)in_size;
  const double scale = (double)(in1 - in0) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 1.0 * filterscale;
  r.ksize = (int)ceil(support) * 2 + 1;
  r.bounds.resize(2 * out_size);
  r.kk.assign((size_t)out_size * r.ksize, 0);
  std::vector<double> k(r.ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      double t = ((x + xmin - center + 0.5) * ss);
      if (t < 0.0) t = -t;
      const double w = t < 1.0 ? 1.0 - t : 0.0;
      k[x] = w;
      ww += w;
    }
    for (int x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    for (int x = 0; x < r.ksize; ++x) {
      const double v = x < xmax ? k[x] : 0.0;
      r.kk[(size_t)xx * r.ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << aug::kPrecisionBits)) : (int)(0.5 + v * (1 << aug::kPrecisionBits));
    }
    r.bounds[2 * xx] = xmin;
    r.bounds[2 * xx + 1] = xmax;
  }
  return r;
}

// one CTA per distinct source row: mm[2s], mm[2s+1] = min, max over every byte of row rows[s]
__global__ void __launch_bounds__(kMinmaxThreads) aug_minmax_kernel(const uint8_t* __restrict__ data, int64_t per,
                                                                    const int64_t* __restrict__ rows, uint8_t* __restrict__ mm) {
  const uint8_t* p = data + rows[blockIdx.x] * per;
  unsigned lo = 255, hi = 0;
  if ((per & 3) == 0) {  // the row starts 4-byte aligned
    const uint32_t* p4 = reinterpret_cast<const uint32_t*>(p);
    for (int64_t i = threadIdx.x; i < per / 4; i += blockDim.x) {
      const uint32_t v = __ldg(p4 + i);
      const uint32_t a = __vminu4(v, v >> 16), b = __vmaxu4(v, v >> 16);  // bytes 0, 1: over bytes (0, 2), (1, 3)
      lo = min(lo, min(a & 0xffu, (a >> 8) & 0xffu));
      hi = max(hi, max(b & 0xffu, (b >> 8) & 0xffu));
    }
  } else {
    for (int64_t i = threadIdx.x; i < per; i += blockDim.x) {
      const unsigned v = __ldg(p + i);
      lo = min(lo, v);
      hi = max(hi, v);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  __shared__ unsigned s_lo[kMinmaxThreads / 32], s_hi[kMinmaxThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    s_lo[warp] = lo;
    s_hi[warp] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
      lo = min(lo, s_lo[w]);
      hi = max(hi, s_hi[w]);
    }
    mm[2 * blockIdx.x] = (uint8_t)lo;
    mm[2 * blockIdx.x + 1] = (uint8_t)hi;
  }
}

struct CropArgs {
  const fg_aug* augs;
  const int* slot;          // per descriptor: its source row's entry of mm (warped descriptors only)
  const uint8_t* mm;        // [distinct rows][min, max]
  const int *hb, *hk, *vb, *vk;  // Pillow coefficients: horizontal (Wo outputs), vertical (Ho outputs)
  int kh, kv;
  const uint8_t* src;
  int Cs, Hs, Ws;
  uint8_t* dst;  // the first destination row
  int Ho, Wo;
};

// one CTA per output row
__global__ void __launch_bounds__(kCropThreads, 4) aug_crop_kernel(CropArgs a) {
  __shared__ uint8_t crop[3 * kPlane];  // [Cs][84][84]
  __shared__ uint8_t hor[3 * kPlane];   // [Cs][84][Wo]
  __shared__ double m[9];
  const fg_aug* d = a.augs + blockIdx.x;
  if (threadIdx.x < 9) m[threadIdx.x] = d->m[threadIdx.x];
  __syncthreads();
  const int Cs = a.Cs, Hs = a.Hs, Ws = a.Ws;
  const int64_t plane = (int64_t)Hs * Ws;
  const uint8_t* s = a.src + d->src * (Cs * plane);
  if (!d->warp) {
    for (int i = threadIdx.x; i < Cs * kPlane; i += blockDim.x) {
      const int ch = i / kPlane, yx = i - ch * kPlane, y = yx / aug::kCrop, x = yx - y * aug::kCrop;
      crop[i] = s[ch * plane + (int64_t)(aug::kCropY + y) * Ws + aug::kCropX + x];
    }
  } else {
    const double b = d->brightness;
    const bool flip = d->hflip != 0;
    const int sl = a.slot[blockIdx.x];
    const double lo = aug::as_float(aug::brighten(a.mm[2 * sl], b)), hi = aug::as_float(aug::brighten(a.mm[2 * sl + 1], b));
    for (int i = threadIdx.x; i < kPlane; i += blockDim.x) {
      const int y = i / aug::kCrop, x = i - y * aug::kCrop;
      double c, r;
      if (!aug::sample_point(m, aug::kCropX + x, aug::kCropY + y, &c, &r)) {
        for (int ch = 0; ch < Cs; ++ch) crop[ch * kPlane + i] = aug::clip_store(0.0, lo, hi);
        continue;
      }
      const aug::Taps t = aug::taps(c, r, Hs, Ws);
      const int c0 = t.c0 < 0 ? -1 : (flip ? Ws - 1 - t.c0 : t.c0), c1 = t.c1 < 0 ? -1 : (flip ? Ws - 1 - t.c1 : t.c1);
      for (int ch = 0; ch < Cs; ++ch) {
        const uint8_t* p = s + ch * plane;
        auto px = [&](int rr, int cc) -> double {
          return (rr < 0 || cc < 0) ? 0.0 : aug::as_float(aug::brighten(__ldg(p + (int64_t)rr * Ws + cc), b));
        };
        const double out = aug::bilinear(t, px(t.r0, c0), px(t.r0, c1), px(t.r1, c0), px(t.r1, c1));
        crop[ch * kPlane + i] = aug::clip_store(out, lo, hi);
      }
    }
  }
  __syncthreads();
  const int Ho = a.Ho, Wo = a.Wo;
  for (int i = threadIdx.x; i < Cs * aug::kCrop * Wo; i += blockDim.x) {
    const int row = i / Wo, xo = i - row * Wo;  // row = ch * 84 + y
    const int xmin = __ldg(a.hb + 2 * xo), xmax = __ldg(a.hb + 2 * xo + 1);
    const int* k = a.hk + xo * a.kh;
    const uint8_t* in = crop + row * aug::kCrop + xmin;
    int ss = 1 << (aug::kPrecisionBits - 1);
    for (int x = 0; x < xmax; ++x) ss += (int)in[x] * __ldg(k + x);
    hor[i] = aug::clip8(ss);
  }
  __syncthreads();
  uint8_t* out = a.dst + (int64_t)blockIdx.x * Cs * Ho * Wo;
  for (int i = threadIdx.x; i < Cs * Ho * Wo; i += blockDim.x) {
    const int r = i / Wo, xo = i - r * Wo, ch = r / Ho, yo = r - ch * Ho;
    const int ymin = __ldg(a.vb + 2 * yo), ymax = __ldg(a.vb + 2 * yo + 1);
    const int* k = a.vk + yo * a.kv;
    const uint8_t* in = hor + (ch * aug::kCrop + ymin) * Wo + xo;
    int ss = 1 << (aug::kPrecisionBits - 1);
    for (int y = 0; y < ymax; ++y) ss += (int)in[y * Wo] * __ldg(k + y);
    out[i] = aug::clip8(ss);
  }
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

}  // namespace

extern "C" {

int fg_lfw_aug_params(uint64_t seed, int64_t first_src, int64_t n_src, int n_aug, int src_h, int src_w, fg_aug* out) {
  FG_REQUIRE(out && first_src >= 0 && n_src >= 1 && n_aug >= 0 && n_aug <= 999 && src_h >= 1 && src_w >= 1,
             "fg_lfw_aug_params: need out, first_src >= 0, n_src >= 1, 0 <= n_aug <= 999, positive sizes");
  // ImageAugmenter.create_aug_matrices centres on (int(width/2), int(height/2)), and augment() passes shape[0] (the
  // height) as the width
  const double shx = (double)(src_h / 2), shy = (double)(src_w / 2);
  const double kDeg = M_PI / 180.0;  // np.deg2rad
  for (int64_t i = first_src; i < first_src + n_src; ++i) {
    for (int a = 0; a <= n_aug; ++a) {
      fg_aug& g = out[(i - first_src) * (1 + n_aug) + a];
      g.src = i;
      g.warp = a > 0;
      for (int k = 0; k < 9; ++k) g.m[k] = (k % 4 == 0) ? 1.0 : 0.0;
      g.hflip = 0;
      g.brightness = 1.0;
      if (a == 0) continue;
      // generate_dataset.py's distributions: scale U[0.82, 1.10) on both axes, randint(-8, 8) degrees, no shear,
      // randint(-5, 5) px on each axis, hflip with p = 1/2, brightness U[0.9, 1.1)
      const double s = 0.82 + (1.10 - 0.82) * aug::draw(seed, i, a, 0);
      const double rho = aug::draw_int(seed, i, a, 1, -8, 8) * kDeg;
      const double tx = aug::draw_int(seed, i, a, 2, -5, 5), ty = aug::draw_int(seed, i, a, 3, -5, 5);
      g.hflip = aug::draw(seed, i, a, 4) < 0.5;
      g.brightness = 0.9 + (1.1 - 0.9) * aug::draw(seed, i, a, 5);
      // forward F = T(+shift) . A . T(-shift), A = [[s cos, -s sin, tx], [s sin, s cos, ty], [0, 0, 1]]
      const double A0 = s * cos(rho), A1 = -(s * sin(rho)), A3 = s * sin(rho), A4 = s * cos(rho);
      const double F2 = -(A0 * shx + A1 * shy) + tx + shx, F5 = -(A3 * shx + A4 * shy) + ty + shy;
      // its inverse in closed form, third row exactly [0, 0, 1]
      const double det = A0 * A4 - A1 * A3;
      g.m[0] = A4 / det;
      g.m[1] = -A1 / det;
      g.m[2] = (A1 * F5 - A4 * F2) / det;
      g.m[3] = -A3 / det;
      g.m[4] = A0 / det;
      g.m[5] = (A3 * F2 - A0 * F5) / det;
    }
  }
  return FG_OK;
}

int fg_dataset_augment(fg_dataset* src, fg_dataset* dst, int64_t dst_first, const fg_aug* augs, int64_t n) {
  if (!src || !src->c || !dst || !dst->c) {
    fg_set_error("fg_dataset_augment: null fg_dataset");
    return FG_ERR_INVALID;
  }
  FG_REQUIRE(src->c == dst->c, "fg_dataset_augment: the two caches belong to different contexts");
  FG_REQUIRE(augs && n >= 1 && n <= INT32_MAX && dst_first >= 0 && dst_first + n <= dst->N,
             "fg_dataset_augment: rows [%lld, %lld) outside the destination's [0, %lld)", (long long)dst_first,
             (long long)(dst_first + n), (long long)dst->N);
  FG_REQUIRE(src->Cs == dst->Cs, "fg_dataset_augment: %d source channels, %d destination channels", src->Cs, dst->Cs);
  FG_REQUIRE(src->Hs >= aug::kCropY + aug::kCrop && src->Ws >= aug::kCropX + aug::kCrop,
             "fg_dataset_augment: the crop box (rows %d..%d, cols %d..%d) is not inside the %dx%d source", aug::kCropY,
             aug::kCropY + aug::kCrop - 1, aug::kCropX, aug::kCropX + aug::kCrop - 1, src->Ws, src->Hs);
  FG_REQUIRE(dst->Hs >= 1 && dst->Hs <= aug::kCrop && dst->Ws >= 1 && dst->Ws <= aug::kCrop,
             "fg_dataset_augment: destination %dx%d: each side must be in [1, %d] (the crop is only shrunk)", dst->Ws,
             dst->Hs, aug::kCrop);
  std::vector<int64_t> rows;
  for (int64_t i = 0; i < n; ++i) {
    const fg_aug& g = augs[i];
    FG_REQUIRE(g.src >= 0 && g.src < src->N, "fg_dataset_augment: descriptor %lld: source row %lld outside [0, %lld)",
               (long long)i, (long long)g.src, (long long)src->N);
    FG_REQUIRE((g.warp == 0 || g.warp == 1) && (g.hflip == 0 || g.hflip == 1),
               "fg_dataset_augment: descriptor %lld: warp and hflip must be 0 or 1", (long long)i);
    FG_REQUIRE(std::isfinite(g.brightness) && g.brightness >= 0.0,
               "fg_dataset_augment: descriptor %lld: brightness %g is not finite and >= 0", (long long)i, g.brightness);
    for (int k = 0; k < 9; ++k)
      FG_REQUIRE(std::isfinite(g.m[k]), "fg_dataset_augment: descriptor %lld: m[%d] is not finite", (long long)i, k);
    if (g.warp) rows.push_back(g.src);
  }
  std::sort(rows.begin(), rows.end());
  rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
  std::vector<int> slot(n, 0);
  for (int64_t i = 0; i < n; ++i)
    if (augs[i].warp) slot[i] = (int)(std::lower_bound(rows.begin(), rows.end(), augs[i].src) - rows.begin());
  const Coeffs h = pillow_coeffs(aug::kCrop, dst->Ws), v = pillow_coeffs(aug::kCrop, dst->Hs);

  // one device buffer: [descriptors][slots][rows][h bounds][h weights][v bounds][v weights][min/max]
  const size_t o_slot = align16(sizeof(fg_aug) * n);
  const size_t o_rows = o_slot + align16(sizeof(int) * n);
  const size_t o_hb = o_rows + align16(sizeof(int64_t) * rows.size());
  const size_t o_hk = o_hb + align16(sizeof(int) * h.bounds.size());
  const size_t o_vb = o_hk + align16(sizeof(int) * h.kk.size());
  const size_t o_vk = o_vb + align16(sizeof(int) * v.bounds.size());
  const size_t o_mm = o_vk + align16(sizeof(int) * v.kk.size());
  const size_t total = o_mm + 2 * rows.size() + 16;
  std::vector<uint8_t> host(o_mm);
  memcpy(host.data(), augs, sizeof(fg_aug) * n);
  memcpy(host.data() + o_slot, slot.data(), sizeof(int) * n);
  if (!rows.empty()) memcpy(host.data() + o_rows, rows.data(), sizeof(int64_t) * rows.size());
  memcpy(host.data() + o_hb, h.bounds.data(), sizeof(int) * h.bounds.size());
  memcpy(host.data() + o_hk, h.kk.data(), sizeof(int) * h.kk.size());
  memcpy(host.data() + o_vb, v.bounds.data(), sizeof(int) * v.bounds.size());
  memcpy(host.data() + o_vk, v.kk.data(), sizeof(int) * v.kk.size());

  fg_ctx* c = dst->c;
  FG_CUDA(cudaSetDevice(c->device));
  uint8_t* buf = nullptr;
  FG_CUDA(cudaMalloc((void**)&buf, total));
  int rc = FG_OK;
  auto fail = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess && rc == FG_OK) {
      fg_set_error("fg_dataset_augment: %s: %s", what, cudaGetErrorString(e));
      rc = FG_ERR_CUDA;
    }
    return e != cudaSuccess;
  };
  do {
    if (fail(cudaMemcpyAsync(buf, host.data(), o_mm, cudaMemcpyHostToDevice, c->stream), "upload")) break;
    const int64_t per = (int64_t)src->Cs * src->Hs * src->Ws;
    if (!rows.empty()) {
      aug_minmax_kernel<<<(int)rows.size(), kMinmaxThreads, 0, c->stream>>>(src->data, per,
                                                                            reinterpret_cast<const int64_t*>(buf + o_rows), buf + o_mm);
      c->launches++;
      if (fail(cudaGetLastError(), "aug_minmax_kernel")) break;
    }
    CropArgs a;
    a.augs = reinterpret_cast<const fg_aug*>(buf);
    a.slot = reinterpret_cast<const int*>(buf + o_slot);
    a.mm = buf + o_mm;
    a.hb = reinterpret_cast<const int*>(buf + o_hb);
    a.hk = reinterpret_cast<const int*>(buf + o_hk);
    a.vb = reinterpret_cast<const int*>(buf + o_vb);
    a.vk = reinterpret_cast<const int*>(buf + o_vk);
    a.kh = h.ksize;
    a.kv = v.ksize;
    a.src = src->data;
    a.Cs = src->Cs;
    a.Hs = src->Hs;
    a.Ws = src->Ws;
    a.dst = dst->data + dst_first * (int64_t)dst->Cs * dst->Hs * dst->Ws;
    a.Ho = dst->Hs;
    a.Wo = dst->Ws;
    aug_crop_kernel<<<(int)n, kCropThreads, 0, c->stream>>>(a);
    c->launches++;
    if (fail(cudaGetLastError(), "aug_crop_kernel")) break;
    fail(cudaStreamSynchronize(c->stream), "synchronize");
  } while (0);
  cudaFree(buf);
  return rc;
}

}  // extern "C"
