// Bandwidth-bound kernels used by the coarse-to-fine nets (models_c2f.lua) and by the stand-alone L-op
// entry points: table ops (JoinTable / CAddTable), nn.SpatialMaxPooling(2,2), nn.Dropout / nn.SpatialDropout,
// nn.SpatialUpSamplingNearest(2), nn.SpatialAveragePooling(2,2,2,2), nn.Sigmoid.
// NHWC variants feed the fused nets (channels fastest => a warp reads consecutive channels of one pixel);
// NCHW variants serve the nn.Module boundary directly, without a layout round trip.
#include <cmath>

#include "fg_internal.h"
#include "k_f16split.cuh"
#include "k_misc.h"

#define LAUNCH_CHECK(c)                 \
  do {                                  \
    (c)->launches++;                    \
    FG_CUDA(cudaGetLastError());        \
  } while (0)

namespace {
inline int grid_for(int64_t n, int block, int cap = 132 * 16) {
  int64_t g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}
#define GRID_STRIDE(i, n) \
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// nn.JoinTable(2,2) of {noise [B][1][HW], cond [B][C][HW]} written as NHWC [B][HW][1+C]   (models_c2f.lua:116)
__global__ void join_to_nhwc_kernel(const float* __restrict__ noise, const float* __restrict__ cond, float* __restrict__ out,
                                    int B, int C, int HW) {
  const int C1 = C + 1;
  const int64_t n = (int64_t)B * HW * C1;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C1);
    const int64_t r = i / C1;
    const int q = (int)(r % HW);
    const int64_t b = r / HW;
    out[i] = ch == 0 ? noise[b * HW + q] : cond[(b * C + (ch - 1)) * HW + q];
  }
}
__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int64_t n) {
  GRID_STRIDE(i, n) out[i] = a[i] + b[i];
}

// first strict maximum in row-major window order (THNN SpatialMaxPooling: `val > maxval`)
__device__ __forceinline__ int argmax4(float v0, float v1, float v2, float v3, float* best) {
  int j = 0;
  float m = v0;
  if (v1 > m) { m = v1; j = 1; }
  if (v2 > m) { m = v2; j = 2; }
  if (v3 > m) { m = v3; j = 3; }
  *best = m;
  return j;
}
__global__ void maxpool2_fwd_nhwc_kernel(const float* __restrict__ h, float* __restrict__ p, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = (int64_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo);
    r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    const int64_t base = ((b * H + 2 * yo) * W + 2 * xo) * C + ch, rs = (int64_t)W * C;
    float m;
    argmax4(h[base], h[base + C], h[base + rs], h[base + rs + C], &m);
    p[i] = m;
  }
}
__global__ void maxpool2_bwd_nhwc_kernel(const float* __restrict__ dp, const float* __restrict__ h, float* __restrict__ dh,
                                         int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = (int64_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo);
    r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    const int64_t base = ((b * H + 2 * yo) * W + 2 * xo) * C + ch, rs = (int64_t)W * C;
    float m;
    const int j = argmax4(h[base], h[base + C], h[base + rs], h[base + rs + C], &m);
    const float g = dp[i];
    dh[base] = j == 0 ? g : 0.f;
    dh[base + C] = j == 1 ? g : 0.f;
    dh[base + rs] = j == 2 ? g : 0.f;
    dh[base + rs + C] = j == 3 ? g : 0.f;
  }
}
// y[b][q][ch] = x * mask[b*stride + moff + ch*HW + q] * scale  (the mask follows the reference's NCHW element order)
__global__ void dropout_nhwc_kernel(const float* __restrict__ x, const float* __restrict__ masks, int64_t stride, int moff,
                                    int HW, int C, float scale, float* __restrict__ y, int B) {
  const int64_t n = (int64_t)B * HW * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    const int64_t r = i / C;
    const int q = (int)(r % HW);
    const int64_t b = r / HW;
    y[i] = x[i] * masks[b * stride + moff + (int64_t)ch * HW + q] * scale;
  }
}
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__global__ void bernoulli_keep_kernel(float* __restrict__ out, int64_t n, uint64_t seed, float p_drop,
                                      const uint64_t* __restrict__ seed_dev) {
  if (seed_dev) seed += *seed_dev * 2;  // the step seed lives in device memory (captured steps), see k_masks_generate
  GRID_STRIDE(i, n) {
    const uint64_t r = splitmix64(seed * 0x100000001B3ull + (uint64_t)i);
    const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
    out[i] = u >= p_drop ? 1.f : 0.f;
  }
}

// ---- NCHW (nn.Module boundary) -------------------------------------------------------------------
__global__ void up2_fwd_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t BC, int H, int W) {
  const int H2 = 2 * H, W2 = 2 * W;
  const int64_t n = BC * H2 * W2;
  GRID_STRIDE(i, n) {
    const int xo = (int)(i % W2);
    const int64_t r = i / W2;
    const int yo = (int)(r % H2);
    const int64_t bc = r / H2;
    y[i] = x[(bc * H + (yo >> 1)) * W + (xo >> 1)];
  }
}
__global__ void up2_bwd_nchw_kernel(const float* __restrict__ dy, float* __restrict__ dx, int64_t BC, int H, int W) {
  const int W2 = 2 * W;
  const int64_t n = BC * H * W;
  GRID_STRIDE(i, n) {
    const int xi = (int)(i % W);
    const int64_t r = i / W;
    const int yi = (int)(r % H);
    const int64_t bc = r / H;
    const int64_t base = (bc * 2 * H + 2 * yi) * W2 + 2 * xi;
    dx[i] = (dy[base] + dy[base + 1]) + (dy[base + W2] + dy[base + W2 + 1]);
  }
}
// H, W are the INPUT sizes of the pooling layer
__global__ void avgpool2_fwd_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t BC, int H, int W) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = BC * Ho * Wo;
  GRID_STRIDE(i, n) {
    const int xo = (int)(i % Wo);
    const int64_t r = i / Wo;
    const int yo = (int)(r % Ho);
    const int64_t bc = r / Ho;
    const int64_t base = (bc * H + 2 * yo) * W + 2 * xo;
    y[i] = (x[base] + x[base + 1] + x[base + W] + x[base + W + 1]) * 0.25f;
  }
}
__global__ void avgpool2_bwd_nchw_kernel(const float* __restrict__ dy, float* __restrict__ dx, int64_t BC, int H, int W) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = BC * H * W;
  GRID_STRIDE(i, n) {
    const int xi = (int)(i % W);
    const int64_t r = i / W;
    const int yi = (int)(r % H);
    const int64_t bc = r / H;
    dx[i] = (yi < 2 * Ho && xi < 2 * Wo) ? dy[(bc * Ho + (yi >> 1)) * Wo + (xi >> 1)] * 0.25f : 0.f;
  }
}
__global__ void maxpool2_fwd_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t BC, int H, int W) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = BC * Ho * Wo;
  GRID_STRIDE(i, n) {
    const int xo = (int)(i % Wo);
    const int64_t r = i / Wo;
    const int yo = (int)(r % Ho);
    const int64_t bc = r / Ho;
    const int64_t base = (bc * H + 2 * yo) * W + 2 * xo;
    float m;
    argmax4(x[base], x[base + 1], x[base + W], x[base + W + 1], &m);
    y[i] = m;
  }
}
__global__ void maxpool2_bwd_nchw_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx,
                                         int64_t BC, int H, int W) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t n = BC * H * W;
  GRID_STRIDE(i, n) {
    const int xi = (int)(i % W);
    const int64_t r = i / W;
    const int yi = (int)(r % H);
    const int64_t bc = r / H;
    float g = 0.f;
    if (yi < 2 * Ho && xi < 2 * Wo) {
      const int yo = yi >> 1, xo = xi >> 1;
      const int64_t base = (bc * H + 2 * yo) * W + 2 * xo;
      float m;
      const int j = argmax4(x[base], x[base + 1], x[base + W], x[base + W + 1], &m);
      if (j == ((yi & 1) << 1 | (xi & 1))) g = dy[(bc * Ho + yo) * Wo + xo];
    }
    dx[i] = g;
  }
}
// inner = HW for nn.SpatialDropout (one flag per (n,c) plane), 1 for nn.Dropout (one flag per element)
__global__ void dropout_nchw_kernel(const float* __restrict__ x, const float* __restrict__ mask, float scale, int inner,
                                    float* __restrict__ y, int64_t n) {
  GRID_STRIDE(i, n) y[i] = x[i] * mask[i / inner] * scale;
}
__global__ void scale_kernel(const float* __restrict__ x, float scale, float* __restrict__ y, int64_t n) {
  GRID_STRIDE(i, n) y[i] = x[i] * scale;
}

// ---- channel padding around the tensor-core kernels (layers whose small side has < 64 channels) ----------
// x = hi + lo with hi exactly representable in TF32 (round to nearest on the 13 dropped mantissa bits)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  const uint32_t b = __float_as_uint(x);
  hi = __uint_as_float((b + 0x1000u) & 0xFFFFE000u);
  lo = x - hi;
}
// src [P][Cs] -> hi/lo [P][Cp], channels >= Cs are zero
__global__ void pad_split_kernel(const float* __restrict__ src, float* __restrict__ hi, float* __restrict__ lo, int64_t P,
                                 int Cs, int Cp) {
  const int64_t n = P * Cp;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % Cp);
    float h = 0.f, l = 0.f;
    if (ch < Cs) split_tf32(src[(i / Cp) * Cs + ch], h, l);
    hi[i] = h;
    lo[i] = l;
  }
}
// the same into the 3xFP16 split (halves), values scaled by the power of two derived from amax_slot[0] (tc_amax)
__global__ void pad_split_h_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, int64_t P,
                                   int Cs, int Cp, float* __restrict__ amax_slot) {
  const float s = amax_slot ? scale_for_amax(amax_slot[0]) : 1.f;
  if (amax_slot && blockIdx.x == 0 && threadIdx.x == 0) amax_slot[1] = 1.f / s;
  const int64_t n = P * Cp;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % Cp);
    __half h = __float2half_rn(0.f), l = h;
    if (ch < Cs) split_f16(src[(i / Cp) * Cs + ch] * s, h, l);
    hi[i] = h;
    lo[i] = l;
  }
}
__global__ void pack_pad_split_h_kernel(const float* __restrict__ W, __half* __restrict__ hi, __half* __restrict__ lo, int N,
                                        int Np, int Cc, int KK) {
  const int64_t n = (int64_t)N * Cc * KK;
  GRID_STRIDE(i, n) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc), row = (int)(r / Cc);
    __half h, l;
    split_f16(W[i], h, l);
    const int64_t j = ((int64_t)t * Np + row) * Cc + ch;
    hi[j] = h;
    lo[j] = l;
  }
}
// dst[p][n] = src[p][n] + bias[n] for n < Cs  (src rows are Cp wide)
__global__ void compact_bias_kernel(const float* __restrict__ src, const float* __restrict__ bias, float* __restrict__ dst,
                                    int64_t P, int Cs, int Cp) {
  const int64_t n = P * Cs;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % Cs);
    dst[i] = src[(i / Cs) * Cp + ch] + (bias ? bias[ch] : 0.f);
  }
}
// W [N][Cc][KK] -> TF32 hi/lo of the tap-major pack [t][Np][Cc] (rows >= N are never written: keep them zero)
__global__ void pack_pad_split_kernel(const float* __restrict__ W, float* __restrict__ hi, float* __restrict__ lo, int N,
                                      int Np, int Cc, int KK) {
  const int64_t n = (int64_t)N * Cc * KK;
  GRID_STRIDE(i, n) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc), row = (int)(r / Cc);
    float h, l;
    split_tf32(W[i], h, l);
    const int64_t j = ((int64_t)t * Np + row) * Cc + ch;
    hi[j] = h;
    lo[j] = l;
  }
}
// dW[n][c][t] += G[t][n][c] for n < N, G rows padded to Np
__global__ void unpack_wgrad_pad_kernel(const float* __restrict__ G, float* __restrict__ dW, int N, int Np, int Cc, int KK) {
  const int64_t n = (int64_t)N * Cc * KK;
  GRID_STRIDE(i, n) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc), row = (int)(r / Cc);
    dW[i] += G[((int64_t)t * Np + row) * Cc + ch];
  }
}
// roles swapped (big channel count on the M side): dW[n][c][t] += Gt[KK-1-t][c][n], Gt = [KK][Cc][Np]
__global__ void unpack_wgrad_swapped_kernel(const float* __restrict__ Gt, float* __restrict__ dW, int N, int Np, int Cc,
                                            int KK) {
  const int64_t n = (int64_t)N * Cc * KK;
  GRID_STRIDE(i, n) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc), row = (int)(r / Cc);
    dW[i] += Gt[((int64_t)(KK - 1 - t) * Cc + ch) * Np + row];
  }
}
}  // namespace

int k_pad_split(fg_ctx* c, const float* src, float* hi, float* lo, int64_t P, int Cs, int Cp) {
  pad_split_kernel<<<grid_for(P * Cp, 256), 256, 0, c->stream>>>(src, hi, lo, P, Cs, Cp);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_pad_split_h(fg_ctx* c, const float* src, float* hi, float* lo, int64_t P, int Cs, int Cp, float* amax_slot) {
  pad_split_h_kernel<<<grid_for(P * Cp, 256), 256, 0, c->stream>>>(src, reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo), P,
                                                                   Cs, Cp, amax_slot);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_pack_pad_split_h(fg_ctx* c, const float* W, float* hi, float* lo, int N, int Np, int Cc, int KK) {
  pack_pad_split_h_kernel<<<grid_for((int64_t)N * Cc * KK, 256), 256, 0, c->stream>>>(W, reinterpret_cast<__half*>(hi),
                                                                                      reinterpret_cast<__half*>(lo), N, Np, Cc, KK);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_compact_bias(fg_ctx* c, const float* src, const float* bias, float* dst, int64_t P, int Cs, int Cp) {
  compact_bias_kernel<<<grid_for(P * Cs, 256), 256, 0, c->stream>>>(src, bias, dst, P, Cs, Cp);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_pack_pad_split(fg_ctx* c, const float* W, float* hi, float* lo, int N, int Np, int Cc, int KK) {
  pack_pad_split_kernel<<<grid_for((int64_t)N * Cc * KK, 256), 256, 0, c->stream>>>(W, hi, lo, N, Np, Cc, KK);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_unpack_wgrad_pad(fg_ctx* c, const float* G, float* dW, int N, int Np, int Cc, int KK) {
  unpack_wgrad_pad_kernel<<<grid_for((int64_t)N * Cc * KK, 256), 256, 0, c->stream>>>(G, dW, N, Np, Cc, KK);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_unpack_wgrad_swapped(fg_ctx* c, const float* Gt, float* dW, int N, int Np, int Cc, int KK) {
  unpack_wgrad_swapped_kernel<<<grid_for((int64_t)N * Cc * KK, 256), 256, 0, c->stream>>>(Gt, dW, N, Np, Cc, KK);
  LAUNCH_CHECK(c);
  return FG_OK;
}

int k_join_to_nhwc(fg_ctx* c, const float* noise, const float* cond, float* out, int B, int C, int HW) {
  join_to_nhwc_kernel<<<grid_for((int64_t)B * HW * (C + 1), 256), 256, 0, c->stream>>>(noise, cond, out, B, C, HW);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_add(fg_ctx* c, const float* a, const float* b, float* out, int64_t n) {
  add_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(a, b, out, n);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_maxpool2_fwd(fg_ctx* c, const float* h, float* p, int B, int H, int W, int C) {
  maxpool2_fwd_nhwc_kernel<<<grid_for((int64_t)B * (H / 2) * (W / 2) * C, 256), 256, 0, c->stream>>>(h, p, B, H, W, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_maxpool2_bwd(fg_ctx* c, const float* dp, const float* h, float* dh, int B, int H, int W, int C) {
  maxpool2_bwd_nhwc_kernel<<<grid_for((int64_t)B * (H / 2) * (W / 2) * C, 256), 256, 0, c->stream>>>(dp, h, dh, B, H, W, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_dropout_nhwc(fg_ctx* c, const float* x, const float* masks, int64_t stride, int moff, int HW, int C, float scale,
                   float* y, int B) {
  dropout_nhwc_kernel<<<grid_for((int64_t)B * HW * C, 256), 256, 0, c->stream>>>(x, masks, stride, moff, HW, C, scale, y, B);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_bernoulli_keep(fg_ctx* c, float* out, int64_t n, uint64_t seed, float p_drop, const uint64_t* seed_dev) {
  bernoulli_keep_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(out, n, seed, p_drop, seed_dev);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_up2_fwd_nchw(fg_ctx* c, const float* x, float* y, int64_t BC, int H, int W) {
  up2_fwd_nchw_kernel<<<grid_for(BC * H * W * 4, 256), 256, 0, c->stream>>>(x, y, BC, H, W);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_up2_bwd_nchw(fg_ctx* c, const float* dy, float* dx, int64_t BC, int H, int W) {
  up2_bwd_nchw_kernel<<<grid_for(BC * H * W, 256), 256, 0, c->stream>>>(dy, dx, BC, H, W);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_avgpool2_fwd_nchw(fg_ctx* c, const float* x, float* y, int64_t BC, int H, int W) {
  avgpool2_fwd_nchw_kernel<<<grid_for(BC * (H / 2) * (W / 2), 256), 256, 0, c->stream>>>(x, y, BC, H, W);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_avgpool2_bwd_nchw(fg_ctx* c, const float* dy, float* dx, int64_t BC, int H, int W) {
  avgpool2_bwd_nchw_kernel<<<grid_for(BC * H * W, 256), 256, 0, c->stream>>>(dy, dx, BC, H, W);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_maxpool2_fwd_nchw(fg_ctx* c, const float* x, float* y, int64_t BC, int H, int W) {
  maxpool2_fwd_nchw_kernel<<<grid_for(BC * (H / 2) * (W / 2), 256), 256, 0, c->stream>>>(x, y, BC, H, W);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_maxpool2_bwd_nchw(fg_ctx* c, const float* x, const float* dy, float* dx, int64_t BC, int H, int W) {
  maxpool2_bwd_nchw_kernel<<<grid_for(BC * H * W, 256), 256, 0, c->stream>>>(x, dy, dx, BC, H, W);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_dropout_nchw(fg_ctx* c, const float* x, const float* mask, float scale, int inner, float* y, int64_t n) {
  if (mask)
    dropout_nchw_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(x, mask, scale, inner, y, n);
  else
    scale_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(x, scale, y, n);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// out[i] = sum over s of parts[s * n + i], always in split order (deterministic split-K reduction)
__global__ void splitk_reduce_kernel(const float* __restrict__ parts, int splits, int64_t n, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s = parts[i];
    for (int k = 1; k < splits; ++k) s += parts[(int64_t)k * n + i];
    out[i] = s;
  }
}
int k_splitk_reduce(fg_ctx* c, const float* parts, int splits, int64_t n, float* out) {
  splitk_reduce_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(parts, splits, n, out);
  LAUNCH_CHECK(c);
  return FG_OK;
}
