// wgmma / TMA implicit-GEMM convolutions for sm_90a with error-compensated 3xTF32
// (hi*hi + hi*lo + lo*hi, fp32 accumulation in registers) so results stay within fp32 parity.
//
// Both kernels view a stride-1 "same" convolution as a sum over filter taps of shifted GEMMs and feed
// the tensor cores with plain TILED TMA boxes of the NHWC activation tensors (out-of-image rows /
// columns are zero-filled by TMA, which implements the zero padding for free):
//
//   tapconv (forward + dgrad):  D[pixel m][n]  = sum_taps A_tap[m][c] * W_tap[n][c]
//       A_tap = box(32 ch, bw, bh, bb) of 128 pixels at spatial offset (dy,dx)  -> K-major operand
//       W_tap = box(32 ch, BN rows) of the packed weights [tap][n][c]          -> K-major operand
//   wgrad:                      D[n][c]        = sum_pixels dY[p][n] * X[p+off][c]
//       dY, X boxes (32 ch, 32 pixels)                                          -> MN-major operands
//
// nn.SpatialUpSamplingNearest(2) -> conv5x5 is executed on the LOW-RES tensor: output phase (py,px)
// only sees low-res offsets {-1,0,1}^2 (SURVEY.md 7.3), either with the 25 original taps ("dense")
// or with the weights pre-summed to 9 taps per phase ("collapsed", 2.78x fewer MMAs).
//
// Pipeline per CTA (384 threads): warpgroups 0-1 = wgmma issue + epilogue (64 accumulator rows each),
// warpgroup 2 = TMA producer.  3 smem stages of {A_hi, A_lo, B_hi, B_lo}, 128B-swizzled, mbarrier full/empty
// rings (k_conv_tc_kernels.cuh).
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <queue>
#include <vector>

#include "fg_internal.h"
#include "k_conv_tc.h"
#include "k_f16split.cuh"
#include "k_wgmma.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}
// pure spin (mbarrier.test_wait never suspends the thread): for the single-thread producer / MMA-issue roles, where the
// wake-up latency of a suspended try_wait sits on the critical path of the stage ring
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// wgmma shared-memory matrix descriptor:
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset (0: every tile is 1024-aligned)
//   | [62,64) layout (1 = SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (1ull << 62);
}

constexpr int kStages = 3;
constexpr int64_t kGridCap = 132 * 16;  // grid-stride elementwise kernels: 16 CTAs per SM of an H100
constexpr uint32_t kABytes = 128 * 128;  // 128 rows x 32 fp32

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

#include "k_conv_tc_kernels.cuh"

// ------------------------------------------------------------------------------------------------
// elementwise helpers of the tensor-core path
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  // hi: mantissa rounded to 10 bits (what a tf32 MMA consumes exactly), lo: exact fp32 remainder
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  lo = x - hi;
}
template <bool ALIGNED>
__global__ void split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int64_t n4) {
  const float4* x4 = reinterpret_cast<const float4*>(x);
  float4* h4 = reinterpret_cast<float4*>(hi);
  float4* l4 = reinterpret_cast<float4*>(lo);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = ALIGNED ? x4[i] : make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
    float4 h, l;
    split_tf32(v.x, h.x, l.x);
    split_tf32(v.y, h.y, l.y);
    split_tf32(v.z, h.z, l.z);
    split_tf32(v.w, h.w, l.w);
    h4[i] = h;
    l4[i] = l;
  }
}

__global__ void amax_kernel(const float* __restrict__ x, int64_t n4, unsigned* __restrict__ slot) {
  const float4* x4 = reinterpret_cast<const float4*>(x);
  float m = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = x4[i];
    m = fmaxf(fmaxf(m, fmaxf(finite_abs(v.x), finite_abs(v.y))), fmaxf(finite_abs(v.z), finite_abs(v.w)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  // non-negative floats order like their bits; a plain load first so that only warps raising the maximum issue the atomic
  if ((threadIdx.x & 31) == 0 && m > 0.f && __float_as_uint(m) > *reinterpret_cast<volatile unsigned*>(slot))
    atomicMax(slot, __float_as_uint(m));
}
template <bool ALIGNED>
__global__ void split_h_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, int64_t n4,
                               const float* __restrict__ amax_slot, float* __restrict__ inv_out) {
  float s = 1.f;
  if (amax_slot) {
    s = scale_for_amax(amax_slot[0]);
    if (blockIdx.x == 0 && threadIdx.x == 0) *inv_out = 1.f / s;  // exact: s is a power of two
  }
  const float4* x4 = reinterpret_cast<const float4*>(x);
  uint2* h2 = reinterpret_cast<uint2*>(hi);
  uint2* l2 = reinterpret_cast<uint2*>(lo);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = ALIGNED ? x4[i] : make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
    __half h[4], l[4];
    split_f16(v.x * s, h[0], l[0]);
    split_f16(v.y * s, h[1], l[1]);
    split_f16(v.z * s, h[2], l[2]);
    split_f16(v.w * s, h[3], l[3]);
    h2[i] = *reinterpret_cast<uint2*>(h);
    l2[i] = *reinterpret_cast<uint2*>(l);
  }
}

// up2 -> 5x5 collapses to 3x3 per output phase: 5x5 rows/cols {0,1}{2,3}{4} (even phase) or {0}{1,2}{3,4} (odd)
__device__ __forceinline__ void group_range(int parity, int t, int& lo, int& hi) {
  if (parity == 0) {
    lo = t == 0 ? 0 : (t == 1 ? 2 : 4);
    hi = t == 0 ? 1 : (t == 1 ? 3 : 4);
  } else {
    lo = t == 0 ? 0 : (t == 1 ? 1 : 3);
    hi = t == 0 ? 0 : (t == 1 ? 2 : 4);
  }
}
// W[N][Cc][5][5] -> fwd[ph][ty][tx][n][c] (hi/lo) and dgrad[ph][ty][tx][c][n] (hi/lo)
template <class T> struct SplitTo;
template <> struct SplitTo<float> {
  static __device__ __forceinline__ void run(float x, float& hi, float& lo) { split_tf32(x, hi, lo); }
};
template <> struct SplitTo<__half> {
  static __device__ __forceinline__ void run(float x, __half& hi, __half& lo) { split_f16(x, hi, lo); }
};
template <class T>
__global__ void pack_collapsed_kernel(const float* __restrict__ W, T* __restrict__ f_hi, T* __restrict__ f_lo,
                                      T* __restrict__ d_hi, T* __restrict__ d_lo, int N, int Cc) {
  const int64_t total = (int64_t)36 * N * Cc;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % Cc);
    int64_t r = i / Cc;
    const int n = (int)(r % N);
    const int tp = (int)(r / N);  // ph*9 + ty*3 + tx
    const int ph = tp / 9, ty = (tp % 9) / 3, tx = tp % 3;
    int h0, h1, w0, w1;
    group_range(ph >> 1, ty, h0, h1);
    group_range(ph & 1, tx, w0, w1);
    const float* w = W + ((int64_t)n * Cc + ch) * 25;
    float s = 0.f;
    for (int kh = h0; kh <= h1; ++kh)
      for (int kw = w0; kw <= w1; ++kw) s += w[kh * 5 + kw];
    T hi, lo;
    SplitTo<T>::run(s, hi, lo);
    f_hi[i] = hi;
    f_lo[i] = lo;
    const int64_t j = ((int64_t)tp * Cc + ch) * N + n;
    d_hi[j] = hi;
    d_lo[j] = lo;
  }
}
// generic: W[N][Cc][KK] -> fwd[t][n][c] hi/lo, dgrad[KK-1-t][c][n] hi/lo
template <class T>
__global__ void pack_split_kernel(const float* __restrict__ W, T* __restrict__ f_hi, T* __restrict__ f_lo,
                                  T* __restrict__ d_hi, T* __restrict__ d_lo, int N, int Cc, int KK) {
  const int64_t total = (int64_t)N * Cc * KK;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc);
    const int n = (int)(r / Cc);
    T hi, lo;
    SplitTo<T>::run(W[i], hi, lo);
    const int64_t jf = ((int64_t)t * N + n) * Cc + ch;
    f_hi[jf] = hi;
    f_lo[jf] = lo;
    if (d_hi) {
      const int64_t jd = ((int64_t)(KK - 1 - t) * Cc + ch) * N + n;
      d_hi[jd] = hi;
      d_lo[jd] = lo;
    }
  }
}
// The two packs want opposite thread orders (forward: channel fastest, dgrad: output row fastest); written from one
// thread order, one of them degenerates into 2-byte scattered stores (31 us per 5x5 layer).  These variants stage a
// 16 x 16 (n, c) tile of the weights in shared memory (coalesced 1.6 KB rows) and write each pack from its own order:
// every global access is a full 32-byte sector.  Same sums in the same order as the element-wise kernels above.
template <class T>
__global__ void __launch_bounds__(256) pack_collapsed_tile_kernel(const float* __restrict__ W, T* __restrict__ f_hi,
                                                                  T* __restrict__ f_lo, T* __restrict__ d_hi,
                                                                  T* __restrict__ d_lo, int N, int Cc) {
  __shared__ float w[16][16 * 25 + 1];
  const int n0 = blockIdx.y * 16, c0 = blockIdx.x * 16;
  for (int i = threadIdx.x; i < 16 * 400; i += 256) {
    const int nl = i / 400, r = i - nl * 400;
    w[nl][r] = W[((int64_t)(n0 + nl) * Cc + c0) * 25 + r];
  }
  __syncthreads();
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
    // pass 0: forward pack, channel fastest; pass 1: dgrad pack, output row fastest
    const int nl = pass == 0 ? (threadIdx.x >> 4) : (threadIdx.x & 15);
    const int cl = pass == 0 ? (threadIdx.x & 15) : (threadIdx.x >> 4);
    const float* p = &w[nl][cl * 25];
    for (int tp = blockIdx.z * 9; tp < blockIdx.z * 9 + 9; ++tp) {  // grid.z = the 4 output phases
      const int ph = tp / 9, ty = (tp % 9) / 3, tx = tp % 3;
      int h0, h1, w0, w1;
      group_range(ph >> 1, ty, h0, h1);
      group_range(ph & 1, tx, w0, w1);
      float s = 0.f;
      for (int kh = h0; kh <= h1; ++kh)
        for (int kw = w0; kw <= w1; ++kw) s += p[kh * 5 + kw];
      T hi, lo;
      SplitTo<T>::run(s, hi, lo);
      if (pass == 0) {
        const int64_t i = ((int64_t)tp * N + n0 + nl) * Cc + c0 + cl;
        f_hi[i] = hi;
        f_lo[i] = lo;
      } else {
        const int64_t j = ((int64_t)tp * Cc + c0 + cl) * N + n0 + nl;
        d_hi[j] = hi;
        d_lo[j] = lo;
      }
    }
  }
}
template <class T, int KK>
__global__ void __launch_bounds__(256) pack_split_tile_kernel(const float* __restrict__ W, T* __restrict__ f_hi,
                                                              T* __restrict__ f_lo, T* __restrict__ d_hi,
                                                              T* __restrict__ d_lo, int N, int Cc) {
  __shared__ float w[16][16 * KK + 1];
  const int n0 = blockIdx.y * 16, c0 = blockIdx.x * 16;
  for (int i = threadIdx.x; i < 16 * 16 * KK; i += 256) {
    const int nl = i / (16 * KK), r = i - nl * 16 * KK;
    w[nl][r] = W[((int64_t)(n0 + nl) * Cc + c0) * KK + r];
  }
  __syncthreads();
#pragma unroll 1
  for (int pass = 0; pass < (d_hi ? 2 : 1); ++pass) {
    const int nl = pass == 0 ? (threadIdx.x >> 4) : (threadIdx.x & 15);
    const int cl = pass == 0 ? (threadIdx.x & 15) : (threadIdx.x >> 4);
    for (int t = blockIdx.z; t < KK; t += gridDim.z) {  // grid.z splits the taps
      T hi, lo;
      SplitTo<T>::run(w[nl][cl * KK + t], hi, lo);
      if (pass == 0) {
        const int64_t jf = ((int64_t)t * N + n0 + nl) * Cc + c0 + cl;
        f_hi[jf] = hi;
        f_lo[jf] = lo;
      } else {
        const int64_t jd = ((int64_t)(KK - 1 - t) * Cc + c0 + cl) * N + n0 + nl;
        d_hi[jd] = hi;
        d_lo[jd] = lo;
      }
    }
  }
}
// collapsed wgrad G[ph][ty][tx][n][c] -> dW[n][c][5][5] += sum over the 4 phases
__global__ void combine_collapsed_wgrad_kernel(const float* __restrict__ G, float* __restrict__ dW, int N, int Cc) {
  const int64_t total = (int64_t)N * Cc * 25;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % 25);
    const int64_t r = i / 25;
    const int ch = (int)(r % Cc);
    const int n = (int)(r / Cc);
    const int kh = t / 5, kw = t % 5;
    float s = 0.f;
#pragma unroll
    for (int ph = 0; ph < 4; ++ph) {
      const int py = ph >> 1, px = ph & 1;
      const int ty = py == 0 ? (kh < 2 ? 0 : (kh < 4 ? 1 : 2)) : (kh < 1 ? 0 : (kh < 3 ? 1 : 2));
      const int tx = px == 0 ? (kw < 2 ? 0 : (kw < 4 ? 1 : 2)) : (kw < 1 ? 0 : (kw < 3 ? 1 : 2));
      s += G[(((int64_t)(ph * 9 + ty * 3 + tx)) * N + n) * Cc + ch];
    }
    dW[i] += s;
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int get_encode() {
  if (g_encode) return FG_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  FG_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) {
    fg_set_error("cuTensorMapEncodeTiled is not available in this driver");
    return FG_ERR_UNSUPPORTED;
  }
  g_encode = (EncodeTiledFn)fn;
  return FG_OK;
}

// 4-D map over an NHWC fp32 tensor view: dims (C, W, H, B) with explicit byte strides
// pair = true: `base` is a BF16 pair tensor (2*C bf16 per pixel, same byte strides); the box takes 2*bc elements
int make_map4(CUtensorMap* m, const float* base, int C, int W, int H, int B, int64_t sW, int64_t sH, int64_t sB, int bc,
              int bw, int bh, int bb, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B, bool pair = false, bool f16 = false) {
  const int mul = pair ? 2 : 1;
  cuuint64_t dims[4] = {(cuuint64_t)C * mul, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)sW, (cuuint64_t)sH, (cuuint64_t)sB};
  cuuint32_t box[4] = {(cuuint32_t)bc * mul, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bb};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = g_encode(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : (pair ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32), 4, (void*)base, dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fg_set_error("cuTensorMapEncodeTiled(4d) failed: %d (C=%d W=%d H=%d B=%d box %d,%d,%d,%d)", (int)r, C, W, H, B, bc, bw,
                 bh, bb);
    return FG_ERR_CUDA;
  }
  return FG_OK;
}
// 5-D map for the MN-major wgrad operands: dims (32 ch-in-group, W, H, B, C/32 groups); the box takes `ngroups`
// channel groups of one 32-pixel box so the tile lands as [group][pixel][32 ch], unswizzled (the kernel transposes it)
// f16: groups of 64 fp16 channels (128 bytes), SWIZZLE_128B (the canonical MN-major wgmma layout)
int make_map5(CUtensorMap* m, const float* base, int C, int W, int H, int B, int64_t sW, int64_t sH, int64_t sB, int bw,
              int bh, int bb, int ngroups, bool f16 = false) {
  const int gch = f16 ? 64 : 32;
  cuuint64_t dims[5] = {(cuuint64_t)gch, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B, (cuuint64_t)(C / gch)};
  cuuint64_t strides[4] = {(cuuint64_t)sW, (cuuint64_t)sH, (cuuint64_t)sB, 128};
  cuuint32_t box[5] = {(cuuint32_t)gch, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bb, (cuuint32_t)ngroups};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)base, dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, f16 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fg_set_error("cuTensorMapEncodeTiled(5d) failed: %d (C=%d W=%d H=%d B=%d box %d,%d,%d x%d)", (int)r, C, W, H, B, bw, bh,
                 bb, ngroups);
    return FG_ERR_CUDA;
  }
  return FG_OK;
}
int make_map2(CUtensorMap* m, const float* base, int cols, int64_t rows, int bc, int br, bool pair = false, bool f16 = false) {
  const int mul = pair ? 2 : 1;
  cuuint64_t dims[2] = {(cuuint64_t)cols * mul, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * (f16 ? 2 : 4)};
  cuuint32_t box[2] = {(cuuint32_t)bc * mul, (cuuint32_t)br};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encode(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : (pair ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32), 2, (void*)base, dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fg_set_error("cuTensorMapEncodeTiled(2d) failed: %d (cols=%d rows=%lld box %d,%d)", (int)r, cols, (long long)rows, bc, br);
    return FG_ERR_CUDA;
  }
  return FG_OK;
}

// pixel box of `npix` pixels for a WxH image: returns false if no exact tiling exists
bool pick_box(int H, int W, int npix, int* bw, int* bh, int* bb) {
  if (W <= 0 || H <= 0) return false;
  if (W >= npix) {
    if (W % npix) return false;
    *bw = npix; *bh = 1; *bb = 1;
    return true;
  }
  if (npix % W) return false;
  const int rows = npix / W;
  if (rows <= H) {
    if (H % rows) return false;
    *bw = W; *bh = rows; *bb = 1;
    return true;
  }
  if (rows % H) return false;
  *bw = W; *bh = H; *bb = rows / H;
  return true;
}

template <int BN>
constexpr size_t fwd_smem() { return (size_t)kStages * (2 * kABytes + 2 * BN * 128) + 256 + 5 * 8 * BN * 4 + 1024; }
// F16: 3 TMA stages; TF32: 2 TMA stages + the K-major copy of one (same bytes per stage)
template <int BN>
constexpr size_t wg_smem() { return (size_t)3 * (2 * 4 * 4096 + 2 * (BN / 32) * 4096) + 128 + 1024; }
// 3 stages, then {full, empty}[3] and the id-slot ring (full, empty, ids) of bwd_pair_tc_kernel
template <int BN>
constexpr size_t bwd_smem() { return (size_t)kStages * fwd_stage_bytes<BN>() + 256 + 1024; }


// ------------------------------------------------------------------------------------------------
// tensor-pipe probe: the issue rate of back-to-back wgmmas (m64 x N x 8 tf32 or m64 x N x 16 f16, two warpgroups
// per SM) with both operands resident in shared memory -- no TMA, no epilogue.  bench.py runs it at bench clocks;
// the number is the measured MMA peak the 3-term convolutions are normalised by.
// ------------------------------------------------------------------------------------------------
template <int N, bool F16 = false>
__global__ void __launch_bounds__(256, 1) tf32_peak_kernel(int iters, float* sink) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr uint32_t kFoot = (128 + N) * 128;  // A: 128 rows, B: N rows of 128 bytes
  for (uint32_t i = threadIdx.x; i < kFoot / 4; i += blockDim.x) reinterpret_cast<float*>(smem)[i] = 1.f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy smem writes -> visible to the MMA
  __syncthreads();
  const uint32_t sa = smem_u32(smem);
  const uint64_t a = make_desc(sa + (threadIdx.x >> 7) * 64 * 128, 16, 1024), b = make_desc(sa + 128 * 128, 16, 1024);
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  for (int i = 0; i < iters; ++i) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_op<N, F16, false>(acc, a + (uint64_t)(k * 2), b + (uint64_t)(k * 2), 1);
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s += acc[i];
  if (s == 1234.5f) *sink = s;  // never taken; keeps the accumulators live
}

}  // namespace

// -> TFLOP/s of the MMAs (2*M*N*K per instruction) over all SMs, best of `reps` event-timed launches.
// FG_TF32_PROBE_N=128 probes the N=128 instruction shape; FG_TF32_PROBE_F16=1 the same loop with f16 operands
// (K = 16 per instruction) -- the rate the 3xFP16 kernels run at
int tc_tf32_peak(fg_ctx* c, int iters, int reps, double* tflops) {
  const char* env = getenv("FG_TF32_PROBE_N");
  const int N = env && atoi(env) == 128 ? 128 : 256;
  const bool f16 = getenv("FG_TF32_PROBE_F16") && atoi(getenv("FG_TF32_PROBE_F16"));
  const int kSmem = (128 + N) * 128 + 1024;
  auto kern = f16 ? (N == 128 ? tf32_peak_kernel<128, true> : tf32_peak_kernel<256, true>)
                  : (N == 128 ? tf32_peak_kernel<128> : tf32_peak_kernel<256>);
  FG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  cudaEvent_t e0, e1;
  FG_CUDA(cudaEventCreate(&e0));
  FG_CUDA(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {  // first launch = warm-up
    FG_CUDA(cudaEventRecord(e0, c->stream));
    kern<<<c->sm_count, 256, kSmem, c->stream>>>(iters, c->io_dev);
    LAUNCH_CHECK(c);
    FG_CUDA(cudaEventRecord(e1, c->stream));
    FG_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    FG_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    if (r > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  const double flops = (double)c->sm_count * iters * 4.0 * 2.0 * 128 * N * (f16 ? 16 : 8);
  *tflops = flops / (best * 1e-3) / 1e12;
  return FG_OK;
}

// plain (un-swizzled) 4-D TMA map over a dense NHWC fp32 tensor with the given box -- for the HBM-shaped kernels
// that only use TMA as a deep-prefetch copy engine (k_conv_edge.cu)
int tc_encode_nhwc_box(CUtensorMap* m, const float* base, int C, int W, int H, int B, int bc, int bw, int bh, int bb) {
  FG_TRY(get_encode());
  const int64_t sW = (int64_t)C * 4, sH = sW * W, sB = sH * H;
  return make_map4(m, base, C, W, H, B, sW, sH, sB, bc, bw, bh, bb, CU_TENSOR_MAP_SWIZZLE_NONE);
}

int tc_init(fg_ctx* c) {
  (void)c;
  FG_TRY(get_encode());
  FG_CUDA(cudaFuncSetAttribute(tapconv_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<64>()));
  FG_CUDA(cudaFuncSetAttribute(tapconv_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<128>()));
  FG_CUDA(cudaFuncSetAttribute(tapconv_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<64>()));
  FG_CUDA(cudaFuncSetAttribute(tapconv_tc_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<128>()));
  FG_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<64>()));
  FG_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<128>()));
  FG_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<64>()));
  FG_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem<128>()));
  FG_CUDA(cudaFuncSetAttribute(bwd_pair_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<128>()));
  return FG_OK;
}
void tc_destroy(fg_ctx* c) { (void)c; }

int tc_split(fg_ctx* c, const float* x, float* hi, float* lo, int64_t n) {
  if (n % 4) {
    fg_set_error("tc_split: element count must be a multiple of 4");
    return FG_ERR_INVALID;
  }
  int64_t g = (n / 4 + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  if (reinterpret_cast<uintptr_t>(x) % 16 == 0) split_kernel<true><<<(int)g, 256, 0, c->stream>>>(x, hi, lo, n / 4);
  else split_kernel<false><<<(int)g, 256, 0, c->stream>>>(x, hi, lo, n / 4);  // e.g. a weight block inside the flat parameter vector
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_amax(fg_ctx* c, const float* x, int64_t n, float* amax_slot) {
  if (n % 4 || reinterpret_cast<uintptr_t>(x) % 16) {
    fg_set_error("tc_amax: needs a 16-byte aligned tensor with a multiple of 4 elements");
    return FG_ERR_INVALID;
  }
  FG_CUDA(cudaMemsetAsync(amax_slot, 0, 2 * sizeof(float), c->stream));
  int64_t g = (n / 4 + 255) / 256;
  if (g > kGridCap / 2) g = kGridCap / 2;
  amax_kernel<<<(int)g, 256, 0, c->stream>>>(x, n / 4, reinterpret_cast<unsigned*>(amax_slot));
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_split_h(fg_ctx* c, const float* x, float* hh, float* hl, int64_t n, float* amax_slot, float* inv_out) {
  if (amax_slot && !inv_out) inv_out = amax_slot + 1;
  if (n % 4) {
    fg_set_error("tc_split_h: element count must be a multiple of 4");
    return FG_ERR_INVALID;
  }
  int64_t g = (n / 4 + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  __half *h = reinterpret_cast<__half*>(hh), *l = reinterpret_cast<__half*>(hl);
  if (reinterpret_cast<uintptr_t>(x) % 16 == 0) split_h_kernel<true><<<(int)g, 256, 0, c->stream>>>(x, h, l, n / 4, amax_slot, inv_out);
  else split_h_kernel<false><<<(int)g, 256, 0, c->stream>>>(x, h, l, n / 4, amax_slot, inv_out);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_pack_split_h(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc, int KK) {
  if (KK == 9 && N % 16 == 0 && Cc % 16 == 0) {
    pack_split_tile_kernel<__half, 9><<<dim3(Cc / 16, N / 16, 3), 256, 0, c->stream>>>(W, (__half*)f_hi, (__half*)f_lo, (__half*)d_hi,
                                                                                    (__half*)d_lo, N, Cc);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  int64_t g = ((int64_t)N * Cc * KK + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  pack_split_kernel<__half><<<(int)g, 256, 0, c->stream>>>(W, (__half*)f_hi, (__half*)f_lo, (__half*)d_hi, (__half*)d_lo, N, Cc, KK);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_pack_collapsed_h(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc) {
  if (N % 16 == 0 && Cc % 16 == 0) {
    pack_collapsed_tile_kernel<__half><<<dim3(Cc / 16, N / 16, 4), 256, 0, c->stream>>>(W, (__half*)f_hi, (__half*)f_lo, (__half*)d_hi,
                                                                                     (__half*)d_lo, N, Cc);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  int64_t g = ((int64_t)36 * N * Cc + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  pack_collapsed_kernel<__half><<<(int)g, 256, 0, c->stream>>>(W, (__half*)f_hi, (__half*)f_lo, (__half*)d_hi, (__half*)d_lo, N, Cc);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_pack_split(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc, int KK) {
  if (KK == 9 && N % 16 == 0 && Cc % 16 == 0) {
    pack_split_tile_kernel<float, 9><<<dim3(Cc / 16, N / 16, 3), 256, 0, c->stream>>>(W, f_hi, f_lo, d_hi, d_lo, N, Cc);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  int64_t g = ((int64_t)N * Cc * KK + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  pack_split_kernel<float><<<(int)g, 256, 0, c->stream>>>(W, f_hi, f_lo, d_hi, d_lo, N, Cc, KK);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_pack_collapsed(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc) {
  if (N % 16 == 0 && Cc % 16 == 0) {
    pack_collapsed_tile_kernel<float><<<dim3(Cc / 16, N / 16, 4), 256, 0, c->stream>>>(W, f_hi, f_lo, d_hi, d_lo, N, Cc);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  int64_t g = ((int64_t)36 * N * Cc + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  pack_collapsed_kernel<float><<<(int)g, 256, 0, c->stream>>>(W, f_hi, f_lo, d_hi, d_lo, N, Cc);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int tc_combine_collapsed_wgrad(fg_ctx* c, const float* G, float* dW, int N, int Cc) {
  int64_t g = ((int64_t)N * Cc * 25 + 255) / 256;
  if (g > kGridCap) g = kGridCap;
  combine_collapsed_wgrad_kernel<<<(int)g, 256, 0, c->stream>>>(G, dW, N, Cc);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// K-blocks (32 channels of one tap) accumulated in the wgmma accumulators before the consumers promote them into fp32
// registers.  The drift of a tensor-core accumulation grows with the length of the run (DESIGN.md section 5), every
// promotion drains the consumer's wgmma pipeline, so the chunk is a trade: convolution forward / dgrad 12, wgrad and
// the Linear layers (K = pixels resp. up to 16384 features) 8 resp. 4.  FG_TC_CHUNK / FG_TC_CHUNK_FWD override for
// experiments.
static int tc_chunk(bool forward_type = false) {
  static int v[2] = {-1, -1};
  if (v[0] < 0) {
    const char* e = getenv("FG_TC_CHUNK");
    v[0] = e ? atoi(e) : 0;
    const char* f = getenv("FG_TC_CHUNK_FWD");
    v[1] = f ? atoi(f) : v[0];
  }
  const int d = forward_type ? 12 : 4;
  const int x = v[forward_type ? 1 : 0];
  return x >= 1 ? x : d;
}

static int launch_tapconv(fg_ctx* c, const TcFwdParams& p, int BN, int f16 = 0) {
  dim3 grid(std::min(p.ntiles, std::max(1, c->sm_count - c->reserve_sms)));
  note_conv(c, FG_KERNEL_TAPCONV, 128, BN, f16 ? 2 : 1, 1);
  if (f16) {
    if (BN == 128) tapconv_tc_kernel<128, true><<<grid, kTcThreads, fwd_smem<128>(), c->stream>>>(p);
    else tapconv_tc_kernel<64, true><<<grid, kTcThreads, fwd_smem<64>(), c->stream>>>(p);
  } else if (BN == 128) tapconv_tc_kernel<128><<<grid, kTcThreads, fwd_smem<128>(), c->stream>>>(p);
  else tapconv_tc_kernel<64><<<grid, kTcThreads, fwd_smem<64>(), c->stream>>>(p);
  LAUNCH_CHECK(c);
  return FG_OK;
}

bool tc_conv_eligible(const ConvGeom& g) {
  int bw, bh, bb;
  const int Hl = g.H / g.ups, Wl = g.W / g.ups;
  if (g.Cin % 32 || g.Cout % 64) return false;
  if (g.ups == 2 && g.k != 5) return false;
  if (g.k > 9 || !(g.k & 1)) return false;
  return pick_box(Hl, Wl, 128, &bw, &bh, &bb) && pick_box(Hl, Wl, 32, &bw, &bh, &bb);
}

// Forward-type launch.  x_hi/x_lo: [B][H/ups][W/ups][Cin]; w_hi/w_lo: packed [tapw][Cout][Cin];
// mode: 0 plain k x k conv (taps k*k, weights [t][n][c]);
//       1 up2+5x5 dense (25 taps per output phase, weights [25][n][c]);
//       2 up2+5x5 collapsed (9 taps per phase, weights [36][n][c])
int tc_stat_parts(const ConvGeom& g, int mode) {
  int bw, bh, bb;
  const int Hl = g.H / g.ups, Wl = g.W / g.ups;
  if (!pick_box(Hl, Wl, 128, &bw, &bh, &bb)) return 0;
  const int per_phase = bb == 1 ? g.B * (Wl / bw) * (Hl / bh) : (g.B + bb - 1) / bb;
  return per_phase * (mode == 0 ? 1 : 4);
}

int tc_conv_fwd(fg_ctx* c, const float* x_hi, const float* x_lo, const float* w_hi, const float* w_lo,
                const float* bias, float* out, ConvGeom g, int mode, float* stats, int* n_parts, int f16, const float* oscale,
                const float* oscale2) {
  TcFwdParams p;
  memset(&p, 0, sizeof(p));
  const int Hl = g.H / g.ups, Wl = g.W / g.ups;
  if (!pick_box(Hl, Wl, 128, &p.bw, &p.bh, &p.bb)) {
    fg_set_error("tc_conv_fwd: no 128-pixel box for %dx%d", Hl, Wl);
    return FG_ERR_UNSUPPORTED;
  }
  const int es = f16 ? 2 : 4, ke = f16 ? 64 : 32;  // element bytes, K elements of one 128-byte block
  if (g.Cin % ke) {
    fg_set_error("tc_conv_fwd: %d input channels are not a multiple of %d", g.Cin, ke);
    return FG_ERR_UNSUPPORTED;
  }
  const bool h = f16 != 0;
  const int64_t sW = (int64_t)g.Cin * es, sH = sW * Wl, sB = sH * Hl;
  FG_TRY(make_map4(&p.a_hi[0], x_hi, g.Cin, Wl, Hl, g.B, sW, sH, sB, ke, p.bw, p.bh, p.bb, CU_TENSOR_MAP_SWIZZLE_128B, false, h));
  FG_TRY(make_map4(&p.a_lo[0], x_lo, g.Cin, Wl, Hl, g.B, sW, sH, sB, ke, p.bw, p.bh, p.bb, CU_TENSOR_MAP_SWIZZLE_128B, false, h));
  // N tile: 128 unless halving it keeps the same number of waves on the SMs (few-tile layers such as
  // D.C4's dgrad or the Linear layers): a BN=64 tile costs ~0.6 of a BN=128 tile
  int BN = g.Cout % 128 == 0 ? 128 : 64;
  if (BN == 128) {
    const int mt = (mode == 0 ? 1 : 4) * (p.bb == 1 ? g.B * (Wl / p.bw) * (Hl / p.bh) : (g.B + p.bb - 1) / p.bb);
    const int t128 = mt * (g.Cout / 128), t64 = mt * (g.Cout / 64);
    const int w128 = (t128 + c->sm_count - 1) / c->sm_count, w64 = (t64 + c->sm_count - 1) / c->sm_count;
    if (w64 * 6 < w128 * 10) BN = 64;
  }
  int ntapw;
  if (mode == 0) {
    const int pad = (g.k - 1) / 2;
    p.nphase = 1;
    p.ntaps = g.k * g.k;
    ntapw = p.ntaps;
    for (int t = 0; t < p.ntaps; ++t) {
      p.dy[t] = (int8_t)(t / g.k - pad);
      p.dx[t] = (int8_t)(t % g.k - pad);
      p.widx[t] = (int16_t)t;
    }
  } else if (mode == 1) {
    p.nphase = 4;
    p.ntaps = 25;
    ntapw = 25;
    for (int ph = 0; ph < 4; ++ph)
      for (int t = 0; t < 25; ++t) {
        const int kh = t / 5, kw = t % 5, py = ph >> 1, px = ph & 1;
        // floor((py + kh - 2) / 2) without relying on negative division
        p.dy[ph * 25 + t] = (int8_t)(((py + kh - 2) + 4) / 2 - 2);
        p.dx[ph * 25 + t] = (int8_t)(((px + kw - 2) + 4) / 2 - 2);
        p.widx[ph * 25 + t] = (int16_t)t;
      }
  } else {
    p.nphase = 4;
    p.ntaps = 9;
    ntapw = 36;
    for (int ph = 0; ph < 4; ++ph)
      for (int t = 0; t < 9; ++t) {
        p.dy[ph * 9 + t] = (int8_t)(t / 3 - 1);
        p.dx[ph * 9 + t] = (int8_t)(t % 3 - 1);
        p.widx[ph * 9 + t] = (int16_t)(ph * 9 + t);
      }
  }
  FG_TRY(make_map2(&p.b_hi, w_hi, g.Cin, (int64_t)ntapw * g.Cout, ke, BN, false, h));
  FG_TRY(make_map2(&p.b_lo, w_lo, g.Cin, (int64_t)ntapw * g.Cout, ke, BN, false, h));
  p.kpt = g.Cin / ke;
  p.oscale = oscale ? oscale : oscale2;
  p.oscale2 = oscale ? oscale2 : nullptr;
  p.Cout = g.Cout;
  p.B = g.B; p.H = Hl; p.W = Wl;
  p.tiles_x = Wl / p.bw;
  p.tiles_y = Hl / p.bh;
  p.tiles_per_phase = p.bb == 1 ? g.B * p.tiles_x * p.tiles_y : (g.B + p.bb - 1) / p.bb;
  p.out = out;
  p.bias = bias;
  p.stats = stats;
  if (n_parts) *n_parts = p.tiles_per_phase * p.nphase;
  p.out_H = g.H; p.out_W = g.W;
  p.out_scale = g.ups;
  p.ntiles = p.tiles_per_phase * p.nphase * (g.Cout / BN);
  p.chunk = tc_chunk(g.H * g.W > 1);  // Linear layers (1x1 images, K up to 16384) keep the short chunk
  // fp16: a 128-byte K block holds twice the K elements, so the same chunk is a 2x longer accumulation run (K = 768 for
  // the convolutions); measured <= 1.3e-6 of fp64 on every isolated launch (the TF32 path's level) and 2 % faster than 6
  if (f16 && g.H * g.W == 1) p.chunk = std::max(1, p.chunk / 2);
  return launch_tapconv(c, p, BN, f16);
}


// dgrad of an up2+5x5 conv straight to the LOW-RES input gradient (the 2x2 sum of the upsample backward is
// implicit: all 4 output phases accumulate into the same accumulator).  dy_hi/lo: [B][H][W][Cout] full-res;
// wd_hi/lo: collapsed dgrad pack [36][Cin][Cout]; out: [B][H/2][W/2][Cin].
static int dgrad_ups_params(const float* dy_hi, const float* dy_lo, const float* wd_hi, const float* wd_lo, float* out,
                            ConvGeom g, int f16, const float* oscale, TcFwdParams& p, int* BN_out) {
  memset(&p, 0, sizeof(p));
  const int Hl = g.H / 2, Wl = g.W / 2;
  if (!pick_box(Hl, Wl, 128, &p.bw, &p.bh, &p.bb)) return FG_ERR_UNSUPPORTED;
  const int Cy = g.Cout;  // contraction runs over the forward conv's output channels
  const int es = f16 ? 2 : 4, ke = f16 ? 64 : 32;
  const bool h = f16 != 0;
  if (Cy % ke) return FG_ERR_UNSUPPORTED;
  for (int ph = 0; ph < 4; ++ph) {
    const int py = ph >> 1, px = ph & 1;
    const int64_t off_bytes = ((int64_t)py * g.W + px) * Cy * es;
    const float* b_hi = reinterpret_cast<const float*>(reinterpret_cast<const char*>(dy_hi) + off_bytes);
    const float* b_lo = reinterpret_cast<const float*>(reinterpret_cast<const char*>(dy_lo) + off_bytes);
    const int64_t sW = (int64_t)2 * Cy * es, sH = (int64_t)2 * g.W * Cy * es, sB = (int64_t)g.H * g.W * Cy * es;
    FG_TRY(make_map4(&p.a_hi[ph], b_hi, Cy, Wl, Hl, g.B, sW, sH, sB, ke, p.bw, p.bh, p.bb, CU_TENSOR_MAP_SWIZZLE_128B, false, h));
    FG_TRY(make_map4(&p.a_lo[ph], b_lo, Cy, Wl, Hl, g.B, sW, sH, sB, ke, p.bw, p.bh, p.bb, CU_TENSOR_MAP_SWIZZLE_128B, false, h));
  }
  const int BN = g.Cin % 128 == 0 ? 128 : 64;
  p.nphase = 1;
  p.ntaps = 36;
  for (int ph = 0; ph < 4; ++ph)
    for (int t = 0; t < 9; ++t) {
      // forward: out_ph[y,x] reads Xlow[y+ty-1, x+tx-1]  =>  dXlow[y,x] reads dY_ph[y-(ty-1), x-(tx-1)]
      p.dy[ph * 9 + t] = (int8_t)(1 - t / 3);
      p.dx[ph * 9 + t] = (int8_t)(1 - t % 3);
      p.amap[ph * 9 + t] = (int8_t)ph;
      p.widx[ph * 9 + t] = (int16_t)(ph * 9 + t);
    }
  FG_TRY(make_map2(&p.b_hi, wd_hi, Cy, (int64_t)36 * g.Cin, ke, BN, false, h));
  FG_TRY(make_map2(&p.b_lo, wd_lo, Cy, (int64_t)36 * g.Cin, ke, BN, false, h));
  p.kpt = Cy / ke;
  p.oscale = oscale;
  p.Cout = g.Cin;
  p.B = g.B; p.H = Hl; p.W = Wl;
  p.tiles_x = Wl / p.bw;
  p.tiles_y = Hl / p.bh;
  p.tiles_per_phase = p.bb == 1 ? g.B * p.tiles_x * p.tiles_y : (g.B + p.bb - 1) / p.bb;
  p.out = out;
  p.bias = nullptr;
  p.out_H = Hl; p.out_W = Wl;
  p.out_scale = 1;
  p.ntiles = p.tiles_per_phase * (g.Cin / BN);
  p.chunk = tc_chunk(true);
  *BN_out = BN;
  return FG_OK;
}
int tc_conv_dgrad_ups(fg_ctx* c, const float* dy_hi, const float* dy_lo, const float* wd_hi, const float* wd_lo,
                      float* out, ConvGeom g, int f16, const float* oscale) {
  TcFwdParams p;
  int BN;
  FG_TRY(dgrad_ups_params(dy_hi, dy_lo, wd_hi, wd_lo, out, g, f16, oscale, p, &BN));
  return launch_tapconv(c, p, BN, f16);
}

// K splits of a weight gradient: about one wave of `base` CTAs per split
static int wgrad_splits(const fg_ctx* c, int base, int kblocks) {
  const int splits = std::min(std::max(1, c->sm_count / base), kblocks);
  const int per = (kblocks + splits - 1) / splits;
  return (kblocks + per - 1) / per;
}

// wgrad.  x_hi/lo: [B][H/ups][W/ups][Cin]; dy_hi/lo: [B][H][W][Cout]; out (overwritten):
//   ups==1: [k*k][Cout][Cin]          ups==2: collapsed [36][Cout][Cin]
// Fills p for `splits` K splits; the caller sets p.out / p.split_stride.  *ntt_out: tile-taps, *BN_out: Cin tile.
static int wgrad_params(fg_ctx* c, const float* x_hi, const float* x_lo, const float* dy_hi, const float* dy_lo, ConvGeom g,
                        int f16, const float* oscale, const float* oscale2, TcWgParams& p, int* BN_out, int* ntt_out,
                        int* splits_out) {
  memset(&p, 0, sizeof(p));
  const int Hl = g.H / g.ups, Wl = g.W / g.ups;
  const bool h = f16 != 0;
  const int es = h ? 2 : 4, gch = h ? 64 : 32;  // element bytes; channels per 128-byte group
  if (!pick_box(Hl, Wl, h ? 64 : 32, &p.bw, &p.bh, &p.bb)) return FG_ERR_UNSUPPORTED;
  if (g.Cin % 64 || g.Cout % 128) return FG_ERR_UNSUPPORTED;
  const int BN = g.Cin % 128 == 0 ? 128 : 64;
  {
    const int64_t sW = (int64_t)g.Cin * es, sH = sW * Wl, sB = sH * Hl;
    const int ngx = BN / gch;
    FG_TRY(make_map5(&p.x_hi, x_hi, g.Cin, Wl, Hl, g.B, sW, sH, sB, p.bw, p.bh, p.bb, ngx, h));
    FG_TRY(make_map5(&p.x_lo, x_lo, g.Cin, Wl, Hl, g.B, sW, sH, sB, p.bw, p.bh, p.bb, ngx, h));
  }
  const int ngy = 128 / gch;
  int ntt;
  if (g.ups == 1) {
    const int64_t sW = (int64_t)g.Cout * es, sH = sW * g.W, sB = sH * g.H;
    FG_TRY(make_map5(&p.dy_hi[0], dy_hi, g.Cout, g.W, g.H, g.B, sW, sH, sB, p.bw, p.bh, p.bb, ngy, h));
    FG_TRY(make_map5(&p.dy_lo[0], dy_lo, g.Cout, g.W, g.H, g.B, sW, sH, sB, p.bw, p.bh, p.bb, ngy, h));
    const int pad = (g.k - 1) / 2;
    ntt = g.k * g.k;
    for (int t = 0; t < ntt; ++t) {
      p.dy[t] = (int8_t)(t / g.k - pad);
      p.dx[t] = (int8_t)(t % g.k - pad);
      p.phase[t] = 0;
    }
  } else {
    for (int ph = 0; ph < 4; ++ph) {
      const int py = ph >> 1, px = ph & 1;
      const int64_t off_bytes = ((int64_t)py * g.W + px) * g.Cout * es;
      const float* b_hi = reinterpret_cast<const float*>(reinterpret_cast<const char*>(dy_hi) + off_bytes);
      const float* b_lo = reinterpret_cast<const float*>(reinterpret_cast<const char*>(dy_lo) + off_bytes);
      const int64_t sW = (int64_t)2 * g.Cout * es, sH = (int64_t)2 * g.W * g.Cout * es, sB = (int64_t)g.H * g.W * g.Cout * es;
      FG_TRY(make_map5(&p.dy_hi[ph], b_hi, g.Cout, Wl, Hl, g.B, sW, sH, sB, p.bw, p.bh, p.bb, ngy, h));
      FG_TRY(make_map5(&p.dy_lo[ph], b_lo, g.Cout, Wl, Hl, g.B, sW, sH, sB, p.bw, p.bh, p.bb, ngy, h));
    }
    ntt = 36;
    for (int ph = 0; ph < 4; ++ph)
      for (int t = 0; t < 9; ++t) {
        p.dy[ph * 9 + t] = (int8_t)(t / 3 - 1);
        p.dx[ph * 9 + t] = (int8_t)(t % 3 - 1);
        p.phase[ph * 9 + t] = (int8_t)ph;
      }
  }
  p.Cout = g.Cout;
  p.Cin = g.Cin;
  p.tiles_x = Wl / p.bw;
  p.tiles_y = Hl / p.bh;
  p.kblocks = p.bb == 1 ? g.B * p.tiles_x * p.tiles_y : (g.B + p.bb - 1) / p.bb;
  const int splits = wgrad_splits(c, ntt * (g.Cout / 128) * (g.Cin / BN), p.kblocks);
  p.kb_per_split = (p.kblocks + splits - 1) / splits;
  p.oscale = oscale ? oscale : oscale2;
  p.oscale2 = oscale ? oscale2 : nullptr;
  p.chunk = tc_chunk() == 4 && !getenv("FG_TC_CHUNK") ? ((int64_t)g.H * g.W > 1 ? 8 : 4) : tc_chunk();  // wgrad of convolutions 8, of Linear layers 4
  if (h) p.chunk = std::max(1, p.chunk / 2);  // an fp16 K block holds 64 pixels
  *BN_out = BN;
  *ntt_out = ntt;
  *splits_out = splits;
  return FG_OK;
}
int tc_conv_wgrad(fg_ctx* c, const float* x_hi, const float* x_lo, const float* dy_hi, const float* dy_lo, float* out,
                  ConvGeom g, int f16, const float* oscale, const float* oscale2) {
  TcWgParams p;
  int BN, ntt, splits;
  FG_TRY(wgrad_params(c, x_hi, x_lo, dy_hi, dy_lo, g, f16, oscale, oscale2, p, &BN, &ntt, &splits));
  const int64_t size = (int64_t)ntt * g.Cout * g.Cin;
  p.out = splits > 1 ? c->splitk_ws : out;  // splits x base CTAs <= one per SM: fits splitk_ws
  p.split_stride = size;
  if (splits > 1 && splits * size > (int64_t)c->splitk_ws_elems) {  // an unsplit gradient goes straight to `out`
    fg_set_error("tc_conv_wgrad: %d splits of %lld elements exceed the split-K workspace", splits, (long long)size);
    return FG_ERR_UNSUPPORTED;
  }
  dim3 grid(ntt, (g.Cout / 128) * (g.Cin / BN), splits);
  note_conv(c, FG_KERNEL_WGRAD_TC, 128, BN, f16 ? 2 : 1, splits);
  if (f16) {
    if (BN == 128) wgrad_tc_kernel<128, true><<<grid, kTcThreads, wg_smem<128>(), c->stream>>>(p);
    else wgrad_tc_kernel<64, true><<<grid, kTcThreads, wg_smem<64>(), c->stream>>>(p);
  } else if (BN == 128) wgrad_tc_kernel<128><<<grid, kTcThreads, wg_smem<128>(), c->stream>>>(p);
  else wgrad_tc_kernel<64><<<grid, kTcThreads, wg_smem<64>(), c->stream>>>(p);
  LAUNCH_CHECK(c);
  return splits > 1 ? k_splitk_reduce(c, c->splitk_ws, splits, size, out) : FG_OK;
}

// The merged launch covers the shapes where both halves run BN = 128 tiles and the weight gradient is not split
// (fewer than two waves of its items fit on the GPU), so that every item is the unsplit tile of today's kernels.
bool tc_bwd_pair_eligible(const fg_ctx* c, const ConvGeom& g) {
  int bw, bh, bb;
  const int Hl = g.H / 2, Wl = g.W / 2;
  if (g.ups != 2 || g.k != 5 || g.Cin % 128 || g.Cout % 128) return false;
  if (!pick_box(Hl, Wl, 128, &bw, &bh, &bb) || !pick_box(Hl, Wl, 64, &bw, &bh, &bb)) return false;
  const int kblocks = bb == 1 ? g.B * (Wl / bw) * (Hl / bh) : (g.B + bb - 1) / bb;
  return wgrad_splits(c, 36 * (g.Cout / 128) * (g.Cin / 128), kblocks) == 1;
}

static int bwd_pair_ctas(const fg_ctx* c, int nitems) {
  int ctas = std::min(nitems, std::max(1, c->sm_count - c->reserve_sms));
  return c->bwd_merge_ctas > 0 ? std::min(ctas, c->bwd_merge_ctas) : ctas;
}

// Does the merged launch finish sooner than the two launches?  Both schedules in K-block times: two launches = the
// weight-gradient wave, then the dgrad tiles in waves; merged = the items handed out longest first to the CTA that
// frees up first.  The merged estimate must win by 5 %: next to each other the two kinds share the L2 bandwidth that
// the weight gradient had to itself (G.C1 at batch 256 ties at 400 K-block times and measured 5 % slower merged).
bool tc_bwd_pair_pays(const fg_ctx* c, const ConvGeom& g) {
  if (!tc_bwd_pair_eligible(c, g)) return false;
  int bw, bh, bb, tw, th, tb;
  const int Hl = g.H / 2, Wl = g.W / 2;
  pick_box(Hl, Wl, 64, &bw, &bh, &bb);
  pick_box(Hl, Wl, 128, &tw, &th, &tb);
  const int64_t wlen = bb == 1 ? g.B * (Wl / bw) * (Hl / bh) : (g.B + bb - 1) / bb;  // K blocks of a wgrad item
  const int64_t dlen = 36 * (g.Cout / 64);                                             // K blocks of a dgrad tile
  const int nwg = 36 * (g.Cout / 128) * (g.Cin / 128);
  const int ntiles = (tb == 1 ? g.B * (Wl / tw) * (Hl / th) : (g.B + tb - 1) / tb) * (g.Cin / 128);
  const int sms = std::max(1, c->sm_count - c->reserve_sms);
  const int64_t two = wlen + (int64_t)((ntiles + sms - 1) / sms) * dlen;
  std::priority_queue<int64_t, std::vector<int64_t>, std::greater<int64_t>> free_at;  // when each CTA frees up
  for (int i = 0, n = bwd_pair_ctas(c, nwg + ntiles); i < n; ++i) free_at.push(0);
  int64_t merged = 0;
  for (int id = 0; id < nwg + ntiles; ++id) {
    const int64_t end = free_at.top() + (id < nwg ? wlen : dlen);
    free_at.pop();
    free_at.push(end);
    merged = std::max(merged, end);
  }
  return merged * 20 < two * 19;
}

int tc_conv_bwd_ups(fg_ctx* c, const float* x_hi, const float* x_lo, const float* dy_hi, const float* dy_lo,
                    const float* wd_hi, const float* wd_lo, float* wg_out, float* dh, ConvGeom g, const float* oscale_dy,
                    const float* oscale_x) {
  if (!tc_bwd_pair_eligible(c, g)) {
    fg_set_error("tc_conv_bwd_ups: no merged backward for Cin %d, Cout %d at %dx%d, batch %d", g.Cin, g.Cout, g.H, g.W, g.B);
    return FG_ERR_UNSUPPORTED;
  }
  TcBwdParams p;
  memset(&p, 0, sizeof(p));
  int wBN, ntt, splits, dBN;
  FG_TRY(wgrad_params(c, x_hi, x_lo, dy_hi, dy_lo, g, 1, oscale_dy, oscale_x, p.wg, &wBN, &ntt, &splits));
  FG_TRY(dgrad_ups_params(dy_hi, dy_lo, wd_hi, wd_lo, dh, g, 1, oscale_dy, p.dg, &dBN));
  if (wBN != 128 || dBN != 128 || splits != 1) {
    fg_set_error("tc_conv_bwd_ups: unexpected tiling (wgrad BN %d, %d splits, dgrad BN %d)", wBN, splits, dBN);
    return FG_ERR_UNSUPPORTED;
  }
  p.wg.out = wg_out;
  p.wg.split_stride = 0;
  p.claim = c->bwd_claim;
  p.nwg = ntt * (g.Cout / 128) * (g.Cin / 128);
  p.nitems = p.nwg + p.dg.ntiles;
  const int ctas = bwd_pair_ctas(c, p.nitems);
  FG_CUDA(cudaMemsetAsync(c->bwd_claim, 0, sizeof(int), c->stream));  // part of a captured step: reset on every replay
  bwd_pair_tc_kernel<128><<<ctas, kTcThreads, bwd_smem<128>(), c->stream>>>(p);
  LAUNCH_CHECK(c);
  return FG_OK;
}
