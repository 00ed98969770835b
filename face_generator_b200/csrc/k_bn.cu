// BatchNorm per-channel reductions at HBM speed (NHWC, C % 4 == 0): every thread owns 4 consecutive channels
// (one float4 per pixel row), blockDim/(C/4) pixel rows are in flight per block iteration, accumulation in
// double, one shared-memory tree per block, then the per-block partials are added in block order (k_ordered.cuh).
//   stats   : acc[c] += sum z,            acc[C+c] += sum z^2                       (forward, models.lua:65,70)
//   bwd     : acc[c] += sum g,            acc[C+c] += sum g*xhat,  *dslope += sum_{u<=0} dh*u
//             with u = gamma*xhat+beta, g = dh*(u>0 ? 1 : a)                         (backward of BN+PReLU)
#include "fg_internal.h"
#include "k_ordered.cuh"

#define LAUNCH_CHECK(c)                 \
  do {                                  \
    (c)->launches++;                    \
    FG_CUDA(cudaGetLastError());        \
  } while (0)

namespace {
template <bool BWD>
__global__ void __launch_bounds__(256) bn_reduce4_kernel(const float* __restrict__ z, const float* __restrict__ dh,
                                                         const float* __restrict__ mean, const float* __restrict__ istd,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta,
                                                         const float* __restrict__ slope, double* __restrict__ acc,
                                                         float* __restrict__ dslope, int64_t P, int C,
                                                         int64_t rows_per_block, double* __restrict__ ws,
                                                         unsigned* __restrict__ ticket) {
  extern __shared__ double sm[];  // [2][lanes][C]
  const int C4 = C >> 2;
  const int lanes = blockDim.x / C4;
  const int c4 = threadIdx.x % C4, lane = threadIdx.x / C4;
  const int ch = c4 * 4;
  const int64_t r0 = blockIdx.x * rows_per_block, r1 = min(P, r0 + rows_per_block);
  const float4* z4 = reinterpret_cast<const float4*>(z);
  const float4* d4 = reinterpret_cast<const float4*>(dh);
  double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0}, ss = 0;
  float m[4], is[4], ga[4], be[4];
  float a = 1.f;
  bool act = false;
  if (BWD) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      m[j] = mean[ch + j];
      is[j] = istd[ch + j];
      ga[j] = gamma[ch + j];
      be[j] = beta[ch + j];
    }
    act = slope != nullptr;
    if (act) a = *slope;
  }
  if (lane < lanes) {
    int64_t r = r0 + lane;
    if (!BWD) {
      // 4 independent 16-byte loads in flight per thread (a single dependent load per iteration left the kernel at
      // ~36 % of the HBM rate); accumulation stays in double
      for (; r + 3 * (int64_t)lanes < r1; r += 4 * (int64_t)lanes) {
        const float4 v0 = z4[r * C4 + c4], v1 = z4[(r + lanes) * C4 + c4], v2 = z4[(r + 2 * (int64_t)lanes) * C4 + c4],
                     v3 = z4[(r + 3 * (int64_t)lanes) * C4 + c4];
        const float a[4][4] = {{v0.x, v0.y, v0.z, v0.w}, {v1.x, v1.y, v1.z, v1.w}, {v2.x, v2.y, v2.z, v2.w}, {v3.x, v3.y, v3.z, v3.w}};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[j] += ((double)a[0][j] + (double)a[1][j]) + ((double)a[2][j] + (double)a[3][j]);
          q[j] += (double)a[0][j] * (double)a[0][j] + (double)a[1][j] * (double)a[1][j] + (double)a[2][j] * (double)a[2][j] +
                  (double)a[3][j] * (double)a[3][j];
        }
      }
    }
    auto bwd_row = [&](const float4& v, const float4& d) {
      const float zv[4] = {v.x, v.y, v.z, v.w};
      const float dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (zv[j] - m[j]) * is[j];
        float g = dv[j];
        if (act) {
          const float u = ga[j] * xh + be[j];
          if (!(u > 0.f)) {
            g = a * dv[j];
            ss += (double)dv[j] * (double)u;
          }
        }
        s[j] += (double)g;
        q[j] += (double)g * (double)xh;
      }
    };
    if (BWD) {  // two rows = four independent 16-byte loads in flight
      for (; r + lanes < r1; r += 2 * (int64_t)lanes) {
        const float4 v0 = z4[r * C4 + c4], d0 = d4[r * C4 + c4], v1 = z4[(r + lanes) * C4 + c4], d1 = d4[(r + lanes) * C4 + c4];
        bwd_row(v0, d0);
        bwd_row(v1, d1);
      }
    }
    for (; r < r1; r += lanes) {
      const float4 v = z4[r * C4 + c4];
      if (!BWD) {
        const float zv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[j] += (double)zv[j];
          q[j] += (double)zv[j] * (double)zv[j];
        }
      } else {
        bwd_row(v, d4[r * C4 + c4]);
      }
    }
  }
  double* s0 = sm;
  double* s1 = sm + (size_t)lanes * C;
  if (lane < lanes) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      s0[lane * C + ch + j] = s[j];
      s1[lane * C + ch + j] = q[j];
    }
  }
  __syncthreads();
  // this block's row of partials: [sum | sum of squares / products | PReLU slope sum]
  double* row = ws + (int64_t)blockIdx.x * (2 * C + 1);
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    double a0 = 0, a1 = 0;
    for (int l = 0; l < lanes; ++l) {
      a0 += s0[l * C + i];
      a1 += s1[l * C + i];
    }
    row[i] = a0;
    row[C + i] = a1;
  }
  if (threadIdx.x == 0) row[2 * C] = 0.0;
  if (BWD && act && dslope) {
    // block-wide sum of ss
    __shared__ double red[32];
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < 32) {
      double v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (threadIdx.x == 0) row[2 * C] = v;
    }
  }
  if (ordered_last_block(ticket)) {
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] += ordered_sum(ws, gridDim.x, 2 * C + 1, i);
    if (BWD && dslope && threadIdx.x == 0) *dslope += (float)ordered_sum(ws, gridDim.x, 2 * C + 1, 2 * C);
    ordered_release(ticket);
  }
}
}  // namespace

bool k_bn4_ok(int C) { return C % 4 == 0 && C >= 16 && C <= 1024 && 256 % (C / 4) == 0; }

int k_bn_stats4(fg_ctx* c, const float* z, double* acc, int64_t P, int C) {
  FG_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * C, c->stream));
  const int lanes = 256 / (C / 4);
  int grid = (int)std::min<int64_t>((int64_t)c->sm_count * 8, (P + lanes * 4 - 1) / (lanes * 4));
  if (grid < 1) grid = 1;
  const int64_t rpb = (P + grid - 1) / grid;
  FG_TRY(red_check(c, grid, 2 * C + 1));
  bn_reduce4_kernel<false><<<grid, 256, sizeof(double) * 2 * lanes * C, c->stream>>>(z, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                                                   nullptr, acc, nullptr, P, C, rpb, c->red_ws,
                                                                                   c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_bn_bwd_reduce4(fg_ctx* c, const float* dh, const float* z, const float* mean, const float* istd, const float* gamma,
                     const float* beta, const float* slope, double* acc, float* dslope, int64_t P, int C) {
  FG_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * C, c->stream));
  const int lanes = 256 / (C / 4);
  int grid = (int)std::min<int64_t>((int64_t)c->sm_count * 8, (P + lanes * 4 - 1) / (lanes * 4));
  if (grid < 1) grid = 1;
  const int64_t rpb = (P + grid - 1) / grid;
  FG_TRY(red_check(c, grid, 2 * C + 1));
  bn_reduce4_kernel<true><<<grid, 256, sizeof(double) * 2 * lanes * C, c->stream>>>(z, dh, mean, istd, gamma, beta, slope, acc,
                                                                                  dslope, P, C, rpb, c->red_ws, c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}
