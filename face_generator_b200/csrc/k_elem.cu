// Bandwidth-bound kernels of the G/D train step (everything that is not a convolution/GEMM):
// layout changes at the ABI, weight packing, BatchNorm statistics/apply/backward, PReLU, pooling,
// dropout, sigmoid+BCE, penalty+clamp+Adam.  All tensors NHWC fp32, channels fastest, so a warp
// reads consecutive channels of one pixel (coalesced 128B lines); per-channel reductions keep
// double accumulators per block (warp-shuffle / smem trees) and add the per-block partials in block order.
//
// Reference semantics: SURVEY.md section 8a; nn.* classes named per kernel below.
#include <cmath>

#include "convl.h"
#include "fg_internal.h"
#include "k_f16split.cuh"
#include "k_ordered.cuh"

__device__ __forceinline__ int perm_idx(int j, int A, int S) {
  if (A == 0) return j;
  return (j % S) * A + (j / S);
}

__global__ void fill_kernel(float* p, float v, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}
int k_fill(fg_ctx* c, float* p, float v, int64_t n) {
  if (n <= 0) return FG_OK;
  fill_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(p, v, n);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// NCHW <-> NHWC (only used at the ABI: images have C in {1,3}; L-op tensors any C)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int HW) {
  const int64_t n = (int64_t)B * C * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    const int64_t r = i / C;
    const int p = (int)(r % HW);
    const int b = (int)(r / HW);
    dst[i] = src[((int64_t)b * C + ch) * HW + p];
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int HW) {
  const int64_t n = (int64_t)B * C * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(i % HW);
    const int64_t r = i / HW;
    const int ch = (int)(r % C);
    const int b = (int)(r / C);
    dst[i] = src[((int64_t)b * HW + p) * C + ch];
  }
}
int k_nchw_to_nhwc(fg_ctx* c, const float* src, float* dst, int B, int C, int HW) {
  nchw_to_nhwc_kernel<<<grid_for((int64_t)B * C * HW, 256), 256, 0, c->stream>>>(src, dst, B, C, HW);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_nhwc_to_nchw(fg_ctx* c, const float* src, float* dst, int B, int C, int HW) {
  nhwc_to_nchw_kernel<<<grid_for((int64_t)B * C * HW, 256), 256, 0, c->stream>>>(src, dst, B, C, HW);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// weight packing (reference layout [N][Cc][KK] -> tap-major packs)
// ------------------------------------------------------------------------------------------------
__global__ void pack_weights_kernel(const float* __restrict__ W, float* __restrict__ Wp, float* __restrict__ Wpd, int N,
                                    int Cc, int KK, int nA, int nS, int cA, int cS) {
  const int64_t total = (int64_t)N * Cc * KK;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc);
    const int n = (int)(r / Cc);
    const int n2 = perm_idx(n, nA, nS), c2 = perm_idx(ch, cA, cS);
    const float w = W[i];
    if (Wp) Wp[((int64_t)t * N + n2) * Cc + c2] = w;
    if (Wpd) Wpd[((int64_t)(KK - 1 - t) * Cc + c2) * N + n2] = w;
  }
}
int k_pack_weights(fg_ctx* c, const float* W, float* Wp, float* Wpd, int N, int Cc, int KK, int nA, int nS, int cA,
                   int cS) {
  pack_weights_kernel<<<grid_for((int64_t)N * Cc * KK, 256), 256, 0, c->stream>>>(W, Wp, Wpd, N, Cc, KK, nA, nS, cA, cS);
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void unpack_wgrad_kernel(const float* __restrict__ dWp, float* __restrict__ dW, int N, int Cc, int KK, int nA,
                                    int nS, int cA, int cS) {
  const int64_t total = (int64_t)N * Cc * KK;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % KK);
    const int64_t r = i / KK;
    const int ch = (int)(r % Cc);
    const int n = (int)(r / Cc);
    const int n2 = perm_idx(n, nA, nS), c2 = perm_idx(ch, cA, cS);
    dW[i] += dWp[((int64_t)t * N + n2) * Cc + c2];
  }
}
int k_unpack_wgrad(fg_ctx* c, const float* dWp, float* dW, int N, int Cc, int KK, int nA, int nS, int cA, int cS) {
  unpack_wgrad_kernel<<<grid_for((int64_t)N * Cc * KK, 256), 256, 0, c->stream>>>(dWp, dW, N, Cc, KK, nA, nS, cA, cS);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// out[j] += sum_p X[p][perm(j)]   (bias gradients)
__global__ void colsum_kernel(const float* __restrict__ X, float* __restrict__ out, int64_t P, int N, int nA, int nS,
                              int64_t rows_per_block, double* __restrict__ ws, unsigned* __restrict__ ticket) {
  __shared__ double sm[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = blockIdx.y * rows_per_block;
  const int64_t r1 = min(P, r0 + rows_per_block);
  double s = 0;
  if (col < N)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += X[r * N + col];
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    double t = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
    // inverse permutation: column col == perm(j)  =>  j = perm^-1(col) = perm with (A,S) swapped
    const int j = nA == 0 ? col : (col % nA) * nS + (col / nA);
    ws[(int64_t)blockIdx.y * N + j] = t;  // row blockIdx.y: the blocks of one row slice cover all N columns
  }
  if (ordered_last_block(ticket)) {
    for (int j = threadIdx.y * blockDim.x + threadIdx.x; j < N; j += blockDim.x * blockDim.y)
      out[j] += (float)ordered_sum(ws, gridDim.y, N, j);
    ordered_release(ticket);
  }
}
int k_colsum_add(fg_ctx* c, const float* X, float* out, int64_t P, int N, int nA, int nS) {
  int gy = (int)std::min<int64_t>(256, (P + 255) / 256);
  if (gy < 1) gy = 1;
  const int64_t rpb = (P + gy - 1) / gy;
  dim3 grid((N + 31) / 32, gy), block(32, 8);
  FG_TRY(red_check(c, gy, N));
  colsum_kernel<<<grid, block, 0, c->stream>>>(X, out, P, N, nA, nS, rpb, c->red_ws, c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// nn.PReLU (one shared slope)
// ------------------------------------------------------------------------------------------------
__global__ void prelu_fwd_kernel(const float* __restrict__ z, const float* __restrict__ slope, float* __restrict__ h,
                                 int64_t n, unsigned* __restrict__ amax) {
  const float a = *slope;
  float am = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = z[i];
    const float o = v > 0.f ? v : a * v;
    h[i] = o;
    am = fmaxf(am, finite_abs(o));
  }
  amax_commit(amax, am);
}
int k_prelu_fwd(fg_ctx* c, const float* z, const float* slope, float* h, int64_t n) {
  prelu_fwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(z, slope, h, n, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}

// load dh at low-res pixel (b,y,x,ch); pool=1: dh is [B][2H][2W][C], return the 2x2 sum
// (backward of nn.SpatialUpSamplingNearest(2))
__device__ __forceinline__ float load_dh(const float* __restrict__ dh, int b, int y, int x, int ch, int H, int W, int C,
                                         int pool) {
  if (!pool) return dh[(((int64_t)b * H + y) * W + x) * C + ch];
  const int64_t base = (((int64_t)b * 2 * H + 2 * y) * 2 * W + 2 * x) * C + ch;
  const int64_t rs = (int64_t)2 * W * C;
  return (dh[base] + dh[base + C]) + (dh[base + rs] + dh[base + rs + C]);
}

__global__ void prelu_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ z,
                                 const float* __restrict__ slope, float* __restrict__ dz, float* __restrict__ dslope, int B,
                                 int H, int W, int C, int pool, unsigned* __restrict__ amax, double* __restrict__ ws,
                                 unsigned* __restrict__ ticket) {
  const float a = *slope;
  const int64_t n = (int64_t)B * H * W * C;
  double s = 0;
  float am = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int x = (int)(r % W);
    r /= W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    const float g = load_dh(dh, b, y, x, ch, H, W, C, pool);
    const float v = z[i];
    if (v > 0.f) {
      dz[i] = g;
      am = fmaxf(am, finite_abs(g));
    } else {
      dz[i] = a * g;
      am = fmaxf(am, finite_abs(a * g));
      s += (double)g * (double)v;
    }
  }
  amax_commit(amax, am);
  s = block_sum(s);
  if (!dslope) return;
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *dslope += (float)ordered_sum(ws, gridDim.x, 1, 0);
    ordered_release(ticket);
  }
}
int k_prelu_bwd(fg_ctx* c, const float* dh, const float* z, const float* slope, float* dz, float* dslope, int B, int H,
                int W, int C, int pool) {
  const int64_t n = (int64_t)B * H * W * C;
  prelu_bwd_kernel<<<grid_for(n, 256, 132 * 8), 256, 0, c->stream>>>(dh, z, slope, dz, dslope, B, H, W, C, pool, take_amax(c),
                                                                    c->red_ws, c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// nn.SpatialBatchNormalization (training: batch mean / biased variance, eps=1e-5, momentum 0.1)
// ------------------------------------------------------------------------------------------------
// acc[0..C) += sum_p z, acc[C..2C) += sum_p z^2   (double; caller zeroes acc)
__global__ void bn_stats_kernel(const float* __restrict__ z, double* __restrict__ acc, int64_t P, int C,
                                int64_t rows_per_block, double* __restrict__ ws, unsigned* __restrict__ ticket) {
  extern __shared__ double sm[];  // [2][blockDim]
  const int lanes = blockDim.x / C;
  const int ch = threadIdx.x % C, lane = threadIdx.x / C;
  const int64_t r0 = blockIdx.x * rows_per_block, r1 = min(P, r0 + rows_per_block);
  double s = 0, s2 = 0;
  for (int64_t r = r0 + lane; r < r1; r += lanes) {
    const double v = z[r * C + ch];
    s += v;
    s2 += v * v;
  }
  sm[threadIdx.x] = s;
  sm[blockDim.x + threadIdx.x] = s2;
  __syncthreads();
  if (lane == 0) {
    for (int l = 1; l < lanes; ++l) {
      s += sm[l * C + ch];
      s2 += sm[blockDim.x + l * C + ch];
    }
    ws[(int64_t)blockIdx.x * 2 * C + ch] = s;
    ws[(int64_t)blockIdx.x * 2 * C + C + ch] = s2;
  }
  if (ordered_last_block(ticket)) {
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] += ordered_sum(ws, gridDim.x, 2 * C, i);
    ordered_release(ticket);
  }
}
static inline int bn_block(int C) {
  int lanes = 256 / C;
  if (lanes < 1) lanes = 1;
  return C * lanes;
}
int k_bn_stats(fg_ctx* c, const float* z, double* acc, int64_t P, int C) {
  if (k_bn4_ok(C)) return k_bn_stats4(c, z, acc, P, C);  // float4 / multi-row version (k_bn.cu)
  if (C > 1024) {
    fg_set_error("BatchNorm with C=%d > 1024 unsupported", C);
    return FG_ERR_UNSUPPORTED;
  }
  FG_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * C, c->stream));
  const int block = bn_block(C);
  int grid = (int)std::min<int64_t>(c->sm_count * 4, (P + 63) / 64);
  if (grid < 1) grid = 1;
  const int64_t rpb = (P + grid - 1) / grid;
  FG_TRY(red_check(c, grid, 2 * C));
  bn_stats_kernel<<<grid, block, sizeof(double) * 2 * block, c->stream>>>(z, acc, P, C, rpb, c->red_ws, c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void bn_finalize_kernel(const double* __restrict__ acc, float* __restrict__ mean, float* __restrict__ istd,
                                   float* __restrict__ run_mean, float* __restrict__ run_var, int64_t P, int C) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= C) return;
  const double n = (double)P;
  const double m = acc[ch] / n;
  double var = acc[C + ch] / n - m * m;
  if (var < 0) var = 0;
  mean[ch] = (float)m;
  istd[ch] = (float)(1.0 / sqrt(var + 1e-5));
  if (run_mean) run_mean[ch] = 0.9f * run_mean[ch] + 0.1f * (float)m;
  if (run_var) run_var[ch] = 0.9f * run_var[ch] + 0.1f * (float)(P > 1 ? var * n / (n - 1.0) : var);
}
int k_bn_finalize(fg_ctx* c, double* acc, float* mean, float* istd, float* run_mean, float* run_var, int64_t P, int C) {
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, c->stream>>>(acc, mean, istd, run_mean, run_var, P, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// BatchNorm statistics from the per-tile partials the tensor-core convolution wrote in its epilogue
// (part[tile][3][C]: over the tile's n_i valid pixels the sums s_i of z and q_i of z^2, and the sum m2_i of squared
// deviations from the tile's mean s_i / n_i).  The one-pass variance sum q_i / n - mean^2 is exact enough while the
// channel's mean square is within kBnOnePassRatio of var + eps: it then loses less than 4 of fp32's bits of the
// variance to cancellation.  Beyond that (a mean far from 0 against the spread, or a variance below eps) the variance
// comes from the third partial instead: with r = tile 0's mean, sum (s_i - n_i r) and sum m2_i + (s_i - n_i r)^2 / n_i
// are double sums without cancellation.  Grid (C/32, S slices): a block of 32 channels x 8 thread groups sums its slice
// of the tiles in a fixed order and writes a per-slice partial; the block that finishes LAST (atomic ticket per channel
// group) adds the S slice partials in slice order and finalises.  Every sum has a fixed order whatever the
// scheduling => data-parallel replicas stay bit-identical.
constexpr int kBnSlices = 32;
constexpr double kBnOnePassRatio = 16.0;
// valid pixels of epilogue tile i: tiles are 128 pixels of one output phase (nphase phases, phase fastest); only the
// last tile of each phase can be short, when its box holds several images and the batch ends inside it
__device__ __forceinline__ double bn_tile_count(int i, int nphase, int64_t phase_pixels) {
  return (double)min((int64_t)128, phase_pixels - (int64_t)(i / nphase) * 128);
}
__global__ void __launch_bounds__(256) bn_finalize_parts_kernel(const float* __restrict__ part, int nparts, int nphase,
                                                                double* __restrict__ slice_acc,
                                                                unsigned int* __restrict__ ticket, float* __restrict__ mean,
                                                                float* __restrict__ istd, float* __restrict__ run_mean,
                                                                float* __restrict__ run_var, int64_t P, int C) {
  __shared__ double sm[4][8][32];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int ch = blockIdx.x * 32 + lane;
  const int per = (nparts + kBnSlices - 1) / kBnSlices;
  const int i0 = blockIdx.y * per, i1 = min(nparts, i0 + per);
  const int64_t pp = P / nphase;
  const double r = ch < C ? (double)part[ch] / bn_tile_count(0, nphase, pp) : 0.0;
  double s = 0, q = 0, ds = 0, dq = 0;
  if (ch < C)
    for (int i = i0 + g; i < i1; i += 8) {
      const double si = (double)part[((int64_t)i * 3 + 0) * C + ch];
      s += si;
      q += (double)part[((int64_t)i * 3 + 1) * C + ch];
      const double n = bn_tile_count(i, nphase, pp), d = si - n * r;
      ds += d;
      dq += (double)part[((int64_t)i * 3 + 2) * C + ch] + d * d * (n == 128.0 ? 1.0 / 128 : 1.0 / n);
    }
  sm[0][g][lane] = s;
  sm[1][g][lane] = q;
  sm[2][g][lane] = ds;
  sm[3][g][lane] = dq;
  __syncthreads();
  if (g == 0 && ch < C) {
    for (int k = 1; k < 8; ++k) {
      s += sm[0][k][lane];
      q += sm[1][k][lane];
      ds += sm[2][k][lane];
      dq += sm[3][k][lane];
    }
    slice_acc[((int64_t)blockIdx.y * 4 + 0) * C + ch] = s;
    slice_acc[((int64_t)blockIdx.y * 4 + 1) * C + ch] = q;
    slice_acc[((int64_t)blockIdx.y * 4 + 2) * C + ch] = ds;
    slice_acc[((int64_t)blockIdx.y * 4 + 3) * C + ch] = dq;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket + blockIdx.x, 1u) == (unsigned)kBnSlices - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x == 0) ticket[blockIdx.x] = 0;  // ready for the next launch
  if (g != 0 || ch >= C) return;
  s = q = ds = dq = 0;
  for (int k = 0; k < kBnSlices; ++k) {
    s += slice_acc[((int64_t)k * 4 + 0) * C + ch];
    q += slice_acc[((int64_t)k * 4 + 1) * C + ch];
    ds += slice_acc[((int64_t)k * 4 + 2) * C + ch];
    dq += slice_acc[((int64_t)k * 4 + 3) * C + ch];
  }
  const double n = (double)P;
  const double m = s / n;
  double var = q / n - m * m;
  if (var < 0) var = 0;
  if (q / n > kBnOnePassRatio * (var + 1e-5)) var = fmax(0.0, (dq - ds * (ds / n)) / n);  // the one pass cancelled
  mean[ch] = (float)m;
  istd[ch] = (float)(1.0 / sqrt(var + 1e-5));
  if (run_mean) run_mean[ch] = 0.9f * run_mean[ch] + 0.1f * (float)m;
  if (run_var) run_var[ch] = 0.9f * run_var[ch] + 0.1f * (float)(P > 1 ? var * n / (n - 1.0) : var);
}
// slice_ws: kBnSlices * 4 * C doubles + (C/32) tickets (zeroed once at allocation)
int k_bn_finalize_parts(fg_ctx* c, const float* part, int nparts, int nphase, float* mean, float* istd, float* run_mean,
                        float* run_var, int64_t P, int C) {
  double* acc = c->bn_slice_acc;
  unsigned int* ticket = reinterpret_cast<unsigned int*>(acc + (size_t)kBnSlices * 4 * 256);
  bn_finalize_parts_kernel<<<dim3((C + 31) / 32, kBnSlices), 256, 0, c->stream>>>(part, nparts, nphase, acc, ticket, mean, istd,
                                                                                run_mean, run_var, P, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void bn_eval_prep_kernel(const float* __restrict__ rm, const float* __restrict__ rv, float* __restrict__ mean,
                                    float* __restrict__ istd, int C) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= C) return;
  mean[ch] = rm[ch];
  istd[ch] = 1.0f / sqrtf(rv[ch] + 1e-5f);
}
int k_bn_eval_prep(fg_ctx* c, const float* rm, const float* rv, float* mean, float* istd, int C) {
  bn_eval_prep_kernel<<<(C + 127) / 128, 128, 0, c->stream>>>(rm, rv, mean, istd, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// h = prelu(gamma * ((z-mean)*istd) + beta)     (slope == nullptr: plain BN output)
__global__ void bn_prelu_apply_kernel(const float* __restrict__ z, const float* __restrict__ mean,
                                      const float* __restrict__ istd, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, const float* __restrict__ slope,
                                      float* __restrict__ h, float* __restrict__ hi, float* __restrict__ lo, int64_t n4,
                                      int C, unsigned* __restrict__ amax) {
  float am = 0.f;
  const bool act = slope != nullptr;
  const float a = act ? *slope : 1.f;
  const float4* z4 = reinterpret_cast<const float4*>(z);
  float4* h4 = reinterpret_cast<float4*>(h);
  float4* hi4 = reinterpret_cast<float4*>(hi);
  float4* lo4 = reinterpret_cast<float4*>(lo);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)((i * 4) % C);
    const float4 v = z4[i];
    const float4 m = *reinterpret_cast<const float4*>(mean + ch);
    const float4 s = *reinterpret_cast<const float4*>(istd + ch);
    // gamma/beta live inside the flat parameter vector at arbitrary (unaligned) offsets: scalar loads
    const float4 g = make_float4(gamma[ch], gamma[ch + 1], gamma[ch + 2], gamma[ch + 3]);
    const float4 b = make_float4(beta[ch], beta[ch + 1], beta[ch + 2], beta[ch + 3]);
    float4 o;
    o.x = g.x * ((v.x - m.x) * s.x) + b.x;
    o.y = g.y * ((v.y - m.y) * s.y) + b.y;
    o.z = g.z * ((v.z - m.z) * s.z) + b.z;
    o.w = g.w * ((v.w - m.w) * s.w) + b.w;
    if (act) {
      o.x = o.x > 0.f ? o.x : a * o.x;
      o.y = o.y > 0.f ? o.y : a * o.y;
      o.z = o.z > 0.f ? o.z : a * o.z;
      o.w = o.w > 0.f ? o.w : a * o.w;
    }
    if (h) h4[i] = o;
    am = amax4(am, o.x, o.y, o.z, o.w);
    if (hi) {  // TF32 hi/lo split for the tensor-core consumer, written here instead of by a separate pass
      float4 vh, vl;
      vh.x = __uint_as_float((__float_as_uint(o.x) + 0x1000u) & 0xFFFFE000u);
      vh.y = __uint_as_float((__float_as_uint(o.y) + 0x1000u) & 0xFFFFE000u);
      vh.z = __uint_as_float((__float_as_uint(o.z) + 0x1000u) & 0xFFFFE000u);
      vh.w = __uint_as_float((__float_as_uint(o.w) + 0x1000u) & 0xFFFFE000u);
      vl = make_float4(o.x - vh.x, o.y - vh.y, o.z - vh.z, o.w - vh.w);
      hi4[i] = vh;
      lo4[i] = vl;
    }
  }
  amax_commit(amax, am);
}
__global__ void bn_prelu_apply_scalar_kernel(const float* __restrict__ z, const float* __restrict__ mean,
                                             const float* __restrict__ istd, const float* __restrict__ gamma,
                                             const float* __restrict__ beta, const float* __restrict__ slope,
                                             float* __restrict__ h, int64_t n, int C) {
  const bool act = slope != nullptr;
  const float a = act ? *slope : 1.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    float o = gamma[ch] * ((z[i] - mean[ch]) * istd[ch]) + beta[ch];
    if (act) o = o > 0.f ? o : a * o;
    h[i] = o;
  }
}
int k_bn_prelu_apply(fg_ctx* c, const float* z, const float* mean, const float* istd, const float* gamma,
                     const float* beta, const float* slope, float* h, int64_t P, int C, float* hi, float* lo) {
  const int64_t n = P * C;
  if (C % 4 == 0) {
    bn_prelu_apply_kernel<<<grid_for(n / 4, 256), 256, 0, c->stream>>>(z, mean, istd, gamma, beta, slope, h, hi, lo, n / 4, C,
                                                                       take_amax(c));
  } else {
    if (hi || !h) {
      fg_set_error("bn_prelu_apply: hi/lo outputs need C %% 4 == 0");
      return FG_ERR_UNSUPPORTED;
    }
    bn_prelu_apply_scalar_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(z, mean, istd, gamma, beta, slope, h, n, C);
  }
  LAUNCH_CHECK(c);
  return FG_OK;
}

// backward pass 1: per channel  acc[ch] += sum g,  acc[C+ch] += sum g*xhat,  *dslope += sum_{u<=0} dh*u
//   u = gamma*xhat+beta (BN output), g = dh * (u>0 ? 1 : a)        (slope==nullptr: g = dh)
__global__ void bn_prelu_bwd_reduce_kernel(const float* __restrict__ dh, const float* __restrict__ z,
                                           const float* __restrict__ mean, const float* __restrict__ istd,
                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                           const float* __restrict__ slope, double* __restrict__ acc,
                                           float* __restrict__ dslope, int B, int H, int W, int C, int pool,
                                           int64_t rows_per_block, double* __restrict__ ws, unsigned* __restrict__ ticket) {
  extern __shared__ double sm[];
  const int lanes = blockDim.x / C;
  const int ch = threadIdx.x % C, lane = threadIdx.x / C;
  const int64_t P = (int64_t)B * H * W;
  const int64_t r0 = blockIdx.x * rows_per_block, r1 = min(P, r0 + rows_per_block);
  const bool act = slope != nullptr;
  const float a = act ? *slope : 1.f;
  const float m = mean[ch], is = istd[ch], ga = gamma[ch], be = beta[ch];
  double sg = 0, sgx = 0, ss = 0;
  for (int64_t r = r0 + lane; r < r1; r += lanes) {
    float d;
    if (pool) {
      const uint32_t ru = (uint32_t)r;
      const int x = (int)(ru % (uint32_t)W);
      const uint32_t q = ru / (uint32_t)W;
      d = load_dh(dh, (int)(q / (uint32_t)H), (int)(q % (uint32_t)H), x, ch, H, W, C, 1);
    } else {
      d = dh[r * C + ch];
    }
    const float xh = (z[r * C + ch] - m) * is;
    float g = d;
    if (act) {
      const float u = ga * xh + be;
      if (!(u > 0.f)) {
        g = a * d;
        ss += (double)d * (double)u;
      }
    }
    sg += g;
    sgx += (double)g * (double)xh;
  }
  sm[threadIdx.x] = sg;
  sm[blockDim.x + threadIdx.x] = sgx;
  __syncthreads();
  if (lane == 0) {
    for (int l = 1; l < lanes; ++l) {
      sg += sm[l * C + ch];
      sgx += sm[blockDim.x + l * C + ch];
    }
    ws[(int64_t)blockIdx.x * (2 * C + 1) + ch] = sg;
    ws[(int64_t)blockIdx.x * (2 * C + 1) + C + ch] = sgx;
  }
  if (act) ss = block_sum(ss);
  if (threadIdx.x == 0) ws[(int64_t)blockIdx.x * (2 * C + 1) + 2 * C] = ss;
  if (ordered_last_block(ticket)) {
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] += ordered_sum(ws, gridDim.x, 2 * C + 1, i);
    if (act && dslope && threadIdx.x == 0) *dslope += (float)ordered_sum(ws, gridDim.x, 2 * C + 1, 2 * C);
    ordered_release(ticket);
  }
}
int k_bn_prelu_bwd_reduce(fg_ctx* c, const float* dh, const float* z, const float* mean, const float* istd,
                          const float* gamma, const float* beta, const float* slope, double* acc, float* dslope, int B,
                          int H, int W, int C, int pool) {
  if (!pool && k_bn4_ok(C))
    return k_bn_bwd_reduce4(c, dh, z, mean, istd, gamma, beta, slope, acc, dslope, (int64_t)B * H * W, C);
  if (C > 1024) return FG_ERR_UNSUPPORTED;
  FG_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * C, c->stream));
  const int64_t P = (int64_t)B * H * W;
  const int block = bn_block(C);
  int grid = (int)std::min<int64_t>(c->sm_count * 4, (P + 63) / 64);
  if (grid < 1) grid = 1;
  const int64_t rpb = (P + grid - 1) / grid;
  FG_TRY(red_check(c, grid, 2 * C + 1));
  bn_prelu_bwd_reduce_kernel<<<grid, block, sizeof(double) * 2 * block, c->stream>>>(dh, z, mean, istd, gamma, beta, slope,
                                                                                  acc, dslope, B, H, W, C, pool, rpb, c->red_ws,
                                                                                  c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// mg[ch] = mean g, mg[C+ch] = mean g*xhat ; dgamma += sum g*xhat ; dbeta += sum g
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ acc, float* __restrict__ mg, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, int64_t P, int C) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= C) return;
  mg[ch] = (float)(acc[ch] / (double)P);
  mg[C + ch] = (float)(acc[C + ch] / (double)P);
  if (dgamma) dgamma[ch] += (float)acc[C + ch];
  if (dbeta) dbeta[ch] += (float)acc[ch];
}
int k_bn_bwd_finalize(fg_ctx* c, double* acc, float* mg, float* dgamma, float* dbeta, int64_t P, int C) {
  bn_bwd_finalize_kernel<<<(C + 127) / 128, 128, 0, c->stream>>>(acc, mg, dgamma, dbeta, P, C);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// backward pass 2: dz = gamma*istd*(g - mean(g) - xhat*mean(g*xhat))
__global__ void bn_prelu_bwd_apply_kernel(const float* __restrict__ dh, const float* __restrict__ z,
                                          const float* __restrict__ mean, const float* __restrict__ istd,
                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                          const float* __restrict__ slope, const float* __restrict__ mg,
                                          float* __restrict__ dz, int B, int H, int W, int C, int pool) {
  const bool act = slope != nullptr;
  const float a = act ? *slope : 1.f;
  const int64_t n = (int64_t)B * H * W * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int x = (int)(r % W);
    r /= W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    const float d = load_dh(dh, b, y, x, ch, H, W, C, pool);
    const float is = istd[ch], ga = gamma[ch];
    const float xh = (z[i] - mean[ch]) * is;
    float g = d;
    if (act) {
      const float u = ga * xh + beta[ch];
      if (!(u > 0.f)) g = a * d;
    }
    dz[i] = ga * is * (g - mg[ch] - xh * mg[C + ch]);
  }
}
// Column sums of a 256-thread block whose thread t owns channels 4 (t % (C/4)) .. +3 (256 % (C/4) == 0): the block sums
// its threads in thread order into row blockIdx.x of ws ([n] doubles: C channel sums, then an optional scalar `extra`
// at index C), and the last block adds the rows in block order to dst[0..C) and, if given, to *extra_dst.
__device__ void block_colsum_rows(const float (&bs)[4], int C, int n, double* ws, unsigned* ticket, float* dst,
                                  float* extra_dst, double extra = 0.0) {
  __shared__ float tb[256][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) tb[threadIdx.x][j] = bs[j];
  __syncthreads();
  const int C4 = C / 4;
  double* row = ws + (int64_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    double s = 0;
    for (int t = i / 4; t < (int)blockDim.x; t += C4) s += tb[t][i & 3];
    row[i] = s;
  }
  if (n > C && threadIdx.x == 0) row[C] = extra;
  if (ordered_last_block(ticket)) {
    if (dst)
      for (int i = threadIdx.x; i < C; i += blockDim.x) dst[i] += (float)ordered_sum(ws, gridDim.x, n, i);
    if (extra_dst && threadIdx.x == 0) *extra_dst += (float)ordered_sum(ws, gridDim.x, n, C);
    ordered_release(ticket);
  }
}

// pool == 0 fast path: float4 along channels, no pixel decode
__global__ void bn_prelu_bwd_apply4_kernel(const float* __restrict__ dh, const float* __restrict__ z,
                                           const float* __restrict__ mean, const float* __restrict__ istd,
                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                           const float* __restrict__ slope, const float* __restrict__ mg,
                                           float* __restrict__ dz, float* __restrict__ hi, float* __restrict__ lo,
                                           float* __restrict__ dbias, int64_t n4, int C, unsigned* __restrict__ amax,
                                           double* __restrict__ ws, unsigned* __restrict__ ticket) {
  float am = 0.f;
  // dbias (optional): += column sums of dz = the gradient of the convolution bias in front of the BatchNorm.  The grid
  // stride is a multiple of C/4, so a thread always sees the same 4 channels: thread-local sums -> block sums in
  // thread order -> per-block rows added in block order (block_colsum_rows)
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
  const bool act = slope != nullptr;
  const float a = act ? *slope : 1.f;
  const float4* dh4 = reinterpret_cast<const float4*>(dh);
  const float4* z4 = reinterpret_cast<const float4*>(z);
  float4* dz4 = reinterpret_cast<float4*>(dz);
  float4* hi4 = reinterpret_cast<float4*>(hi);
  float4* lo4 = reinterpret_cast<float4*>(lo);
  const int C4 = C / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C4) * 4;
    const float4 d = dh4[i], v = z4[i];
    const float dv[4] = {d.x, d.y, d.z, d.w}, zv[4] = {v.x, v.y, v.z, v.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float is = istd[ch + j], ga = gamma[ch + j];
      const float xh = (zv[j] - mean[ch + j]) * is;
      float g = dv[j];
      if (act) {
        const float u = ga * xh + beta[ch + j];
        if (!(u > 0.f)) g = a * g;
      }
      o[j] = ga * is * (g - mg[ch + j] - xh * mg[C + ch + j]);
    }
    dz4[i] = make_float4(o[0], o[1], o[2], o[3]);
    am = amax4(am, o[0], o[1], o[2], o[3]);
    bs[0] += o[0]; bs[1] += o[1]; bs[2] += o[2]; bs[3] += o[3];
    if (hi) {  // TF32 hi/lo split of dz for the tensor-core dgrad / wgrad, written by the producer
      float h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) h[j] = __uint_as_float((__float_as_uint(o[j]) + 0x1000u) & 0xFFFFE000u);
      hi4[i] = make_float4(h[0], h[1], h[2], h[3]);
      lo4[i] = make_float4(o[0] - h[0], o[1] - h[1], o[2] - h[2], o[3] - h[3]);
    }
  }
  amax_commit(amax, am);
  if (dbias) block_colsum_rows(bs, C, C, ws, ticket, dbias, nullptr);
}
int k_bn_prelu_bwd_apply(fg_ctx* c, const float* dh, const float* z, const float* mean, const float* istd,
                         const float* gamma, const float* beta, const float* slope, const float* mg, float* dz, int B,
                         int H, int W, int C, int pool, float* hi, float* lo, float* dbias) {
  const int64_t n = (int64_t)B * H * W * C;
  if (!pool && C % 4 == 0 && C <= 1024 && 256 % (C / 4) == 0) {
    const int grid = grid_for(n / 4, 256);
    FG_TRY(red_check(c, grid, C));
    bn_prelu_bwd_apply4_kernel<<<grid, 256, 0, c->stream>>>(dh, z, mean, istd, gamma, beta, slope, mg, dz, hi, lo, dbias, n / 4,
                                                           C, take_amax(c), c->red_ws, c->red_ticket);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  if (hi) {
    fg_set_error("bn_prelu_bwd_apply: hi/lo outputs need the un-pooled float4 path");
    return FG_ERR_UNSUPPORTED;
  }
  bn_prelu_bwd_apply_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(dh, z, mean, istd, gamma, beta, slope, mg, dz, B, H,
                                                                    W, C, pool);
  LAUNCH_CHECK(c);
  if (dbias) return k_colsum_add(c, dz, dbias, (int64_t)B * H * W, C, 0, 0);  // not fused on this path
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// nn.Sigmoid
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__global__ void sigmoid_fwd_kernel(const float* __restrict__ z, float* __restrict__ y, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = sigmoidf_(z[i]);
}
int k_sigmoid_fwd(fg_ctx* c, const float* z, float* y, int64_t n) {
  sigmoid_fwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(z, y, n);
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void sigmoid_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dz,
                                   int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = y[i];
    dz[i] = dy[i] * v * (1.0f - v);
  }
}
int k_sigmoid_bwd(fg_ctx* c, const float* dy, const float* y, float* dz, int64_t n) {
  sigmoid_bwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(dy, y, dz, n);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_sigmoid_grad_mul(fg_ctx* c, const float* dout, const float* out, float* dlogit, int n) {
  return k_sigmoid_bwd(c, dout, out, dlogit, n);
}

// ------------------------------------------------------------------------------------------------
// dropout masks (throughput mode): counter-based hash RNG, keep flag = u >= p
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// seed_dev (optional): the step seed lives in device memory (so that a captured step can be replayed with a new seed);
// the effective seed is then *seed_dev * 2 + seed
__global__ void masks_generate_kernel(float* __restrict__ masks, int B, uint64_t seed, float p_spatial, float p_drop,
                                      const uint64_t* __restrict__ seed_dev) {
  if (seed_dev) seed += *seed_dev * 2;
  const int64_t n = (int64_t)B * kMaskPerSample;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % kMaskPerSample);
    const uint64_t r = splitmix64(seed * 0x100000001B3ull + (uint64_t)i);
    const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
    masks[i] = u >= (j < 960 ? p_spatial : p_drop) ? 1.f : 0.f;
  }
}
__global__ void set_u64_kernel(uint64_t* dst, uint64_t v) { *dst = v; }
int k_set_u64(fg_ctx* c, uint64_t* dst, uint64_t v) {
  set_u64_kernel<<<1, 1, 0, c->stream>>>(dst, v);
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void seed_roots_kernel(uint64_t* roots, int n) {
  const int j = threadIdx.x;
  if (j >= 1 && j < n) roots[j] = (1ull << 60) | (roots[0] << 8) | (uint64_t)j;
}
int k_seed_roots(fg_ctx* c, uint64_t* roots, int n) {
  seed_roots_kernel<<<1, 32, 0, c->stream>>>(roots, n);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_masks_generate(fg_ctx* c, float* masks, int B, uint64_t seed, float p_spatial, float p_drop, const uint64_t* seed_dev) {
  masks_generate_kernel<<<grid_for((int64_t)B * kMaskPerSample, 256), 256, 0, c->stream>>>(masks, B, seed, p_spatial,
                                                                                          p_drop, seed_dev);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// D conv blocks: PReLU -> SpatialDropout (channel mask, NO rescale) -> SpatialAveragePooling(2,2,2,2)
// ------------------------------------------------------------------------------------------------
// float4 along channels, 32-bit index math (all D tensors have < 2^31 elements and C % 4 == 0)
__device__ __forceinline__ float4 prelu4(float4 v, float a) {
  v.x = v.x > 0.f ? v.x : a * v.x;
  v.y = v.y > 0.f ? v.y : a * v.y;
  v.z = v.z > 0.f ? v.z : a * v.z;
  v.w = v.w > 0.f ? v.w : a * v.w;
  return v;
}
// TF32 hi/lo split of a float4 (hi = mantissa rounded to 10 bits, lo = exact remainder): emitted by the producers of
// the tensor-core operands so that no separate split pass reads the tensor again
__device__ __forceinline__ void split4(const float4& o, float4* hi, float4* lo, uint32_t i) {
  float4 h;
  h.x = __uint_as_float((__float_as_uint(o.x) + 0x1000u) & 0xFFFFE000u);
  h.y = __uint_as_float((__float_as_uint(o.y) + 0x1000u) & 0xFFFFE000u);
  h.z = __uint_as_float((__float_as_uint(o.z) + 0x1000u) & 0xFFFFE000u);
  h.w = __uint_as_float((__float_as_uint(o.w) + 0x1000u) & 0xFFFFE000u);
  hi[i] = h;
  lo[i] = make_float4(o.x - h.x, o.y - h.y, o.z - h.z, o.w - h.w);
}
__global__ void d_act_pool_fwd_kernel(const float* __restrict__ z, const float* __restrict__ slope,
                                      const float* __restrict__ masks, int moff, float eval_scale, float* __restrict__ p,
                                      float4* __restrict__ hi, float4* __restrict__ lo, int B, int H, int W, int C,
                                      unsigned* __restrict__ amax) {
  float am = 0.f;
  const float a = *slope;
  const uint32_t Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const uint32_t n = (uint32_t)B * Ho * Wo * C4;
  const float4* z4 = reinterpret_cast<const float4*>(z);
  float4* p4 = reinterpret_cast<float4*>(p);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t c4 = i % C4;
    uint32_t r = i / C4;
    const uint32_t xo = r % Wo;
    r /= Wo;
    const uint32_t yo = r % Ho, b = r / Ho;
    float4 m = make_float4(eval_scale, eval_scale, eval_scale, eval_scale);
    if (masks) m = *reinterpret_cast<const float4*>(masks + (size_t)b * kMaskPerSample + moff + c4 * 4);
    const uint32_t base = ((b * H + 2 * yo) * W + 2 * xo) * C4 + c4, rs = (uint32_t)W * C4;
    const float4 v0 = prelu4(z4[base], a), v1 = prelu4(z4[base + C4], a), v2 = prelu4(z4[base + rs], a),
                 v3 = prelu4(z4[base + rs + C4], a);
    float4 o;
    o.x = (v0.x * m.x + v1.x * m.x + v2.x * m.x + v3.x * m.x) * 0.25f;
    o.y = (v0.y * m.y + v1.y * m.y + v2.y * m.y + v3.y * m.y) * 0.25f;
    o.z = (v0.z * m.z + v1.z * m.z + v2.z * m.z + v3.z * m.z) * 0.25f;
    o.w = (v0.w * m.w + v1.w * m.w + v2.w * m.w + v3.w * m.w) * 0.25f;
    p4[i] = o;
    am = amax4(am, o.x, o.y, o.z, o.w);
    if (hi) split4(o, hi, lo, i);
  }
  amax_commit(amax, am);
}
int k_d_act_pool_fwd(fg_ctx* c, const float* z, const float* slope, const float* masks, int moff, float eval_scale,
                     float* p, int B, int H, int W, int C, float* hi, float* lo) {
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * C / 4;
  if (C % 4 || (moff % 4) || (int64_t)B * H * W * C >= ((int64_t)1 << 31)) {
    fg_set_error("d_act_pool_fwd: unsupported shape (C %% 4, size)");
    return FG_ERR_UNSUPPORTED;
  }
  d_act_pool_fwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(z, slope, masks, moff, eval_scale, p, reinterpret_cast<float4*>(hi),
                                                                 reinterpret_cast<float4*>(lo), B, H, W, C, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void d_act_pool_bwd_kernel(const float* __restrict__ dp, const float* __restrict__ z,
                                      const float* __restrict__ slope, const float* __restrict__ masks, int moff,
                                      float eval_scale, float* __restrict__ dz, float* __restrict__ dslope,
                                      float4* __restrict__ hi, float4* __restrict__ lo, float* __restrict__ dbias, int B,
                                      int H, int W, int C, unsigned* __restrict__ amax, double* __restrict__ ws,
                                      unsigned* __restrict__ ticket) {
  float am = 0.f;
  // one thread = one pooled pixel x 4 channels: reads dp once, handles its 2x2 window of z / dz.
  // dbias (optional): += column sums of dz (the conv bias gradient); a thread always sees the same 4 channels because the
  // grid stride is a multiple of C/4
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
  const float a = *slope;
  const uint32_t Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const uint32_t n = (uint32_t)B * Ho * Wo * C4;
  const float4* z4 = reinterpret_cast<const float4*>(z);
  const float4* dp4 = reinterpret_cast<const float4*>(dp);
  float4* dz4 = reinterpret_cast<float4*>(dz);
  float s = 0.f;  // per-thread partial over a handful of elements; summed in double across the block
  double sd = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t c4 = i % C4;
    uint32_t r = i / C4;
    const uint32_t xo = r % Wo;
    r /= Wo;
    const uint32_t yo = r % Ho, b = r / Ho;
    float4 m = make_float4(eval_scale, eval_scale, eval_scale, eval_scale);
    if (masks) m = *reinterpret_cast<const float4*>(masks + (size_t)b * kMaskPerSample + moff + c4 * 4);
    const float4 d = dp4[i];
    const float4 g = make_float4(d.x * 0.25f * m.x, d.y * 0.25f * m.y, d.z * 0.25f * m.z, d.w * 0.25f * m.w);
    const uint32_t base = ((b * H + 2 * yo) * W + 2 * xo) * C4 + c4, rs = (uint32_t)W * C4;
    s = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t idx = base + (q & 1) * C4 + (q >> 1) * rs;
      const float4 v = z4[idx];
      float4 o;
      o.x = v.x > 0.f ? g.x : a * g.x;
      o.y = v.y > 0.f ? g.y : a * g.y;
      o.z = v.z > 0.f ? g.z : a * g.z;
      o.w = v.w > 0.f ? g.w : a * g.w;
      if (!(v.x > 0.f)) s = fmaf(g.x, v.x, s);
      if (!(v.y > 0.f)) s = fmaf(g.y, v.y, s);
      if (!(v.z > 0.f)) s = fmaf(g.z, v.z, s);
      if (!(v.w > 0.f)) s = fmaf(g.w, v.w, s);
      dz4[idx] = o;
      am = amax4(am, o.x, o.y, o.z, o.w);
      bs[0] += o.x; bs[1] += o.y; bs[2] += o.z; bs[3] += o.w;
      if (hi) split4(o, hi, lo, idx);
    }
    sd += (double)s;
  }
  amax_commit(amax, am);
  sd = block_sum(sd);
  if (dbias || dslope) block_colsum_rows(bs, dbias ? (int)C : 0, (dbias ? (int)C : 0) + 1, ws, ticket, dbias, dslope, sd);
}
int k_d_act_pool_bwd(fg_ctx* c, const float* dp, const float* z, const float* slope, const float* masks, int moff,
                     float eval_scale, float* dz, float* dslope, int B, int H, int W, int C, float* hi, float* lo,
                     float* dbias) {
  const int64_t n = (int64_t)B * (H / 2) * (W / 2) * C / 4;
  if (C % 4 || (moff % 4) || (int64_t)B * H * W * C >= ((int64_t)1 << 31)) {
    fg_set_error("d_act_pool_bwd: unsupported shape (C %% 4, size)");
    return FG_ERR_UNSUPPORTED;
  }
  const bool fuse = dbias && C <= 512 && 256 % (C / 4) == 0;
  const int grid = grid_for(n, 256, 132 * 8);
  FG_TRY(red_check(c, grid, C + 1));
  d_act_pool_bwd_kernel<<<grid, 256, 0, c->stream>>>(dp, z, slope, masks, moff, eval_scale, dz, dslope,
                                                    reinterpret_cast<float4*>(hi), reinterpret_cast<float4*>(lo),
                                                    fuse ? dbias : nullptr, B, H, W, C, take_amax(c), c->red_ws, c->red_ticket);
  LAUNCH_CHECK(c);
  if (dbias && !fuse) return k_colsum_add(c, dz, dbias, (int64_t)B * H * W, C, 0, 0);
  return FG_OK;
}
// D linear blocks: PReLU -> nn.Dropout(p) (v2: kept / (1-p) in training; identity in eval)
__global__ void lin_act_drop_fwd_kernel(const float* __restrict__ z, const float* __restrict__ slope,
                                        const float* __restrict__ masks, int moff, float scale, float* __restrict__ h,
                                        int B, int N, unsigned* __restrict__ amax) {
  float am = 0.f;
  const float a = *slope;
  const int64_t n = (int64_t)B * N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % N);
    const int b = (int)(i / N);
    const float v = z[i];
    const float act = v > 0.f ? v : a * v;
    const float o = masks ? act * masks[(int64_t)b * kMaskPerSample + moff + j] * scale : act;
    h[i] = o;
    am = fmaxf(am, finite_abs(o));
  }
  amax_commit(amax, am);
}
int k_lin_act_drop_fwd(fg_ctx* c, const float* z, const float* slope, const float* masks, int moff, float scale,
                       float* h, int B, int N) {
  lin_act_drop_fwd_kernel<<<grid_for((int64_t)B * N, 256), 256, 0, c->stream>>>(z, slope, masks, moff, scale, h, B, N, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void lin_act_drop_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ z,
                                        const float* __restrict__ slope, const float* __restrict__ masks, int moff,
                                        float scale, float* __restrict__ dz, float* __restrict__ dslope, int B, int N,
                                        unsigned* __restrict__ amax, double* __restrict__ ws, unsigned* __restrict__ ticket) {
  float am = 0.f;
  const float a = *slope;
  const int64_t n = (int64_t)B * N;
  double s = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % N);
    const int b = (int)(i / N);
    const float g = masks ? dh[i] * masks[(int64_t)b * kMaskPerSample + moff + j] * scale : dh[i];
    const float v = z[i];
    if (v > 0.f) {
      dz[i] = g;
      am = fmaxf(am, finite_abs(g));
    } else {
      dz[i] = a * g;
      am = fmaxf(am, finite_abs(a * g));
      s += (double)g * (double)v;
    }
  }
  amax_commit(amax, am);
  s = block_sum(s);
  if (!dslope) return;
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *dslope += (float)ordered_sum(ws, gridDim.x, 1, 0);
    ordered_release(ticket);
  }
}
int k_lin_act_drop_bwd(fg_ctx* c, const float* dh, const float* z, const float* slope, const float* masks, int moff,
                       float scale, float* dz, float* dslope, int B, int N) {
  lin_act_drop_bwd_kernel<<<grid_for((int64_t)B * N, 256, 132), 256, 0, c->stream>>>(dh, z, slope, masks, moff, scale, dz,
                                                                                   dslope, B, N, take_amax(c), c->red_ws,
                                                                                   c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// nn.Sigmoid + nn.BCECriterion (2015 Lua form, eps=1e-12, sizeAverage), composed exactly like the
// reference chain BCE.backward -> Sigmoid.backward so a saturated sigmoid yields a 0 gradient.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float bce_term(float x, float t) {
  const float eps = 1e-12f;
  return t * logf(x + eps) + (1.0f - t) * logf(1.0f - x + eps);
}
__device__ __forceinline__ float bce_grad(float x, float t, float invN) {
  const float eps = 1e-12f;
  return -(t - x) / (x * (1.0f - x + eps) + eps) * invN;
}
__global__ void sigmoid_bce_kernel(const float* __restrict__ logit, float* __restrict__ out, float* __restrict__ dlogit,
                                   float* __restrict__ loss_out, float* __restrict__ tail4, int B, int n_ones) {
  double s = 0;
  int c0 = 0, c1 = 0, c2 = 0, c3 = 0;
  const float invN = 1.0f / (float)B;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float y = sigmoidf_(logit[i]);
    const float t = i < n_ones ? 1.f : 0.f;
    out[i] = y;
    s += (double)bce_term(y, t);
    dlogit[i] = bce_grad(y, t, invN) * y * (1.0f - y);
    const bool pred1 = y > 0.5f;
    if (t > 0.5f) {
      if (pred1) c0++; else c1++;
    } else {
      if (pred1) c2++; else c3++;
    }
  }
  s = block_sum(s);
  const double d0 = block_sum((double)c0), d1 = block_sum((double)c1), d2 = block_sum((double)c2),
               d3 = block_sum((double)c3);
  if (threadIdx.x == 0) {
    *loss_out = (float)(-s / (double)B);
    if (tail4) {
      tail4[0] = (float)d0;
      tail4[1] = (float)d1;
      tail4[2] = (float)d2;
      tail4[3] = (float)d3;
    }
  }
}
int k_sigmoid_bce(fg_ctx* c, const float* logit, float* out, float* dlogit, float* loss_out, float* tail4, int B,
                  int n_ones) {
  sigmoid_bce_kernel<<<1, 256, 0, c->stream>>>(logit, out, dlogit, loss_out, tail4, B, n_ones);
  LAUNCH_CHECK(c);
  return FG_OK;
}
__global__ void bce_fwd_kernel(const float* __restrict__ x, const float* __restrict__ t, int n, float* __restrict__ loss) {
  double s = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += (double)bce_term(x[i], t[i]);
  s = block_sum(s);
  if (threadIdx.x == 0) *loss = (float)(-s / (double)n);
}
__global__ void bce_bwd_kernel(const float* __restrict__ x, const float* __restrict__ t, int n, float* __restrict__ dx) {
  const float invN = 1.0f / (float)n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dx[i] = bce_grad(x[i], t[i], invN);
}
int k_bce_fwd(fg_ctx* c, const float* x, const float* t, int n, float* loss_out) {
  bce_fwd_kernel<<<1, 256, 0, c->stream>>>(x, t, n, loss_out);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_bce_bwd(fg_ctx* c, const float* x, const float* t, int n, float* dx) {
  bce_bwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(x, t, n, dx);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
// penalty (loss part), gate + Adam step-size preparation, fused penalty+clamp+Adam
// ------------------------------------------------------------------------------------------------
// *loss += l1*||p||_1 + l2*||p||_2^2/2                                    (adversarial.lua:105-106)
__global__ void penalty_loss_kernel(const float* __restrict__ p, int64_t n, float l1, float l2, float* __restrict__ loss,
                                    double* __restrict__ ws, unsigned* __restrict__ ticket) {
  double s1 = 0, s2 = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = p[i];
    s1 += fabs(v);
    s2 += v * v;
  }
  s1 = block_sum(s1);
  s2 = block_sum(s2);
  if (threadIdx.x == 0) ws[blockIdx.x] = l1 * s1 + l2 * s2 * 0.5;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *loss += (float)ordered_sum(ws, gridDim.x, 1, 0);
    ordered_release(ticket);
  }
}
// the optimizer of D may run on the communication stream next to the compute stream's reductions: own workspace
int k_penalty_loss(fg_ctx* c, const float* p, int64_t n, float l1, float l2, float* loss_inout) {
  penalty_loss_kernel<<<grid_for(n, 256, kOptRedRows), 256, 0, c->stream>>>(p, n, l1, l2, loss_inout, c->red_ws_opt,
                                                                           c->red_ticket + 1);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// D: accuracy history + "doTrainD" gate (adversarial.lua:126-178); both nets: t += 1 and
// stepSize = lr*sqrt(1-beta2^t)/(1-beta1^t) in double (interruptable_optimizers.lua:75-87)
// Adagrad / SGD (interruptable_optimizers.lua:7-46, :97-167) use clr = lr / (1 + nevals*lrd) with lrd = 0 (train.lua
// never sets learningRateDecay) => the step size is the learning rate; t counts evaluations (state.evalCounter).
__device__ __forceinline__ float step_size(const fg_hyper& h, int opt, float lr, double t) {
  if (opt != FG_OPT_ADAM) return lr;
  return (float)((double)lr * sqrt(1.0 - pow((double)h.beta2, t)) / (1.0 - pow((double)h.beta1, t)));
}
// accumulate: a later D iteration of the same step -- CONFUSION:add runs in every fevalD (adversarial.lua:115) and
// countTrainedD counts every iteration that stepped (:170), so conf and trained_D add up over the step's iterations
__global__ void gate_prep_kernel(DeviceStats* st, float* acc_hist, int net, fg_hyper h, const float* tail4, float total, int opt,
                                 int accumulate) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (net == FG_NET_D) {
    int interval = h.accs_interval;
    if (interval < 1) interval = 1;
    if (interval > kAccHistMax) interval = kAccHistMax;
    const float correct = tail4[0] + tail4[3];
    const float tV = correct / total;
    for (int i = 0; i < 4; ++i) st->conf[i] = (accumulate ? st->conf[i] : 0) + (int)(tail4[i] + 0.5f);
    st->acc_D = tV;
    acc_hist[st->acc_head] = tV;
    st->acc_head = (st->acc_head + 1) % interval;
    if (st->acc_count < interval) st->acc_count++;
    double m = 0;
    for (int i = 0; i < st->acc_count; ++i) m += acc_hist[i];
    m /= st->acc_count;
    const int go = m < (double)h.D_maxAcc ? 1 : 0;
    st->do_train_D = go;
    st->trained_D = (accumulate ? st->trained_D : 0) + go;
    if (go) {
      st->t_D += 1;
      st->step_D = step_size(h, opt, h.lr_D, (double)st->t_D);
    }
  } else {
    st->do_train_G = 1;
    st->t_G += 1;
    st->step_G = step_size(h, opt, h.lr_G, (double)st->t_G);
  }
}
int k_gate_and_prep(fg_ctx* c, DeviceStats* st, float* acc_hist, int net, const fg_hyper* h, const float* tail4, int B,
                    float world, bool accumulate) {
  gate_prep_kernel<<<1, 32, 0, c->stream>>>(st, acc_hist, net, *h, tail4, (float)B * world, net == FG_NET_D ? c->opt_D : c->opt_G,
                                            accumulate ? 1 : 0);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// fg_optim_step: a module-level step has no batch accuracy, so it opens the update and advances t / the step size of
// `net` only.  The accuracy history, conf, acc_D and trained_D belong to the fused steps' D iterations and stay as
// they are.
__global__ void optim_prep_kernel(DeviceStats* st, int net, fg_hyper h, int opt) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (net == FG_NET_D) {
    st->do_train_D = 1;
    st->t_D += 1;
    st->step_D = step_size(h, opt, h.lr_D, (double)st->t_D);
  } else {
    st->do_train_G = 1;
    st->t_G += 1;
    st->step_G = step_size(h, opt, h.lr_G, (double)st->t_G);
  }
}
int k_optim_prep(fg_ctx* c, DeviceStats* st, int net, const fg_hyper* h) {
  optim_prep_kernel<<<1, 32, 0, c->stream>>>(st, net, *h, net == FG_NET_D ? c->opt_D : c->opt_G);
  LAUNCH_CHECK(c);
  return FG_OK;
}
// g = grad*scale; g += l1_grad*sign(p) + l2*p; clamp; m,v EMA; p -= step*m/(sqrt(v)+eps); grads written back
__global__ void adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            int64_t n, float beta1, float beta2, float eps, float l1_grad, float l2, float clampv,
                            float grad_scale, const float* __restrict__ step_dev, const int* __restrict__ flag_dev,
                            float step_host, int update, int mode, float mom, const int* __restrict__ t_dev) {
  if (flag_dev && *flag_dev == 0) update = 0;
  const float step = step_dev ? *step_dev : step_host;
  const bool first = t_dev ? *t_dev == 1 : false;
  const bool pen = (l1_grad != 0.f) || (l2 != 0.f);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float pv = p[i];
    float gv = g[i] * grad_scale;
    if (pen) {
      const float sg = pv > 0.f ? 1.f : (pv < 0.f ? -1.f : 0.f);
      gv += sg * l1_grad + pv * l2;
    }
    if (clampv != 0.f) gv = fminf(fmaxf(gv, -clampv), clampv);
    g[i] = gv;
    if (!update) continue;
    if (mode == FG_OPT_ADAM) {  // interruptable_optimizers.lua:78-90
      const float mv = m[i] * beta1 + (1.0f - beta1) * gv;
      const float vv = v[i] * beta2 + (1.0f - beta2) * gv * gv;
      m[i] = mv;
      v[i] = vv;
      p[i] = pv - step * mv / (sqrtf(vv) + eps);
    } else if (mode == FG_OPT_ADAGRAD) {  // :33-39  paramVariance += g^2; x -= clr * g / (sqrt(paramVariance) + 1e-10)
      const float vv = v[i] + gv * gv;
      v[i] = vv;
      p[i] = pv - step * gv / (sqrtf(vv) + 1e-10f);
    } else {  // SGD :129-160 (no weight decay / nesterov / per-parameter rates in train.lua); dampening defaults to mom
      float ge = gv;
      if (mom != 0.f) {
        ge = first ? gv : m[i] * mom + (1.0f - mom) * gv;
        m[i] = ge;
      }
      p[i] = pv - step * ge;
    }
  }
}
// ------------------------------------------------------------------------------------------------
// nn.Linear(K, 1) (D's last layer, models.lua:412): a GEMV, one warp per batch row
// ------------------------------------------------------------------------------------------------
__global__ void gemv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                float* __restrict__ out, int B, int K) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= B) return;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s = fmaf(x[(size_t)row * K + k], w[k], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[row] = s + (bias ? bias[0] : 0.f);
}
// dx[b][k] = dy[b] * w[k]
__global__ void gemv_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, int B,
                                  int K) {
  const int n = B * K;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dx[i] = dy[i / K] * w[i % K];
}
// dw[k] += sum_b dy[b] * x[b][k] ; db[0] += sum_b dy[b]
__global__ void gemv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                                  float* __restrict__ db, int B, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < K) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s = fmaf(dy[b], x[(size_t)b * K + k], s);
    dw[k] += s;
  }
  if (k == 0 && db) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += dy[b];
    db[0] += s;
  }
}
int k_gemv_fwd(fg_ctx* c, const float* x, const float* w, const float* bias, float* out, int B, int K) {
  gemv_fwd_kernel<<<(B * 32 + 255) / 256, 256, 0, c->stream>>>(x, w, bias, out, B, K);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_gemv_dgrad(fg_ctx* c, const float* dy, const float* w, float* dx, int B, int K) {
  gemv_dgrad_kernel<<<grid_for((int64_t)B * K, 256), 256, 0, c->stream>>>(dy, w, dx, B, K);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_gemv_wgrad_add(fg_ctx* c, const float* x, const float* dy, float* dw, float* db, int B, int K) {
  gemv_wgrad_kernel<<<(K + 127) / 128, 128, 0, c->stream>>>(x, dy, dw, db, B, K);
  LAUNCH_CHECK(c);
  return FG_OK;
}

int k_adam(fg_ctx* c, float* p, const float* g, float* m, float* v, int64_t n, float beta1, float beta2, float eps,
           float l1_grad, float l2, float clampv, float grad_scale, const float* step_dev, const int* flag_dev,
           float step_host, float* g_out) {
  (void)g_out;
  adam_kernel<<<grid_for(n, 256, 132 * 8), 256, 0, c->stream>>>(p, const_cast<float*>(g), m, v, n, beta1, beta2, eps,
                                                               l1_grad, l2, clampv, grad_scale, step_dev, flag_dev,
                                                               step_host, 1, FG_OPT_ADAM, 0.f, nullptr);
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_optim_update(fg_ctx* c, int mode, float* p, float* g, float* m, float* v, int64_t n, float beta1, float beta2, float eps,
                   float mom, float l1_grad, float l2, float clampv, float grad_scale, const float* step_dev,
                   const int* flag_dev, const int* t_dev) {
  adam_kernel<<<grid_for(n, 256, 132 * 8), 256, 0, c->stream>>>(p, g, m, v, n, beta1, beta2, eps, l1_grad, l2, clampv, grad_scale,
                                                               step_dev, flag_dev, 0.f, 1, mode, mom, t_dev);
  LAUNCH_CHECK(c);
  return FG_OK;
}
