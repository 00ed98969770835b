// fp32 FFMA implicit-GEMM convolution ("first correct path"; also the path for the layers that are
// not dense contractions: D.C1 (K=27), G.C3 (N=3), the Linear layers, odd shapes from the L-op API).
//
//   forward / dgrad :  out[p][n] = bias[n] + sum_{t,c} in[pix(p,t)][c] * Wp[t][n][c]
//   wgrad           :  dWp[t][n][c] = sum_p dY[p][n] * in[pix(p,t)][c]
// with p = (b,y,x) an output pixel, t = (kh,kw) a filter tap and
//   pix(p,t) = (b, (y+kh-pad)/ups, (x+kw-pad)/ups)   (zero outside [0,H)x[0,W))
// ups=2 folds nn.SpatialUpSamplingNearest(2) into the addressing (models.lua:63,68) so the upsampled
// tensor is never materialised.  Everything NHWC so a warp's loads run along channels.
//
// Tiling: 256 threads as 16x16, each thread a TMxTN register tile; BK=16 staged through shared memory.
#include "fg_internal.h"

namespace {
constexpr int BK = 16;

template <int TM, int TN>
__global__ void __launch_bounds__(256) conv_simt_kernel(const float* __restrict__ in, const float* __restrict__ Wp,
                                                        const float* __restrict__ bias, float* __restrict__ out,
                                                        ConvGeom g) {
  constexpr int BM = 16 * TM, BN = 16 * TN;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int P = g.B * g.H * g.W;
  const int p0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int KK = g.k * g.k, pad = (g.k - 1) / 2;
  const int Hin = g.H / g.ups, Win = g.W / g.ups;
  const int sh = g.ups == 2 ? 1 : 0;

  // pixels this thread stages: m = ty + 16*i
  int pb[TM], py[TM], px[TM];
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int p = p0 + ty + 16 * i;
    if (p < P) {
      const int r = p % (g.H * g.W);
      pb[i] = p / (g.H * g.W);
      py[i] = r / g.W;
      px[i] = r % g.W;
    } else {
      pb[i] = 0;
      py[i] = -100000;
      px[i] = 0;
    }
  }
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int t = 0; t < KK; ++t) {
    const int kh = t / g.k, kw = t % g.k;
    const float* aptr[TM];
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int iy = py[i] + kh - pad, ix = px[i] + kw - pad;
      const bool ok = iy >= 0 && iy < g.H && ix >= 0 && ix < g.W;
      aptr[i] = ok ? in + ((int64_t)(pb[i] * Hin + (iy >> sh)) * Win + (ix >> sh)) * g.Cin : nullptr;
    }
    const float* wt = Wp + (int64_t)t * g.Cout * g.Cin;
    for (int c0 = 0; c0 < g.Cin; c0 += BK) {
      const int cc = c0 + tx;
      const bool cok = cc < g.Cin;
#pragma unroll
      for (int i = 0; i < TM; ++i) As[tx][ty + 16 * i] = (cok && aptr[i]) ? __ldg(aptr[i] + cc) : 0.f;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = n0 + ty + 16 * j;
        Bs[tx][ty + 16 * j] = (cok && n < g.Cout) ? __ldg(wt + (int64_t)n * g.Cin + cc) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[TM], b[TN];
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int p = p0 + ty * TM + i;
    if (p >= P) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n < g.Cout) out[(int64_t)p * g.Cout + n] = acc[i][j] + (bias ? bias[n] : 0.f);
    }
  }
}

// Same tiling for a TINY input-channel count (D.C1: Cin = 3, G.C3 dgrad: 3 "input" channels): the
// contraction index is flattened to k = t*Cin + c so that K = k*k*Cin = 27 fills two BK=16 steps instead
// of padding every tap to 16.
template <int TM, int TN>
__global__ void __launch_bounds__(256) conv_simt_flatk_kernel(const float* __restrict__ in, const float* __restrict__ Wp,
                                                              const float* __restrict__ bias, float* __restrict__ out,
                                                              ConvGeom g) {
  constexpr int BM = 16 * TM, BN = 16 * TN;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int P = g.B * g.H * g.W;
  const int p0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int KK = g.k * g.k, pad = (g.k - 1) / 2, Ktot = KK * g.Cin;
  int pb[TM], py[TM], px[TM];
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int p = p0 + ty + 16 * i;
    if (p < P) {
      const int r = p % (g.H * g.W);
      pb[i] = p / (g.H * g.W);
      py[i] = r / g.W;
      px[i] = r % g.W;
    } else {
      pb[i] = 0;
      py[i] = -100000;
      px[i] = 0;
    }
  }
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < Ktot; k0 += BK) {
    const int kk = k0 + tx;
    const bool kok = kk < Ktot;
    const int t = kok ? kk / g.Cin : 0, cc = kok ? kk - t * g.Cin : 0;
    const int kh = t / g.k, kw = t - kh * g.k;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int iy = py[i] + kh - pad, ix = px[i] + kw - pad;
      const bool ok = kok && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W;
      As[tx][ty + 16 * i] = ok ? __ldg(in + ((int64_t)(pb[i] * g.H + iy) * g.W + ix) * g.Cin + cc) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + ty + 16 * j;
      Bs[tx][ty + 16 * j] = (kok && n < g.Cout) ? __ldg(Wp + ((int64_t)t * g.Cout + n) * g.Cin + cc) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < BK; ++q) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[q][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[q][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int p = p0 + ty * TM + i;
    if (p >= P) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n < g.Cout) out[(int64_t)p * g.Cout + n] = acc[i][j] + (bias ? bias[n] : 0.f);
    }
  }
}

// grid: x = n-tile, y = c-tile, z = tap * splits + split
template <int TM, int TN>
__global__ void __launch_bounds__(256) wgrad_simt_kernel(const float* __restrict__ in, const float* __restrict__ dY,
                                                         float* __restrict__ dWp, ConvGeom g, int splits,
                                                         int pix_per_split) {
  constexpr int BM = 16 * TM, BN = 16 * TN;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int P = g.B * g.H * g.W;
  const int n0 = blockIdx.x * BM, c0 = blockIdx.y * BN;
  const int t = blockIdx.z / splits, split = blockIdx.z % splits;
  const int kh = t / g.k, kw = t % g.k, pad = (g.k - 1) / 2;
  const int Hin = g.H / g.ups, Win = g.W / g.ups;
  const int sh = g.ups == 2 ? 1 : 0;
  const int pbeg = split * pix_per_split, pend = min(P, pbeg + pix_per_split);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int pk = pbeg; pk < pend; pk += BK) {
    // A: dY[pk+kk][n0+m], m fastest across threads
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int e = tid + i * 256;
      const int m = e % BM, kk = e / BM;
      const int p = pk + kk, n = n0 + m;
      As[kk][m] = (p < pend && n < g.Cout) ? __ldg(dY + (int64_t)p * g.Cout + n) : 0.f;
    }
    // B: in[pix(pk+kk,t)][c0+j], j fastest
#pragma unroll
    for (int i = 0; i < TN; ++i) {
      const int e = tid + i * 256;
      const int j = e % BN, kk = e / BN;
      const int p = pk + kk, cc = c0 + j;
      float v = 0.f;
      if (p < pend && cc < g.Cin) {
        const int r = p % (g.H * g.W), b = p / (g.H * g.W);
        const int iy = r / g.W + kh - pad, ix = r % g.W + kw - pad;
        if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
          v = __ldg(in + ((int64_t)(b * Hin + (iy >> sh)) * Win + (ix >> sh)) * g.Cin + cc);
      }
      Bs[kk][j] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int n = n0 + ty * TM + i;
    if (n >= g.Cout) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int cc = c0 + tx * TN + j;
      if (cc < g.Cin) {
        // splits > 1: dWp holds one partial per split (k_splitk_reduce adds them in split order)
        dWp[(int64_t)split * g.k * g.k * g.Cout * g.Cin + ((int64_t)t * g.Cout + n) * g.Cin + cc] = acc[i][j];
      }
    }
  }
}
}  // namespace

int k_conv_simt(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, ConvGeom g) {
  const int P = g.B * g.H * g.W;
  const int tn = g.Cout > 64 ? 8 : (g.Cout > 16 ? 4 : 1);
  if (g.Cin < 16 && g.ups == 1 && g.k > 1) {
    note_conv(c, FG_KERNEL_SIMT_FLATK, 8, tn, 0, 1);
    if (g.Cout > 64) {
      dim3 grid((P + 127) / 128, (g.Cout + 127) / 128);
      conv_simt_flatk_kernel<8, 8><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g);
    } else if (g.Cout > 16) {
      dim3 grid((P + 127) / 128, (g.Cout + 63) / 64);
      conv_simt_flatk_kernel<8, 4><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g);
    } else {
      dim3 grid((P + 127) / 128, (g.Cout + 15) / 16);
      conv_simt_flatk_kernel<8, 1><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g);
    }
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  note_conv(c, FG_KERNEL_SIMT, 8, tn, 0, 1);
  if (g.Cout > 64) {
    dim3 grid((P + 127) / 128, (g.Cout + 127) / 128);
    conv_simt_kernel<8, 8><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g);
  } else if (g.Cout > 16) {
    dim3 grid((P + 127) / 128, (g.Cout + 63) / 64);
    conv_simt_kernel<8, 4><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g);
  } else {
    dim3 grid((P + 127) / 128, (g.Cout + 15) / 16);
    conv_simt_kernel<8, 1><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g);
  }
  LAUNCH_CHECK(c);
  return FG_OK;
}

int k_wgrad_simt(fg_ctx* c, const float* in, const float* dY, float* dWp, ConvGeom g) {
  const int P = g.B * g.H * g.W;
  const int KK = g.k * g.k;
  int tm, tn;  // tile = (16*tm over Cout) x (16*tn over Cin)
  if (g.Cout > 64) tm = 8; else if (g.Cout > 16) tm = 4; else tm = 1;
  if (g.Cin > 64) tn = 8; else if (g.Cin > 16) tn = 4; else tn = 1;
  const int gx = (g.Cout + 16 * tm - 1) / (16 * tm), gy = (g.Cin + 16 * tn - 1) / (16 * tn);
  const int base = gx * gy * KK;
  int splits = (c->sm_count * 4 + base - 1) / base;
  const int max_splits = (P + 255) / 256;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  const int64_t size = (int64_t)KK * g.Cout * g.Cin;
  while (splits > 1 && splits * size > (int64_t)c->splitk_ws_elems) --splits;  // partials must fit the split-K workspace
  int pps = (P + splits - 1) / splits;
  pps = (pps + BK - 1) / BK * BK;
  splits = (P + pps - 1) / pps;
  float* dst = splits > 1 ? c->splitk_ws : dWp;
  dim3 grid(gx, gy, KK * splits);
  note_conv(c, FG_KERNEL_WGRAD_SIMT, tm, tn, 0, splits);
#define WG(TM_, TN_) wgrad_simt_kernel<TM_, TN_><<<grid, 256, 0, c->stream>>>(in, dY, dst, g, splits, pps)
  if (tm == 8 && tn == 8) WG(8, 8);
  else if (tm == 8 && tn == 4) WG(8, 4);
  else if (tm == 8 && tn == 1) WG(8, 1);
  else if (tm == 4 && tn == 8) WG(4, 8);
  else if (tm == 4 && tn == 4) WG(4, 4);
  else if (tm == 4 && tn == 1) WG(4, 1);
  else if (tm == 1 && tn == 8) WG(1, 8);
  else if (tm == 1 && tn == 4) WG(1, 4);
  else WG(1, 1);
#undef WG
  LAUNCH_CHECK(c);
  return splits > 1 ? k_splitk_reduce(c, c->splitk_ws, splits, size, dWp) : FG_OK;
}
