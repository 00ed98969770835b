// Convolutions with a tiny channel count on one side (the 3-channel image end of both networks):
//   G.C3  128 -> C(1|3) 3x3   (models.lua:73)      forward = small-N, wgrad = small/big
//   D.C1  C(1|3) -> 64  3x3   (models.lua:385)     dgrad   = small-N, wgrad = small/big
// (the small-K directions, D.C1 forward / G.C3 dgrad, run on the flat-K SIMT tiles of k_conv_simt.cu).
// These are NOT dense contractions (N = 3 / K = 27): they are bound by the traffic of the big activation
// tensor (SURVEY.md 8a rows G12 / D1), so they get bandwidth-shaped kernels instead of GEMM tiles: coalesced
// channel-fastest accesses, the small operand broadcast through shared memory, warp-shuffle reductions.
// All tensors NHWC fp32; 3x3, stride 1, pad 1 (fully unrolled taps so the 9 loads are in flight together).
#include "fg_internal.h"

namespace {
constexpr int kMaxSmallW = 36 * 128;  // 9 * Cs * Cb floats of weights in shared memory

// ---- small output: out[p][n<NS] = bias[n] + sum_{t,c} in[pix(p,t)][c] * Wp[t][n][c] ---------------------
// one warp per pixel, lane owns VEC consecutive channels (C = 32*VEC), warp-shuffle reduction of NS sums
template <int NS, int VEC>
__global__ void __launch_bounds__(256) conv_smalln_kernel(const float* __restrict__ in, const float* __restrict__ Wp,
                                                          const float* __restrict__ bias, float* __restrict__ out, int B,
                                                          int H, int W) {
  constexpr int C = 32 * VEC;
  __shared__ __align__(16) float ws[9 * NS * C];  // [t][n][c]
  for (int i = threadIdx.x; i < 9 * NS * C; i += blockDim.x) ws[i] = Wp[i];
  __syncthreads();
  // A warp walks a run of RL = 8 pixels of one image row with a 3-column sliding window in registers:
  // 3 new vector loads per pixel instead of 9 (the 3x3 neighbourhoods of adjacent pixels overlap 6/9).
  constexpr int RL = 8;
  const int lane = threadIdx.x & 31;
  const uint32_t runs_per_row = (uint32_t)W / RL;
  const uint32_t nruns = (uint32_t)B * H * runs_per_row;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t run = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; run < nruns; run += warps) {
    const int x0 = (int)(run % runs_per_row) * RL;
    const uint32_t row = run / runs_per_row;  // b*H + y
    const int y = (int)(row % (uint32_t)H);
    const float* rowbase = in + (size_t)row * W * C + lane * VEC;
    float col[3][3][VEC];  // [column slot][dy][vec]
    auto load_col = [&](int slot, int xx) {
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const bool ok = (unsigned)(y + dy - 1) < (unsigned)H && (unsigned)xx < (unsigned)W;
        const float* ip = rowbase + ((dy - 1) * W + xx) * C;
        if (VEC == 4) {
          const float4 q = ok ? *reinterpret_cast<const float4*>(ip) : make_float4(0.f, 0.f, 0.f, 0.f);
          col[slot][dy][0] = q.x; col[slot][dy][1 % VEC] = q.y; col[slot][dy][2 % VEC] = q.z; col[slot][dy][3 % VEC] = q.w;
        } else if (VEC == 2) {
          const float2 q = ok ? *reinterpret_cast<const float2*>(ip) : make_float2(0.f, 0.f);
          col[slot][dy][0] = q.x; col[slot][dy][1 % VEC] = q.y;
        } else {
          col[slot][dy][0] = ok ? ip[0] : 0.f;
        }
      }
    };
    load_col(0, x0 - 1);
    load_col(1, x0);
#pragma unroll
    for (int i = 0; i < RL; ++i) {
      load_col((i + 2) % 3, x0 + i + 1);
      float acc[NS];
#pragma unroll
      for (int n = 0; n < NS; ++n) acc[n] = 0.f;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const int t = dy * 3 + dx, slot = (i + dx) % 3;
#pragma unroll
          for (int n = 0; n < NS; ++n) {
            const float* wp = ws + (t * NS + n) * C + lane * VEC;
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[n] = fmaf(col[slot][dy][j], wp[j], acc[n]);
          }
        }
#pragma unroll
      for (int n = 0; n < NS; ++n) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
      }
      if (lane == 0) {
        float* op = out + ((size_t)row * W + x0 + i) * NS;
#pragma unroll
        for (int n = 0; n < NS; ++n) op[n] = acc[n] + (bias ? bias[n] : 0.f);
      }
    }
  }
}

// ---- small contraction: out[p][n] = bias[n] + sum_{t,c<CS} in[pix(p,t)][c] * Wp[t][n][c]  (D.C1 fwd, G.C3 dgrad)
// one thread per (pixel, 4 consecutive output channels): the 9*CS inputs of a pixel are broadcast loads shared by
// the N/4 threads of that pixel, the weights come from shared memory as float4, the output is one float4 store.
template <int CS>
__global__ void __launch_bounds__(256) conv_smallk4_kernel(const float* __restrict__ in, const float* __restrict__ Wp,
                                                           const float* __restrict__ bias, float* __restrict__ out, int B,
                                                           int H, int W, int N) {
  __shared__ __align__(16) float ws[9 * CS * 128];  // [t][c][n]
  for (int i = threadIdx.x; i < 9 * CS * N; i += blockDim.x) {
    const int n = i % N, c = (i / N) % CS, t = i / (N * CS);
    ws[i] = Wp[((size_t)t * N + n) * CS + c];
  }
  __syncthreads();
  const uint32_t N4 = (uint32_t)N >> 2;
  const uint32_t total = (uint32_t)B * H * W * N4;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t n4 = i % N4, p = i / N4;
    const int x = (int)(p % (uint32_t)W), y = (int)((p / (uint32_t)W) % (uint32_t)H);
    float4 acc = bias ? make_float4(bias[n4 * 4], bias[n4 * 4 + 1], bias[n4 * 4 + 2], bias[n4 * 4 + 3])
                      : make_float4(0.f, 0.f, 0.f, 0.f);
    const float* base = in + (size_t)p * CS;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int dy = t / 3 - 1, dx = t % 3 - 1;
      if ((unsigned)(y + dy) >= (unsigned)H || (unsigned)(x + dx) >= (unsigned)W) continue;
      const float* ip = base + (dy * W + dx) * CS;
#pragma unroll
      for (int c = 0; c < CS; ++c) {
        const float v = __ldg(ip + c);
        const float4 w = *reinterpret_cast<const float4*>(ws + (t * CS + c) * N + n4 * 4);
        acc.x = fmaf(v, w.x, acc.x);
        acc.y = fmaf(v, w.y, acc.y);
        acc.z = fmaf(v, w.z, acc.z);
        acc.w = fmaf(v, w.w, acc.w);
      }
    }
    *reinterpret_cast<float4*>(out + (size_t)i * 4) = acc;
  }
}

// ---- weight gradient with one small and one big side ----------------------------------------------------
//   G.C3:  dW[n<Cs][c][t] = sum_p dY[p][n] * X[p+off_t][c]      big = X  (Cb = 128), small = dY, sign = -1
//   D.C1:  dW[n][c<Cs][t] = sum_p dY[p][n] * X[p+off_t][c]      big = dY (Cb = 64),  small = X,  sign = +1
// One thread per big channel walks XS pixels of an image row with a 3x3 sliding window of the small tensor
// in registers (staged per row through shared memory as float4): 3 broadcast LDS.128 + 1 coalesced LDG per
// 9*Cs FMAs, x loop unrolled so the big-tensor loads are batched.  Blocks write per-block partial sums; a
// second tiny kernel reduces them in a fixed order (deterministic, no atomics).
//   window index idx = r*3 + c holds small[y+r-1][x+c-1];  tap t = idx (sign +1) or 8 - idx (sign -1)
template <int CS, int XS>
__global__ void __launch_bounds__(128) wgrad_smallbig_kernel(const float* __restrict__ big, const float* __restrict__ small,
                                                             float* __restrict__ part, int B, int H, int W, int Cb,
                                                             int rows_per_block) {
  __shared__ float4 sm[3][68];
  const int lanes = 128 / Cb;
  const int cb = threadIdx.x % Cb, pl = threadIdx.x / Cb;
  const int x_begin = pl * XS;
  float acc[9][CS];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < CS; ++c) acc[t][c] = 0.f;
  const int BH = B * H;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(BH, r0 + rows_per_block);
  for (int r = r0; r < r1; ++r) {
    const int b = r / H, y = r - b * H;
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * (W + 2); i += 128) {
      const int rr = i / (W + 2), cc = i - rr * (W + 2);
      const int yy = y + rr - 1, xx = cc - 1;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
        const float* sp = small + (((size_t)b * H + yy) * W + xx) * CS;
        v.x = sp[0];
        if (CS > 1) v.y = sp[1 % CS];
        if (CS > 2) v.z = sp[2 % CS];
        if (CS > 3) v.w = sp[3 % CS];
      }
      sm[rr][cc] = v;
    }
    __syncthreads();
    const float* bp = big + ((size_t)r * W + x_begin) * Cb + cb;
    float bv[XS];
#pragma unroll
    for (int i = 0; i < XS; ++i) bv[i] = bp[(size_t)i * Cb];
    float4 w0[3], w1[3], w2[3];
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) {
      w0[rr] = sm[rr][x_begin];
      w1[rr] = sm[rr][x_begin + 1];
    }
#pragma unroll
    for (int i = 0; i < XS; ++i) {
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) {
        w2[rr] = sm[rr][x_begin + i + 2];
        const float4 q[3] = {w0[rr], w1[rr], w2[rr]};
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
          acc[rr * 3 + cc][0] = fmaf(bv[i], q[cc].x, acc[rr * 3 + cc][0]);
          if (CS > 1) acc[rr * 3 + cc][1 % CS] = fmaf(bv[i], q[cc].y, acc[rr * 3 + cc][1 % CS]);
          if (CS > 2) acc[rr * 3 + cc][2 % CS] = fmaf(bv[i], q[cc].z, acc[rr * 3 + cc][2 % CS]);
          if (CS > 3) acc[rr * 3 + cc][3 % CS] = fmaf(bv[i], q[cc].w, acc[rr * 3 + cc][3 % CS]);
        }
        w0[rr] = w1[rr];
        w1[rr] = w2[rr];
      }
    }
  }
  float* dst = part + ((size_t)blockIdx.x * lanes + pl) * (9 * CS * Cb);
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < CS; ++c) dst[(t * CS + c) * Cb + cb] = acc[t][c];
}
// out[slice] = sum over a slice of the partial rows, mapped to the packed [t][n][c] layout (out holds gridDim.y slices
// of `total`; k_splitk_reduce adds them in slice order).  grid.y slices the partial rows so the loads are not one long
// dependent chain per thread.
__global__ void wgrad_small_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int nparts, int CS, int Cb,
                                          int sign, int transposed) {
  const int total = 9 * CS * Cb;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= total) return;
  const int per = (nparts + gridDim.y - 1) / gridDim.y;
  const int i0 = blockIdx.y * per, i1 = min(nparts, i0 + per);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int i = i0;
  for (; i + 3 < i1; i += 4) {
    s0 += part[(size_t)i * total + j];
    s1 += part[(size_t)(i + 1) * total + j];
    s2 += part[(size_t)(i + 2) * total + j];
    s3 += part[(size_t)(i + 3) * total + j];
  }
  for (; i < i1; ++i) s0 += part[(size_t)i * total + j];
  const int idx = j / (CS * Cb), cs = (j / Cb) % CS, cb = j % Cb;
  const int t = sign > 0 ? idx : 8 - idx;
  out[(size_t)blockIdx.y * total + (transposed ? ((size_t)t * Cb + cb) * CS + cs : ((size_t)t * CS + cs) * Cb + cb)] =
      (s0 + s1) + (s2 + s3);
}
}  // namespace

bool k_small_eligible(const ConvGeom& g) {
  const int cs = g.Cin < g.Cout ? g.Cin : g.Cout, cb = g.Cin < g.Cout ? g.Cout : g.Cin;
  if (!(g.ups == 1 && g.k == 3 && cs >= 1 && cs <= 4 && (cb == 32 || cb == 64 || cb == 128))) return false;
  const int xs = g.W / (128 / cb);
  return g.W <= 64 && g.W % (128 / cb) == 0 && (xs == 8 || xs == 16 || xs == 32) &&
         (int64_t)g.B * g.H * g.W * cb < ((int64_t)1 << 31);
}

// forward-type conv: small OUTPUT channel count (G.C3 fwd, D.C1 dgrad) or small INPUT channel count
// (D.C1 fwd, G.C3 dgrad), both with the tap-major pack [t][n][c]
int k_conv_small(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, ConvGeom g) {
  const int64_t P = (int64_t)g.B * g.H * g.W;
  if (g.Cin <= 4) {
    const int64_t total = P * (g.Cout / 4);
    int grid = (int)std::min<int64_t>((total + 255) / 256, c->sm_count * 16);
    switch (g.Cin) {
      case 1: conv_smallk4_kernel<1><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g.B, g.H, g.W, g.Cout); break;
      case 2: conv_smallk4_kernel<2><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g.B, g.H, g.W, g.Cout); break;
      case 3: conv_smallk4_kernel<3><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g.B, g.H, g.W, g.Cout); break;
      default: conv_smallk4_kernel<4><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g.B, g.H, g.W, g.Cout); break;
    }
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  if (g.Cout > 4 || 9 * g.Cout * g.Cin > kMaxSmallW) {
    fg_set_error("k_conv_small: expects Cout <= 4");
    return FG_ERR_UNSUPPORTED;
  }
  if (g.W % 8) {
    fg_set_error("k_conv_small: W must be a multiple of 8");
    return FG_ERR_UNSUPPORTED;
  }
  int grid = (int)std::min<int64_t>((P / 8 * 32 + 255) / 256, c->sm_count * 8);  // one warp per run of 8 pixels
#define SN(NS_, VEC_) conv_smalln_kernel<NS_, VEC_><<<grid, 256, 0, c->stream>>>(in, Wp, bias, out, g.B, g.H, g.W)
  const int vec = g.Cin / 32;
  if (vec == 4) {
    if (g.Cout == 1) SN(1, 4); else if (g.Cout == 2) SN(2, 4); else if (g.Cout == 3) SN(3, 4); else SN(4, 4);
  } else if (vec == 2) {
    if (g.Cout == 1) SN(1, 2); else if (g.Cout == 2) SN(2, 2); else if (g.Cout == 3) SN(3, 2); else SN(4, 2);
  } else {
    if (g.Cout == 1) SN(1, 1); else if (g.Cout == 2) SN(2, 1); else if (g.Cout == 3) SN(3, 1); else SN(4, 1);
  }
#undef SN
  LAUNCH_CHECK(c);
  return FG_OK;
}

// dWp[t][n][c] (overwritten) = sum_p dY[p][n] * X[pix(p,t)][c]   with min(Cin,Cout) <= 4
int k_wgrad_small(fg_ctx* c, const float* in, const float* dY, float* dWp, ConvGeom g) {
  const bool small_out = g.Cout <= 4;  // G.C3: small = dY, big = X (window read mirrored: sign -1)
  const float* big = small_out ? in : dY;
  const float* small = small_out ? dY : in;
  const int Cb = small_out ? g.Cin : g.Cout, Cs = small_out ? g.Cout : g.Cin;
  const int lanes = 128 / Cb, xs = g.W / lanes;
  const int BH = g.B * g.H;
  int rpb = 8;
  int nblocks = (BH + rpb - 1) / rpb;
  while (nblocks * lanes > kSmallMaxParts) {
    rpb *= 2;
    nblocks = (BH + rpb - 1) / rpb;
  }
  const int sign = small_out ? -1 : 1, transposed = small_out ? 0 : 1;
#define WG(CS_, XS_) \
  wgrad_smallbig_kernel<CS_, XS_><<<nblocks, 128, 0, c->stream>>>(big, small, c->small_ws, g.B, g.H, g.W, Cb, rpb)
#define WGX(CS_)                 \
  do {                           \
    if (xs == 8) WG(CS_, 8);     \
    else if (xs == 16) WG(CS_, 16); \
    else WG(CS_, 32);            \
  } while (0)
  switch (Cs) {
    case 1: WGX(1); break;
    case 2: WGX(2); break;
    case 3: WGX(3); break;
    default: WGX(4); break;
  }
#undef WGX
#undef WG
  LAUNCH_CHECK(c);
  const int total = 9 * Cs * Cb;
  constexpr int kSlices = 32;
  wgrad_small_reduce_kernel<<<dim3((total + 127) / 128, kSlices), 128, 0, c->stream>>>(c->small_ws, c->splitk_ws, nblocks * lanes,
                                                                                     Cs, Cb, sign, transposed);
  LAUNCH_CHECK(c);
  return k_splitk_reduce(c, c->splitk_ws, kSlices, total, dWp);
}
