// 3x3 convolutions at the 3-channel image edge of both networks, 32 pixels wide, as HBM-shaped kernels:
//   "reduce"  many -> few channels   G.C3 forward 128 -> C (models.lua:73), D.C1 dgrad 64 -> C (models.lua:385)
//   "expand"  few -> many channels   D.C1 forward C -> 64,                   G.C3 dgrad C -> 128
// Neither is a dense contraction (N = 3 resp. K = 27): the work is one pass over the big activation tensor
// (134 MB at batch 256) with 27 FMAs per element, so FP32 issue and HBM are about equally loaded and the kernels are
// built to waste neither:
//   * the 9*C*4 (<= 144) weights a thread needs live in REGISTERS for the whole launch -- the round-1 kernels fetched
//     a weight from shared memory for every FMA and ran at 0.14 of the HBM roofline;
//   * reduce: the big tensor is staged by TMA (one bulk tensor copy per 4-row strip incl. halo, zero fill = padding)
//     into a double-buffered shared-memory tile, so ~100 KB per SM are in flight while the previous strip is
//     computed; a lane owns 4 (2) channels, 4 pixels are accumulated at a time and the 12 partial sums are combined
//     with a 16-value butterfly transpose-reduce (16 shuffles per 4 pixels instead of 60);
//   * expand: the small tensor (3 MB) is staged through shared memory with a register prefetch of the next strip,
//     a warp covers the 128 (2 x 64) output channels of one pixel, 4 per lane, and streams out one coalesced
//     float4 store per lane and pixel.
// All tensors NHWC fp32, stride 1, pad 1, W = 32, H a multiple of 8.  Other shapes keep the k_conv_small.cu kernels.
#include <cuda.h>

#include <algorithm>

#include "fg_internal.h"
#include "k_conv_tc.h"

namespace {
constexpr int kW = 32;  // image width these kernels are specialised for

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
// explicit shared-space loads: the tile pointer is derived from an integer-aligned base, which hides the address space
// from the compiler (it would emit generic LD, which goes through address translation and the long scoreboard)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------------------------------------
// reduce: out[p][n < NS] = bias[n] + sum_{t, c < 32*VEC} in[pix(p,t)][c] * Wp[t][n][c]
// unit = 4 output rows of one image = a TMA box of 6 rows x 34 columns x C channels (halo rows / columns zero-filled)
// ------------------------------------------------------------------------------------------------
constexpr int kRedRows = 4;
template <int VEC>
constexpr uint32_t red_tile_bytes() { return (kRedRows + 2) * (kW + 2) * 32 * VEC * 4; }

template <int NS, int VEC>
__global__ void __launch_bounds__(256, 1) conv_reduce_kernel(const __grid_constant__ CUtensorMap tmap, const float* __restrict__ Wp,
                                                             const float* __restrict__ bias, float* __restrict__ out, int H,
                                                             int nunits) {
  constexpr int C = 32 * VEC;
  constexpr int PX = NS == 1 ? 16 : 4;  // pixels accumulated before the cross-lane reduction (PX * NS <= 16)
  constexpr uint32_t kTile = red_tile_bytes<VEC>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + 2 * kTile);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int strips = H / kRedRows;
  if (threadIdx.x == 0) {
    mbar_init(full + 0, 1);
    mbar_init(full + 1, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int unit, int buf) {
    const int b = unit / strips, y0 = (unit - b * strips) * kRedRows;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic reads of this buffer (before the barrier) -> TMA write
    mbar_expect_tx(full + buf, kTile);
    tma_load_4d(smem + buf * kTile, &tmap, full + buf, 0, -1, y0 - 1, b);
  };
  if (threadIdx.x == 0 && (int)blockIdx.x < nunits) issue(blockIdx.x, 0);
  // the lane's 9 * NS * VEC weights, for the whole launch
  float w[9][NS][VEC];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int n = 0; n < NS; ++n)
#pragma unroll
      for (int j = 0; j < VEC; ++j) w[t][n][j] = Wp[(t * NS + n) * C + lane * VEC + j];
  float bv = 0.f;  // the lane that stores value k = i*NS + n adds bias[n]
  if (bias && (lane & 15) < PX * NS) bv = bias[(lane & 15) % NS];
  const int row = warp >> 1, xh = (warp & 1) * 16;  // this warp: tile row `row`, pixels [xh, xh + 16)
  int it = 0;
  for (int unit = blockIdx.x; unit < nunits; unit += gridDim.x, ++it) {
    const int buf = it & 1;
    if (threadIdx.x == 0 && unit + (int)gridDim.x < nunits) issue(unit + gridDim.x, buf ^ 1);
    mbar_wait(full + buf, (it >> 1) & 1);
    const uint32_t tile = smem_u32(smem + buf * kTile) + (uint32_t)lane * VEC * 4;  // this lane's channels of tile pixel 0
    const int b = unit / strips, y = (unit - b * strips) * kRedRows + row;
#pragma unroll 1
    for (int g = 0; g < 16 / PX; ++g) {
      const int x0 = xh + g * PX;
      float acc[PX][NS];
#pragma unroll
      for (int i = 0; i < PX; ++i)
#pragma unroll
        for (int n = 0; n < NS; ++n) acc[i][n] = 0.f;
      // column-major walk: tile column x0 + j (= image column x0 + j - 1) feeds pixels j-2 .. j.  The FMA order puts
      // the (up to 9) independent accumulators of a column innermost, so consecutive FMAs never depend on each other.
#pragma unroll
      for (int j = 0; j < PX + 2; ++j) {
        float v[3][VEC];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
          const uint32_t ad = tile + (uint32_t)(((row + dy) * (kW + 2) + x0 + j) * C) * 4;
          if (VEC == 4) {
            const float4 q = lds128(ad);
            v[dy][0] = q.x; v[dy][1 % VEC] = q.y; v[dy][2 % VEC] = q.z; v[dy][3 % VEC] = q.w;
          } else {
            const float2 q = lds64(ad);
            v[dy][0] = q.x; v[dy][1 % VEC] = q.y;
          }
        }
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
          for (int k = 0; k < VEC; ++k)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
              const int i = j - dx;  // output pixel whose tap column dx is this column
              if (i < 0 || i >= PX) continue;
#pragma unroll
              for (int n = 0; n < NS; ++n) acc[i][n] = fmaf(v[dy][k], w[dy * 3 + dx][n][k], acc[i][n]);
            }
      }
      // 16-value butterfly transpose-reduce inside each half-warp, then the two halves are added
      float r[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) r[k] = k < PX * NS ? acc[k / NS][k % NS] : 0.f;
#pragma unroll
      for (int sft = 8; sft >= 1; sft >>= 1) {
        const bool up = (lane & sft) != 0;
#pragma unroll
        for (int k = 0; k < sft; ++k) {
          const float send = up ? r[k] : r[k + sft], keep = up ? r[k + sft] : r[k];
          r[k] = keep + __shfl_xor_sync(0xffffffffu, send, sft);
        }
      }
      const float tot = r[0] + __shfl_xor_sync(0xffffffffu, r[0], 16);
      if (lane < PX * NS) out[((size_t)(b * H + y) * kW + x0) * NS + lane] = tot + bv;  // value k = lane: pixel k / NS, output k % NS
    }
    __syncthreads();  // every warp is done with this buffer before the next iteration's prefetch overwrites it
  }
}

// ------------------------------------------------------------------------------------------------
// expand: out[p][n < N] = bias[n] + sum_{t, c < CS} in[pix(p,t)][c] * Wp[t][n][c]
// unit = 8 output rows of one image; a warp produces one row
// ------------------------------------------------------------------------------------------------
constexpr int kExpRows = 8;
template <int CS, int N>
__global__ void __launch_bounds__(256, 1) conv_expand_kernel(const float* __restrict__ in, const float* __restrict__ Wp,
                                                             const float* __restrict__ bias, float* __restrict__ out, int H,
                                                             int nunits) {
  constexpr int RW = (kW + 2) * 4;                // floats per tile row: one float4 per pixel incl. the two halo pixels
  constexpr int ROWF = kW * CS;                   // floats per image row
  constexpr int NPF = ((kExpRows + 2) * ROWF + 255) / 256;  // prefetch registers per thread
  __shared__ __align__(16) float tile[2][(kExpRows + 2) * RW];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int strips = H / kExpRows;
  for (int i = threadIdx.x; i < 2 * (kExpRows + 2) * RW; i += 256) (&tile[0][0])[i] = 0.f;  // halo / pad lanes stay zero
  // this thread's 4 output channels and their 9 * CS * 4 weights
  const int n4 = (N == 128 ? lane : (lane & 15)) * 4;
  float w[9][CS][4];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < CS; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) w[t][c][j] = Wp[((size_t)t * N + n4 + j) * CS + c];
  float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias) b4 = make_float4(bias[n4], bias[n4 + 1], bias[n4 + 2], bias[n4 + 3]);
  float pf[NPF];
  auto prefetch = [&](int unit) {
    const int b = unit / strips, y0 = (unit - b * strips) * kExpRows;
#pragma unroll
    for (int i = 0; i < NPF; ++i) {
      const int idx = threadIdx.x + 256 * i;
      const int r = idx / ROWF, off = idx - r * ROWF, gy = y0 - 1 + r;
      pf[i] = (r < kExpRows + 2 && gy >= 0 && gy < H) ? in[((size_t)(b * H + gy) * kW) * CS + off] : 0.f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int i = 0; i < NPF; ++i) {
      const int idx = threadIdx.x + 256 * i;
      const int r = idx / ROWF, off = idx - r * ROWF;
      if (r < kExpRows + 2) tile[buf][r * RW + (off / CS + 1) * 4 + off % CS] = pf[i];
    }
  };
  __syncthreads();
  if ((int)blockIdx.x < nunits) {
    prefetch(blockIdx.x);
    stash(0);
  }
  __syncthreads();
  // a thread produces 2 neighbouring pixels per iteration (8 independent accumulator chains, the 4 tile columns they
  // need are loaded once); N = 64: the two half-warps take neighbouring pixel pairs
  constexpr int STEP = N == 128 ? 2 : 4;
  const int xoff = N == 128 ? 0 : 2 * (lane >> 4);
  int it = 0;
  for (int unit = blockIdx.x; unit < nunits; unit += gridDim.x, ++it) {
    const int buf = it & 1;
    const bool more = unit + (int)gridDim.x < nunits;
    if (more) prefetch(unit + gridDim.x);  // in flight while this strip is computed
    const int b = unit / strips, y = (unit - b * strips) * kExpRows + warp;
    const float4* t0 = reinterpret_cast<const float4*>(&tile[buf][warp * RW]);
    float* orow = out + ((size_t)(b * H + y) * kW) * N + n4;
#pragma unroll 1
    for (int xb = 0; xb < kW; xb += STEP) {
      const int x = xb + xoff;
      float4 a0 = b4, a1 = b4;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        float4 col[4];  // tile columns x .. x+3 = image columns x-1 .. x+2 (broadcast within the (half-)warp)
#pragma unroll
        for (int j = 0; j < 4; ++j) col[j] = t0[dy * (kW + 2) + x + j];
#pragma unroll
        for (int dx = 0; dx < 3; ++dx)
#pragma unroll
          for (int c = 0; c < CS; ++c) {
            const float v0 = c == 0 ? col[dx].x : (c == 1 ? col[dx].y : (c == 2 ? col[dx].z : col[dx].w));
            const float v1 = c == 0 ? col[dx + 1].x : (c == 1 ? col[dx + 1].y : (c == 2 ? col[dx + 1].z : col[dx + 1].w));
            const float* wp = w[dy * 3 + dx][c];
            a0.x = fmaf(v0, wp[0], a0.x); a1.x = fmaf(v1, wp[0], a1.x);
            a0.y = fmaf(v0, wp[1], a0.y); a1.y = fmaf(v1, wp[1], a1.y);
            a0.z = fmaf(v0, wp[2], a0.z); a1.z = fmaf(v1, wp[2], a1.z);
            a0.w = fmaf(v0, wp[3], a0.w); a1.w = fmaf(v1, wp[3], a1.w);
          }
      }
      *reinterpret_cast<float4*>(orow + (size_t)x * N) = a0;
      *reinterpret_cast<float4*>(orow + (size_t)(x + 1) * N) = a1;
    }
    if (more) stash(buf ^ 1);  // buf ^ 1 was last read in iteration it - 1 (barrier below)
    __syncthreads();
  }
}

template <int NS, int VEC>
int launch_reduce(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, const ConvGeom& g) {
  CUtensorMap tmap;
  FG_TRY(tc_encode_nhwc_box(&tmap, in, 32 * VEC, g.W, g.H, g.B, 32 * VEC, kW + 2, kRedRows + 2, 1));
  const int nunits = g.B * (g.H / kRedRows);
  const size_t smem = 2 * (size_t)red_tile_bytes<VEC>() + 64 + 128;
  static bool attr_done = false;
  if (!attr_done) {
    FG_CUDA(cudaFuncSetAttribute(conv_reduce_kernel<NS, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  note_conv(c, FG_KERNEL_EDGE_REDUCE, NS, VEC, 0, 1);
  conv_reduce_kernel<NS, VEC><<<std::min(nunits, c->sm_count), 256, smem, c->stream>>>(tmap, Wp, bias, out, g.H, nunits);
  LAUNCH_CHECK(c);
  return FG_OK;
}
template <int CS, int N>
int launch_expand(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, const ConvGeom& g) {
  const int nunits = g.B * (g.H / kExpRows);
  note_conv(c, FG_KERNEL_EDGE_EXPAND, CS, N, 0, 1);
  conv_expand_kernel<CS, N><<<std::min(nunits, c->sm_count), 256, 0, c->stream>>>(in, Wp, bias, out, g.H, nunits);
  LAUNCH_CHECK(c);
  return FG_OK;
}
}  // namespace

bool k_edge_eligible(const ConvGeom& g) {
  if (!(g.ups == 1 && g.k == 3 && g.W == kW && g.H % 8 == 0 && g.H >= 8)) return false;
  const bool reduce = (g.Cout == 1 || g.Cout == 3) && (g.Cin == 64 || g.Cin == 128);
  const bool expand = (g.Cin == 1 || g.Cin == 3 || g.Cin == 4) && (g.Cout == 64 || g.Cout == 128);
  return reduce || expand;
}

// in [B][H][32][Cin], Wp [9][Cout][Cin] (tap-major pack), bias [Cout] or nullptr, out [B][H][32][Cout]
int k_conv_edge(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, ConvGeom g) {
  if (g.Cout <= 3) {
    if (g.Cout == 3 && g.Cin == 128) return launch_reduce<3, 4>(c, in, Wp, bias, out, g);
    if (g.Cout == 3 && g.Cin == 64) return launch_reduce<3, 2>(c, in, Wp, bias, out, g);
    if (g.Cout == 1 && g.Cin == 128) return launch_reduce<1, 4>(c, in, Wp, bias, out, g);
    if (g.Cout == 1 && g.Cin == 64) return launch_reduce<1, 2>(c, in, Wp, bias, out, g);
  } else {
#define EXP(CS_)                                                                 \
  if (g.Cin == CS_) {                                                            \
    if (g.Cout == 128) return launch_expand<CS_, 128>(c, in, Wp, bias, out, g); \
    if (g.Cout == 64) return launch_expand<CS_, 64>(c, in, Wp, bias, out, g);   \
  }
    EXP(1) EXP(3) EXP(4)
#undef EXP
  }
  fg_set_error("k_conv_edge: unsupported shape %d -> %d", g.Cin, g.Cout);
  return FG_ERR_UNSUPPORTED;
}
