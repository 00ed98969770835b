// Device kernels of the wgmma convolution path (included by k_conv_tc.cu after the PTX wrappers).
//
// 3xTF32: x = x_hi + x_lo (TF32 split), product = a_hi*b_hi + a_hi*b_lo + a_lo*b_hi, three wgmmas of N = BN per K
// slice into two register accumulators: main = a_hi*b_hi, cross = a_hi*b_lo + a_lo*b_hi.
//
// CTA = 384 threads: warpgroups 0 and 1 each own 64 of the 128 accumulator rows (issue the wgmmas and run the
// epilogue), warpgroup 2 is the producer (one lane issues the TMA loads).  The producer warpgroup hands its registers
// to the consumers (setmaxnreg): a BN = 128 consumer holds 128 wgmma accumulators plus 64 promoted sums.  Stages of
// {A_hi, A_lo, B_hi, B_lo} flow through full / empty mbarrier rings; a consumer keeps one wgmma group in flight and
// releases a stage once the group that read it has completed.
//
// Numerics: the tensor core's own accumulation is not round-to-nearest, so a long K loop into ONE accumulator drifts
// (growing ~linearly with K).  The kernels therefore accumulate only `chunk` K-blocks in the wgmma accumulators and then
// "promote" them into fp32 registers with round-to-nearest adds.
#pragma once

constexpr int kConsumerThreads = 256;  // two consumer warpgroups
constexpr int kTcThreads = kConsumerThreads + 128;

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }
// register budget of a 384-thread CTA: 2 x 128 x 232 + 128 x 40 <= 64 K
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory"); }

// one wgmma D[64 x N] (+)= A * B; MN = the operands are MN-major (only the FP16 split has a transposed form)
template <int N, bool F16, bool MN>
__device__ __forceinline__ void wgmma_op(float* d, uint64_t a, uint64_t b, int scale_d) {
  if constexpr (F16) {
    constexpr int T = MN ? 1 : 0;
    if constexpr (N == 64) wgmma_f16_n64<T, T>(d, a, b, scale_d);
    else if constexpr (N == 128) wgmma_f16_n128<T, T>(d, a, b, scale_d);
    else wgmma_f16_n256<T, T>(d, a, b, scale_d);
  } else {
    static_assert(!MN, "tf32 wgmma operands are K-major");
    if constexpr (N == 64) wgmma_tf32_n64(d, a, b, scale_d);
    else if constexpr (N == 128) wgmma_tf32_n128(d, a, b, scale_d);
    else wgmma_tf32_n256(d, a, b, scale_d);
  }
}

// the 12 wgmmas of one 128-byte K block (4 K slices), committed as one group.  kstep: descriptor advance per K slice
// (16-byte units).  zero: the block starts a new accumulation run.
template <int BN, bool F16, bool MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                           uint64_t kstep, bool zero) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint64_t ko = (uint64_t)k * kstep;
    const int sd = (zero && k == 0) ? 0 : 1;
    wgmma_op<BN, F16, MN>(acc, a_hi + ko, b_hi + ko, sd);               // main  (+)= a_hi x b_hi
    wgmma_op<BN, F16, MN>(acc + BN / 2, a_hi + ko, b_lo + ko, sd);      // cross (+)= a_hi x b_lo
    wgmma_op<BN, F16, MN>(acc + BN / 2, a_lo + ko, b_hi + ko, 1);       // cross  += a_lo x b_hi
  }
  wgmma_commit();
}

// out[0..BN/2) += main half + cross half of the wgmma accumulators.
// F16 (3xFP16 split operands, see k_conv_tc.cu): the lo halves are stored scaled by 2^11, so the cross half carries 2^11
template <int BN, bool F16>
__device__ __forceinline__ void promote(float (&out)[BN / 2], const float (&acc)[BN]) {
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) out[i] += F16 ? fmaf(acc[BN / 2 + i], 0x1p-11f, acc[i]) : acc[i] + acc[BN / 2 + i];
}

struct FwdTile {
  int ph, b0, y0, x0, n0;
};
template <int BN>
__device__ __forceinline__ FwdTile fwd_decode(const TcFwdParams& p, int tile) {
  const int ntn = p.Cout / BN;
  FwdTile t;
  const int mt = tile / ntn;
  t.n0 = (tile - mt * ntn) * BN;  // n fastest: CTAs running together share the activation tile in L2
  int r = mt / p.nphase;  // the 4 output phases of one pixel tile run back to back: they share the input boxes in L2
  t.ph = mt - r * p.nphase;
  if (p.bb == 1) {
    const int per_img = p.tiles_x * p.tiles_y;
    t.b0 = r / per_img;
    r -= t.b0 * per_img;
    t.y0 = (r / p.tiles_x) * p.bh;
    t.x0 = (r % p.tiles_x) * p.bw;
  } else {
    t.b0 = r * p.bb;
    t.y0 = 0;
    t.x0 = 0;
  }
  return t;
}

// ------------------------------------------------------------------------------------------------
// tapconv: forward / dgrad.  Persistent: CTA i handles tiles i, i+gridDim.x, ...
// The producer and consumer sides of one tile are device functions, shared with bwd_pair_tc_kernel; `kbg` is the
// running K-block counter of the CTA's stage ring (stage kbg % kStages, phase kbg / kStages), carried across tiles.
// ------------------------------------------------------------------------------------------------
template <int BN>
constexpr uint32_t fwd_stage_bytes() { return 2 * kABytes + 2 * BN * 128; }  // {a_hi, a_lo, b_hi, b_lo}

template <int BN, bool F16>
__device__ __forceinline__ void tapconv_load_tile(const TcFwdParams& p, int tile, uint8_t* smem, uint64_t* full,
                                                  uint64_t* empty, uint32_t& kbg) {
  constexpr uint32_t kBBytes = BN * 128;
  constexpr uint32_t kStageBytes = fwd_stage_bytes<BN>();
  constexpr int kKE = F16 ? 64 : 32;  // K elements of one 128-byte K block
  const int nkb = p.ntaps * p.kpt;
  const FwdTile t = fwd_decode<BN>(p, tile);
  for (int kb = 0; kb < nkb; ++kb, ++kbg) {
    const uint32_t s = kbg % kStages, it = kbg / kStages;
    if (it > 0) mbar_wait_spin(empty + s, (it - 1) & 1);
    const int tap = kb / p.kpt, c0 = (kb - tap * p.kpt) * kKE;
    const int ti = t.ph * p.ntaps + tap;
    const int am = p.amap[ti];
    uint8_t* st = smem + s * kStageBytes;
    mbar_expect_tx(full + s, kStageBytes);
    tma_load_4d(st, &p.a_hi[am], full + s, c0, t.x0 + p.dx[ti], t.y0 + p.dy[ti], t.b0);
    tma_load_4d(st + kABytes, &p.a_lo[am], full + s, c0, t.x0 + p.dx[ti], t.y0 + p.dy[ti], t.b0);
    const int wrow = p.widx[ti] * p.Cout + t.n0;
    tma_load_2d(st + 2 * kABytes, &p.b_hi, full + s, c0, wrow);
    tma_load_2d(st + 2 * kABytes + kBBytes, &p.b_lo, full + s, c0, wrow);
  }
}

// consumers: warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) == tile pixels
template <int BN, bool F16>
__device__ __forceinline__ void tapconv_mma_tile(const TcFwdParams& p, int tile, uint8_t* smem, uint64_t* full,
                                                 uint64_t* empty, float* stat_sm, uint32_t& kbg) {
  constexpr uint32_t kBBytes = BN * 128;
  constexpr uint32_t kStageBytes = fwd_stage_bytes<BN>();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, g = lane >> 2, tq = lane & 3;
  const uint32_t aoff = (uint32_t)wg * 64 * 128;  // the warpgroup's 64 rows of the A tile
  const int nkb = p.ntaps * p.kpt;
  const int kChunk = p.chunk;
  const int nchunks = (nkb + kChunk - 1) / kChunk;
  int rowpix[2];
  for (int h = 0; h < 2; ++h) rowpix[h] = wg * 64 + (warp & 3) * 16 + g + 8 * h;
  float acc[BN];
  const FwdTile t = fwd_decode<BN>(p, tile);
  float o[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) o[i] = 0.f;
  for (int ch = 0; ch < nchunks; ++ch) {
    const int nk = min(kChunk, nkb - ch * kChunk);
    int prev = -1;
    for (int j = 0; j < nk; ++j, ++kbg) {
      const uint32_t s = kbg % kStages, it = kbg / kStages;
      const uint32_t sa = smem_u32(smem + s * kStageBytes);
      mbar_wait(full + s, it & 1);
      mma_kblock<BN, F16, false>(acc, make_desc(sa + aoff, 16, 1024), make_desc(sa + kABytes + aoff, 16, 1024),
                                 make_desc(sa + 2 * kABytes, 16, 1024), make_desc(sa + 2 * kABytes + kBBytes, 16, 1024),
                                 2, j == 0);  // +32 bytes per K slice
      wgmma_wait<1>();  // the previous block's group has read its stage
      if (prev >= 0 && lane == 0) mbar_arrive(empty + prev);
      prev = (int)s;
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(empty + prev);
    promote<BN, F16>(o, acc);
  }
  if (p.oscale) {  // operands stored scaled by powers of two (FP16 split): undo it
    const float os = *p.oscale * (p.oscale2 ? *p.oscale2 : 1.f);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) o[i] *= os;
  }
  // fragment element i = 4 j + 2 h + e: row rowpix[h], column 8 j + 2 tq + e
  int b[2];
  float* orow[2];
  for (int h = 0; h < 2; ++h) {
    const int m = rowpix[h];
    const int xi = m % p.bw, yi = (m / p.bw) % p.bh, bi = m / (p.bw * p.bh);
    b[h] = t.b0 + bi;
    const int Y = p.out_scale * (t.y0 + yi) + (t.ph >> 1) * (p.out_scale - 1);
    const int X = p.out_scale * (t.x0 + xi) + (t.ph & 1) * (p.out_scale - 1);
    orow[h] = p.out + (((int64_t)b[h] * p.out_H + Y) * p.out_W + X) * p.Cout + t.n0 + 2 * tq;
  }
  if (p.bias) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) o[i] += p.bias[t.n0 + 8 * (i >> 2) + 2 * tq + (i & 1)];
  }
  if (p.stats) {
    // BatchNorm statistics from the convolution epilogue (nn.SpatialBatchNormalization, models.lua:65,70), three
    // partials per tile and column over its valid pixels: the sums of z and of z^2 and the sum of squared deviations
    // from the tile's mean.  bn_finalize_parts_kernel forms the variance from the first two (one pass) unless that
    // cancels: a channel whose mean is large against its spread, or whose variance is below eps, loses ~2^-24 mean^2 of
    // its variance there, and then combines the third in double.  For the third each warp sums z - s and (z - s)^2
    // over its 16 rows, s = z of its first row (a sample of the same column, so the sums no longer carry the mean), and
    // one thread per column moves the 8 warps' sums to warp 0's shift.  Each warp reduces its rows with shuffles, the
    // 8 warps meet in shared memory; every sum has a fixed order => replicas stay identical.
    const bool v0 = b[0] < p.B, v1 = b[1] < p.B;
    const int nvalid = p.bb == 1 ? 128 : min(p.bb, p.B - t.b0) * p.bw * p.bh;  // = bn_tile_count in k_elem.cu
    const int gi = ((g & 1) << 2) | (g & 2) | ((g & 4) >> 2);  // which of the 8 values lane g is left with (below)
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      // this lane's 2 columns x {z, z^2, z - s, (z - s)^2} summed over its 2 rows: v[2 q + e], q = the quantity
      float v[8];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float z0 = v0 ? o[4 * j + e] : 0.f, z1 = v1 ? o[4 * j + 2 + e] : 0.f;
        v[e] = z0 + z1;
        v[2 + e] = z0 * z0 + z1 * z1;
        const float s = __shfl_sync(0xffffffffu, o[4 * j + e], tq);  // row 16 warp (g = 0, h = 0) of this column
        const float d0 = v0 ? o[4 * j + e] - s : 0.f, d1 = v1 ? o[4 * j + 2 + e] - s : 0.f;
        v[4 + e] = d0 + d1;
        v[6 + e] = fmaf(d0, d0, d1 * d1);
        if (g == 0) stat_sm[(4 * 8 + warp) * BN + 8 * j + 2 * tq + e] = s;
      }
      // sum over the 8 lanes of equal tq (xor 4, 8, 16), halving the values each lane holds at every step: the
      // lane whose mask bit is 0 keeps the lower half.  Each value sees the additions of a plain xor-shuffle tree,
      // in the same pairs.
#pragma unroll
      for (int L = 8, m = 4; L > 1; L >>= 1, m <<= 1) {
        const bool up = (lane & m) != 0;
#pragma unroll
        for (int k = 0; k < L / 2; ++k) {
          const float send = up ? v[k] : v[k + L / 2], keep = up ? v[k + L / 2] : v[k];
          v[k] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
      }
      stat_sm[((gi >> 1) * 8 + warp) * BN + 8 * j + 2 * tq + (gi & 1)] = v[0];
    }
    consumer_sync();
    const int et = threadIdx.x;
    const int mt = tile / (p.Cout / BN);
    if (et < BN) {  // threads [0, BN): the sums of z and z^2
      float s0 = 0.f, s1 = 0.f;
      for (int w = 0; w < 8; ++w) {
        s0 += stat_sm[(0 * 8 + w) * BN + et];
        s1 += stat_sm[(1 * 8 + w) * BN + et];
      }
      p.stats[((int64_t)mt * 3 + 0) * p.Cout + t.n0 + et] = s0;
      p.stats[((int64_t)mt * 3 + 1) * p.Cout + t.n0 + et] = s1;
    } else if (et < 2 * BN) {  // threads [BN, 2 BN): the squared deviations from the tile mean
      // sum over the valid rows of (z - r) and (z - r)^2, r = warp 0's shift: warp w's n rows moved by d = s_w - r
      const int col = et - BN;
      const float r = stat_sm[(4 * 8 + 0) * BN + col];
      float t1 = 0.f, t2 = 0.f;
      for (int w = 0; w < 8; ++w) {
        const float n = (float)max(0, min(16, nvalid - 16 * w));
        const float xs = stat_sm[(2 * 8 + w) * BN + col], ys = stat_sm[(3 * 8 + w) * BN + col];
        const float d = stat_sm[(4 * 8 + w) * BN + col] - r;
        t1 += fmaf(n, d, xs);
        t2 += fmaf(d, fmaf(n, d, 2.f * xs), ys);
      }
      p.stats[((int64_t)mt * 3 + 2) * p.Cout + t.n0 + col] = fmaxf(0.f, fmaf(-t1 / (float)nvalid, t1, t2));
    }
    consumer_sync();
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (b[h] < p.B) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        *reinterpret_cast<float2*>(orow[h] + 8 * j) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
    }
  }
}

template <int BN, bool F16 = false>
__global__ void __launch_bounds__(kTcThreads, 1) tapconv_tc_kernel(const __grid_constant__ TcFwdParams p) {
  constexpr uint32_t kStageBytes = fwd_stage_bytes<BN>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;
  float* stat_sm = reinterpret_cast<float*>(smem + kStages * kStageBytes + 256);  // [5][8 warps][BN] (p.stats only)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = p.ntiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, kConsumerThreads / 32);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    producer_regs();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      prefetch_tmap(&p.b_hi);
      prefetch_tmap(&p.b_lo);
      uint32_t kbg = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) tapconv_load_tile<BN, F16>(p, tile, smem, full, empty, kbg);
    }
    return;
  }

  consumer_regs();
  uint32_t kbg = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) tapconv_mma_tile<BN, F16>(p, tile, smem, full, empty, stat_sm, kbg);
}

// ------------------------------------------------------------------------------------------------
// wgrad: D[n (M=128 of Cout)][c (BN of Cin)] += sum over a pixel range of dY[p][n] * X[p+off][c]
// grid: x = tile-tap, y = mtile * ntiles_n + ntile, z = K split.  Split z stores its sums to its own partial
// (p.out + z * p.split_stride); k_splitk_reduce adds the partials in split order.
// Same three-term scheme: main = dY_hi x X_hi, cross = dY_hi x X_lo + dY_lo x X_hi.
// Both operands are MN-major in memory (channels contiguous, K = pixels).
// F16 (3xFP16 split): a K block is 64 pixels, a channel group 64 channels (128 bytes of fp16); TMA lands the
// canonical MN-major SWIZZLE_128B layout and the wgmmas read it transposed.
// TF32: wgmma takes tf32 operands K-major only, so TMA lands plain [group][32 pixels][32 ch] boxes and the consumers
// transpose each K block into one K-major, 128B-swizzled buffer (rows = channels, 32 pixels = 128 bytes) before the MMAs.
// ------------------------------------------------------------------------------------------------
template <bool F16>
constexpr int wg_stages() { return F16 ? 3 : 2; }

// K-major 128B-swizzled row `n`, K element `k` (< 32) of a tf32 tile
__device__ __forceinline__ uint32_t sw128_off(int n, int k) {
  return (uint32_t)n * 128 + ((uint32_t)((k >> 2) ^ (n & 7)) << 4) + (uint32_t)(k & 3) * 4;
}
// `rows` channels x 32 pixels: staged [rows/32][32 px][32 ch] -> K-major swizzled [rows][32 px]
__device__ __forceinline__ void transpose_block(const uint8_t* src, uint8_t* dst, int rows, int tid) {
  for (int u = tid; u < rows * 8; u += kConsumerThreads) {
    const int q8 = u & 7, r = u >> 3, px = r & 31, grp = r >> 5;
    const float4 v = *reinterpret_cast<const float4*>(src + ((grp * 32 + px) * 32 + q8 * 4) * 4);
    const int n = grp * 32 + q8 * 4;
    *reinterpret_cast<float*>(dst + sw128_off(n + 0, px)) = v.x;
    *reinterpret_cast<float*>(dst + sw128_off(n + 1, px)) = v.y;
    *reinterpret_cast<float*>(dst + sw128_off(n + 2, px)) = v.z;
    *reinterpret_cast<float*>(dst + sw128_off(n + 3, px)) = v.w;
  }
}

template <int BN, bool F16>
struct WgLayout {
  static constexpr int kS = wg_stages<F16>();
  static constexpr int kG = F16 ? 64 : 32;                  // channels per 128-byte group
  static constexpr uint32_t kBox = (F16 ? 64 : 32) * 128;   // one (group x K-block pixels) box: 32 px (tf32) / 64 px (fp16)
  static constexpr uint32_t kAB = (128 / kG) * kBox;        // M = 128 channels of dY
  static constexpr uint32_t kBB = (BN / kG) * kBox;
  static constexpr uint32_t kStageBytes = 2 * kAB + 2 * kBB;  // {dy_hi, dy_lo, x_hi, x_lo}
};

// one weight-gradient work item: tile-tap tt, output block [m0, m0 + 128) x [c0, c0 + BN), K blocks
// [kb_begin, kb_begin + nkb) of split z
struct WgItem {
  int tt, m0, c0, z, kb_begin, nkb;
};
template <int BN>
__device__ __forceinline__ WgItem wg_decode(const TcWgParams& p, int tt, int mn, int z) {
  const int ntn = p.Cin / BN;
  WgItem w;
  w.tt = tt;
  w.m0 = (mn / ntn) * 128;
  w.c0 = (mn % ntn) * BN;
  w.z = z;
  w.kb_begin = z * p.kb_per_split;
  w.nkb = min(p.kblocks, w.kb_begin + p.kb_per_split) - w.kb_begin;
  return w;
}

// producer side of one item (kbg: the running K-block counter of the stage ring, as in tapconv_load_tile)
template <int BN, bool F16>
__device__ __forceinline__ void wgrad_load_item(const TcWgParams& p, const WgItem& w, uint8_t* smem, uint64_t* full,
                                                uint64_t* empty, uint32_t& kbg) {
  using L = WgLayout<BN, F16>;
  const int ph = p.phase[w.tt], dyo = p.dy[w.tt], dxo = p.dx[w.tt];
  for (int i = 0; i < w.nkb; ++i, ++kbg) {
    const int s = kbg % L::kS, it = kbg / L::kS;
    if (it > 0) mbar_wait_spin(empty + s, (it - 1) & 1);
    const int kb = w.kb_begin + i;
    int b0, y0, x0;
    if (p.bb == 1) {
      const int per_img = p.tiles_x * p.tiles_y;
      b0 = kb / per_img;
      const int r = kb % per_img;
      y0 = (r / p.tiles_x) * p.bh;
      x0 = (r % p.tiles_x) * p.bw;
    } else {
      b0 = kb * p.bb;
      y0 = 0;
      x0 = 0;
    }
    uint8_t* st = smem + s * L::kStageBytes;
    mbar_expect_tx(full + s, L::kStageBytes);
    // 5-D maps (group channels, w, h, b, channel-group): ONE bulk copy lands [group][pixel][group channels] = all
    // the boxes of an operand
    tma_load_5d(st, &p.dy_hi[ph], full + s, 0, x0, y0, b0, w.m0 / L::kG);
    tma_load_5d(st + L::kAB, &p.dy_lo[ph], full + s, 0, x0, y0, b0, w.m0 / L::kG);
    tma_load_5d(st + 2 * L::kAB, &p.x_hi, full + s, 0, x0 + dxo, y0 + dyo, b0, w.c0 / L::kG);
    tma_load_5d(st + 2 * L::kAB + L::kBB, &p.x_lo, full + s, 0, x0 + dxo, y0 + dyo, b0, w.c0 / L::kG);
  }
}

// consumer side of one item: the K loop, the promotions and the store of the [n][c] block
template <int BN, bool F16>
__device__ __forceinline__ void wgrad_mma_item(const TcWgParams& p, const WgItem& w, uint8_t* smem, uint64_t* full,
                                               uint64_t* empty, uint32_t& kbg) {
  using L = WgLayout<BN, F16>;
  constexpr uint32_t kBox = L::kBox, kAB = L::kAB, kBB = L::kBB;
  uint8_t* kbuf = smem + L::kS * L::kStageBytes;  // tf32: the K-major copy of one stage
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, g = lane >> 2, tq = lane & 3;
  const int nkb = w.nkb;
  const int kChunk = p.chunk;
  const int nchunks = (nkb + kChunk - 1) / kChunk;
  float acc[BN];
  float o[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) o[i] = 0.f;
  for (int ch = 0; ch < nchunks; ++ch) {
    const int nk = min(kChunk, nkb - ch * kChunk);
    int prev = -1;
    for (int j = 0; j < nk; ++j, ++kbg) {
      const int s = kbg % L::kS, it = kbg / L::kS;
      const uint32_t sa = smem_u32(smem + s * L::kStageBytes);
      mbar_wait(full + s, it & 1);
      if constexpr (F16) {
        // canonical MN-major SWIZZLE_128B layout: atoms of 64 channels x 8 pixels (1 KB), LBO = distance between
        // 64-channel groups (one 8 KB box), SBO = distance between 8-pixel groups (1 KB); one wgmma takes K = 16
        // pixels = 2 KB.  The warpgroup's 64 dY channels are one group.
        mma_kblock<BN, true, true>(acc, make_desc(sa + wg * kBox, kBox, 1024), make_desc(sa + kAB + wg * kBox, kBox, 1024),
                                   make_desc(sa + 2 * kAB, kBox, 1024), make_desc(sa + 2 * kAB + kBB, kBox, 1024), 128, j == 0);
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(empty + prev);
        prev = s;
      } else {
        const uint8_t* st = smem + s * L::kStageBytes;
        transpose_block(st, kbuf, 128, threadIdx.x);                        // dy_hi -> rows [0, 128)
        transpose_block(st + kAB, kbuf + 128 * 128, 128, threadIdx.x);      // dy_lo -> rows [128, 256)
        transpose_block(st + 2 * kAB, kbuf + 256 * 128, BN, threadIdx.x);   // x_hi -> rows [256, 256 + BN)
        transpose_block(st + 2 * kAB + kBB, kbuf + (256 + BN) * 128, BN, threadIdx.x);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to wgmma
        consumer_sync();
        if (lane == 0) mbar_arrive(empty + s);
        const uint32_t ka = smem_u32(kbuf);
        mma_kblock<BN, false, false>(acc, make_desc(ka + wg * 64 * 128, 16, 1024),
                                     make_desc(ka + (128 + wg * 64) * 128, 16, 1024), make_desc(ka + 256 * 128, 16, 1024),
                                     make_desc(ka + (256 + BN) * 128, 16, 1024), 2, j == 0);
        wgmma_wait<0>();
        consumer_sync();  // both warpgroups are done with kbuf
      }
    }
    if constexpr (F16) {
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty + prev);
    }
    promote<BN, F16>(o, acc);
  }
  if (p.oscale) {  // dY (and X) were stored scaled by powers of two
    const float os = *p.oscale * (p.oscale2 ? *p.oscale2 : 1.f);
#pragma unroll
    for (int k = 0; k < BN / 2; ++k) o[k] *= os;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = w.m0 + wg * 64 + (warp & 3) * 16 + g + 8 * h;
    float* orow = p.out + w.z * p.split_stride + ((int64_t)w.tt * p.Cout + n) * p.Cin + w.c0 + 2 * tq;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      orow[8 * j] = o[4 * j + 2 * h];
      orow[8 * j + 1] = o[4 * j + 2 * h + 1];
    }
  }
}

template <int BN, bool F16 = false>
__global__ void __launch_bounds__(kTcThreads, 1) wgrad_tc_kernel(const __grid_constant__ TcWgParams p) {
  using L = WgLayout<BN, F16>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (L::kS + (F16 ? 0 : 1)) * L::kStageBytes);
  uint64_t* empty = full + L::kS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const WgItem w = wg_decode<BN>(p, blockIdx.x, blockIdx.y, blockIdx.z);

  if (threadIdx.x == 0) {
    for (int s = 0; s < L::kS; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, kConsumerThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (w.nkb <= 0) return;

  uint32_t kbg = 0;
  if (warp >= kConsumerThreads / 32) {
    producer_regs();
    if (warp == kConsumerThreads / 32 && lane == 0) wgrad_load_item<BN, F16>(p, w, smem, full, empty, kbg);
    return;
  }
  consumer_regs();
  wgrad_mma_item<BN, F16>(p, w, smem, full, empty, kbg);
}

// ------------------------------------------------------------------------------------------------
// bwd_pair: the weight gradient AND the data gradient of one upsampled 5x5 layer (3xFP16, collapsed) in one
// persistent launch.  Work item ids [0, nwg) are unsplit weight-gradient items (tile-tap, Cout tile, Cin tile; the
// whole K range), [nwg, nitems) the dgrad tiles of tc_conv_dgrad_ups: the long items go out first and the short
// tiles fill in around them.  The producer lane claims the next id from a device counter and hands it to the
// consumers through a small ring of id slots with its own full / empty mbarriers.  Both kinds use the same 64 KB
// stages, so the stage ring runs on across items of either kind and the producer loads the next item while the
// consumers run the current one's epilogue.  Each item runs the body of its own kernel: its result is bit for bit
// what the two separate launches write.
// ------------------------------------------------------------------------------------------------
constexpr int kIdSlots = 2;

template <int BN>
__global__ void __launch_bounds__(kTcThreads, 1) bwd_pair_tc_kernel(const __grid_constant__ TcBwdParams p) {
  using L = WgLayout<BN, true>;
  static_assert(L::kS == kStages && L::kStageBytes == fwd_stage_bytes<BN>(), "one stage ring for both item kinds");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * L::kStageBytes);
  uint64_t* empty = full + kStages;
  uint64_t* id_full = empty + kStages;
  uint64_t* id_empty = id_full + kIdSlots;
  volatile int* ids = reinterpret_cast<volatile int*>(id_empty + kIdSlots);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nmn = (p.wg.Cout / 128) * (p.wg.Cin / BN);  // weight-gradient output blocks per tile-tap

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, kConsumerThreads / 32);
    }
    for (int s = 0; s < kIdSlots; ++s) {
      mbar_init(id_full + s, 1);
      mbar_init(id_empty + s, kConsumerThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  uint32_t kbg = 0;
  if (warp >= kConsumerThreads / 32) {
    producer_regs();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      prefetch_tmap(&p.dg.b_hi);
      prefetch_tmap(&p.dg.b_lo);
      for (uint32_t n = 0;; ++n) {
        const uint32_t slot = n % kIdSlots, use = n / kIdSlots;
        if (use > 0) mbar_wait_spin(id_empty + slot, (use - 1) & 1);
        const int id = atomicAdd(p.claim, 1);
        ids[slot] = id;
        mbar_arrive(id_full + slot);  // release: the consumers' wait on id_full acquires the id
        if (id >= p.nitems) break;
        if (id < p.nwg) wgrad_load_item<BN, true>(p.wg, wg_decode<BN>(p.wg, id / nmn, id % nmn, 0), smem, full, empty, kbg);
        else tapconv_load_tile<BN, true>(p.dg, id - p.nwg, smem, full, empty, kbg);
      }
    }
    return;
  }

  consumer_regs();
  for (uint32_t n = 0;; ++n) {
    const uint32_t slot = n % kIdSlots, use = n / kIdSlots;
    mbar_wait(id_full + slot, use & 1);
    const int id = ids[slot];
    __syncwarp();
    if (lane == 0) mbar_arrive(id_empty + slot);
    if (id >= p.nitems) break;
    if (id < p.nwg) wgrad_mma_item<BN, true>(p.wg, wg_decode<BN>(p.wg, id / nmn, id % nmn, 0), smem, full, empty, kbg);
    else tapconv_mma_tile<BN, true>(p.dg, id - p.nwg, smem, full, empty, nullptr, kbg);
  }
}
