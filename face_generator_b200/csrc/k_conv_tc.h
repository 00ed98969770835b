// Parameter blocks (passed as __grid_constant__) and host entry points of the wgmma conv path.
#pragma once
#include <cuda.h>

#include <cstdint>

#include "fg_internal.h"

constexpr int kTcMaxTaps = 100;

struct alignas(64) TcFwdParams {
  CUtensorMap a_hi[4], a_lo[4];  // activation views (dgrad of an upsampled conv: one per output phase of dY)
  CUtensorMap b_hi, b_lo;        // packed weights, 2-D (Cin, taps*Cout)
  int8_t dy[kTcMaxTaps], dx[kTcMaxTaps], amap[kTcMaxTaps];  // indexed [phase*ntaps + tap]
  int16_t widx[kTcMaxTaps];
  int ntaps, nphase, kpt, Cout;
  int B, H, W;         // tile-enumeration grid (the low-res grid for upsampled convs)
  int bw, bh, bb;      // pixel box of one 128-row M tile
  int tiles_x, tiles_y, tiles_per_phase, ntiles;
  float* out;
  const float* bias;
  float* stats;  // optional [m-tile][2][Cout]: per-tile column sums of the output and of its square (BatchNorm)
  int out_H, out_W, out_scale;
  const float *oscale, *oscale2;  // optional device scalars the accumulators are multiplied by (inverse operand scales)
  int chunk;  // K-blocks accumulated in the wgmma accumulators before they are promoted to fp32 registers
};

struct alignas(64) TcWgParams {
  CUtensorMap dy_hi[4], dy_lo[4];
  CUtensorMap x_hi, x_lo;
  int8_t dy[kTcMaxTaps], dx[kTcMaxTaps], phase[kTcMaxTaps];  // per tile-tap
  int Cout, Cin;
  int bw, bh, bb;      // 32-pixel box of one K block
  int tiles_x, tiles_y;
  int kblocks, kb_per_split;
  float* out;
  int64_t split_stride;  // elements between the partial outputs of two K splits
  const float *oscale, *oscale2;  // optional device scalars multiplied into the result (inverse scales of dY and X)
  int chunk;
};

// weight gradient + data gradient of one upsampled 5x5 layer in one persistent launch (bwd_pair_tc_kernel)
struct alignas(64) TcBwdParams {
  TcWgParams wg;
  TcFwdParams dg;
  int* claim;      // device counter of claimed work items, zeroed before every launch
  int nwg, nitems;  // ids [0, nwg): weight-gradient items, [nwg, nitems): dgrad tiles
};

bool tc_conv_eligible(const ConvGeom& g);
int tc_split(fg_ctx* c, const float* x, float* hi, float* lo, int64_t n);
int tc_pack_split(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc, int KK);
int tc_pack_collapsed(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc);
int tc_combine_collapsed_wgrad(fg_ctx* c, const float* G, float* dW, int N, int Cc);
// stats / n_parts (optional): the kernel also writes per-tile BatchNorm partials [*n_parts][2][Cout] (see TcFwdParams)
// f16 != 0: the four operand pointers are __half arrays holding the FP16 split (tc_split_h / tc_pack_*_h: hi = fp16(x),
// lo = fp16((x - hi) * 2^11)) and the kernel issues f16 MMAs (twice the tensor rate, half the operand bytes);
// oscale: optional device scalar multiplied into the result (inverse of the power-of-two scale tc_split_h applied)
int tc_conv_fwd(fg_ctx* c, const float* x_hi, const float* x_lo, const float* w_hi, const float* w_lo, const float* bias,
                float* out, ConvGeom g, int mode, float* stats = nullptr, int* n_parts = nullptr, int f16 = 0,
                const float* oscale = nullptr, const float* oscale2 = nullptr);
int tc_stat_parts(const ConvGeom& g, int mode);  // number of per-tile partials tc_conv_fwd writes for this geometry
int tc_conv_dgrad_ups(fg_ctx* c, const float* dy_hi, const float* dy_lo, const float* wd_hi, const float* wd_lo, float* out,
                      ConvGeom g, int f16 = 0, const float* oscale = nullptr);
// FP16 split of x (n % 4 == 0) into two __half arrays.  amax_slot (optional, device, 2 floats): x is first scaled by the
// power of two that brings max|x| (slot[0], filled by tc_amax) into [2^14, 2^15); slot[1] receives the inverse scale.
int tc_amax(fg_ctx* c, const float* x, int64_t n, float* amax_slot);
// inv_out (default amax_slot + 1) receives the inverse scale
int tc_split_h(fg_ctx* c, const float* x, float* hh, float* hl, int64_t n, float* amax_slot = nullptr, float* inv_out = nullptr);
int tc_pack_split_h(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc, int KK);
int tc_pack_collapsed_h(fg_ctx* c, const float* W, float* f_hi, float* f_lo, float* d_hi, float* d_lo, int N, int Cc);
int tc_conv_wgrad(fg_ctx* c, const float* x_hi, const float* x_lo, const float* dy_hi, const float* dy_lo, float* out,
                  ConvGeom g, int f16 = 0, const float* oscale = nullptr, const float* oscale2 = nullptr);
// tc_conv_wgrad (into the collapsed [36][Cout][Cin] `wg_out`) and tc_conv_dgrad_ups (into `dh`) of an upsampled 5x5
// layer on the 3xFP16 split, as one launch of bwd_pair_tc_kernel with the same per-tile arithmetic, so the same bits.
// Only for the shapes tc_bwd_pair_eligible accepts.  oscale_dy / oscale_x: inverse operand scales as for the two calls.
bool tc_bwd_pair_eligible(const fg_ctx* c, const ConvGeom& g);
bool tc_bwd_pair_pays(const fg_ctx* c, const ConvGeom& g);  // eligible, and its schedule estimate beats two launches
int tc_conv_bwd_ups(fg_ctx* c, const float* x_hi, const float* x_lo, const float* dy_hi, const float* dy_lo,
                    const float* wd_hi, const float* wd_lo, float* wg_out, float* dh, ConvGeom g, const float* oscale_dy,
                    const float* oscale_x);
int tc_tf32_peak(fg_ctx* c, int iters, int reps, double* tflops);
int tc_encode_nhwc_box(CUtensorMap* m, const float* base, int C, int W, int H, int B, int bc, int bw, int bh, int bb);
