// Host entry points of k_misc.cu (table ops, max pooling, dropout, NCHW pooling/upsampling).
#pragma once
#include "fg_internal.h"

// first strict maximum of a 2x2 window in row-major order (THNN SpatialMaxPooling: `val > maxval`); a NaN in the first
// position passes through
__device__ __forceinline__ int argmax4(float v0, float v1, float v2, float v3, float* best) {
  int j = 0;
  float m = v0;
  if (v1 > m) { m = v1; j = 1; }
  if (v2 > m) { m = v2; j = 2; }
  if (v3 > m) { m = v3; j = 3; }
  *best = m;
  return j;
}

// NHWC (fused nets)
int k_join_to_nhwc(fg_ctx* c, const float* noise_nchw, const float* cond_nchw, float* out_nhwc, int B, int C, int HW);
int k_add(fg_ctx* c, const float* a, const float* b, float* out, int64_t n);
int k_maxpool2_fwd(fg_ctx* c, const float* h, float* p, int B, int H, int W, int C);                  // H,W: input size
int k_maxpool2_bwd(fg_ctx* c, const float* dp, const float* h, float* dh, int B, int H, int W, int C);
// y = x * mask * scale; mask element order is the reference's NCHW flattening: masks[b*stride + moff + ch*HW + q]
int k_dropout_nhwc(fg_ctx* c, const float* x, const float* masks, int64_t stride, int moff, int HW, int C, float scale,
                   float* y, int B);
// 1 with probability 1-p_drop; seed_dev (optional): effective seed = *seed_dev * 2 + seed.  out[i] is element
// offset + i of the stream, so a slice of a longer draw can be drawn on its own.
int k_bernoulli_keep(fg_ctx* c, float* out, int64_t n, uint64_t seed, float p_drop, const uint64_t* seed_dev = nullptr,
                     int64_t offset = 0);
// channel padding around the tensor-core kernels (layers with a narrow output side)
int k_pad_split(fg_ctx* c, const float* src, float* hi, float* lo, int64_t P, int Cs, int Cp);       // [P][Cs] -> TF32 hi/lo [P][Cp]
int k_compact_bias(fg_ctx* c, const float* src, const float* bias, float* dst, int64_t P, int Cs, int Cp);
// 3xFP16-split variants (halves in the same buffers; amax_slot: (max|src|, 1/scale) pair filled by tc_amax / written here)
int k_pad_split_h(fg_ctx* c, const float* src, float* hi, float* lo, int64_t P, int Cs, int Cp, float* amax_slot);
int k_pack_pad_split_h(fg_ctx* c, const float* W, float* hi, float* lo, int N, int Np, int Cc, int KK);
int k_pack_pad_split(fg_ctx* c, const float* W, float* hi, float* lo, int N, int Np, int Cc, int KK);  // W[N][Cc][KK] -> [t][Np][Cc]
int k_unpack_wgrad_pad(fg_ctx* c, const float* G, float* dW, int N, int Np, int Cc, int KK);          // dW += G[t][n<N][c]
int k_unpack_wgrad_swapped(fg_ctx* c, const float* Gt, float* dW, int N, int Np, int Cc, int KK);     // dW += Gt[KK-1-t][c][n<N]
// NCHW (L-op boundary); H,W are the sizes of the layer INPUT
int k_up2_fwd_nchw(fg_ctx* c, const float* x, float* y, int64_t BC, int H, int W);
int k_up2_bwd_nchw(fg_ctx* c, const float* dy, float* dx, int64_t BC, int H, int W);
int k_avgpool2_fwd_nchw(fg_ctx* c, const float* x, float* y, int64_t BC, int H, int W);
int k_avgpool2_bwd_nchw(fg_ctx* c, const float* dy, float* dx, int64_t BC, int H, int W);
int k_maxpool2_fwd_nchw(fg_ctx* c, const float* x, float* y, int64_t BC, int H, int W);
int k_maxpool2_bwd_nchw(fg_ctx* c, const float* x, const float* dy, float* dx, int64_t BC, int H, int W);
int k_dropout_nchw(fg_ctx* c, const float* x, const float* mask, float scale, int inner, float* y, int64_t n);
