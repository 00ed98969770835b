// One convolution / Linear layer of the nets built outside nets.cu (coarse-to-fine nets, --scale 16 nets): weight
// packs, TF32 splits and the forward / backward dispatch over the wgmma, bandwidth-shaped and fp32 FFMA kernels.
#pragma once
#include <vector>

#include "fg_internal.h"

struct ConvL {  // NHWC, stride 1, "same" padding (a strided layer runs at stride 1 and is subsampled by its net)
  int Cin = 0, Cout = 0, k = 1, H = 1;
  int64_t w_off = 0, b_off = 0;
  int cA = 0, cS = 0;  // Linear after View([C][H][W]): column j=c*S+s of the reference <-> our NHWC column s*A+c
  int nA = 0, nS = 0;  // Linear before View([C][H][W]): the same permutation on the output rows (weights, bias, gradients)
  float *Wp = nullptr, *Wpd = nullptr;                                            // fp32 packs [t][n][c], [t'][c][n]
  float* bp = nullptr;                                                            // bias in our row order (nA != 0)
  float *Wf_hi = nullptr, *Wf_lo = nullptr, *Wd_hi = nullptr, *Wd_lo = nullptr;   // TF32 splits of the packs
  float *x_hi = nullptr, *x_lo = nullptr;                                         // split of the input (fwd -> wgrad)
  float* sx = nullptr;       // device (max|x|, 1/scale) of the input's FP16 split (option mma_f16)
  bool packed_f16 = false;   // the hi/lo buffers currently hold the FP16 split (set by convl_pack)
  // Layers whose output side is too narrow for a tensor-core tile still run there with zero-padded channels:
  //   pad_out (Cout <= 4, e.g. the 256->C 7x7 output layer): forward with the weights padded to pad_out rows;
  //           wgrad with the roles swapped (big channel count on the 128-row M side, padded dY on the N side)
  //   pad_dy  (Cout == 64): wgrad with dY padded to the 128 rows the M side needs
  int pad_out = 0, pad_dy = 0;
  float *Wq_hi = nullptr, *Wq_lo = nullptr;  // [t][pad_out][Cin] TF32 hi/lo
  bool need_dgrad = true;
  const char *tf = "", *td = "", *tw = "";
  ConvGeom geom(int B) const { return ConvGeom{B, H, H, Cin, Cout, k, 1}; }
  ConvGeom geom_d(int B) const { return ConvGeom{B, H, H, Cout, Cin, k, 1}; }
};

// what a layer needs from the net that owns it: the allocation list and the shared scratch buffers
struct ConvLEnv {
  fg_ctx* c = nullptr;
  int maxB = 0;
  std::vector<void*>* allocs = nullptr;
  float *ga = nullptr;                          // padded forward output (pad_out layers): maxB * H*H * pad_out floats
  float *dy_hi = nullptr, *dy_lo = nullptr;     // TF32 split of the current dY (largest layer output)
  float *pad_hi = nullptr, *pad_lo = nullptr;   // channel-padded TF32 split of dY (pad_out / pad_dy layers)
  float* ws = nullptr;                          // packed weight-gradient workspace (largest layer)
  float* sdy = nullptr;                         // device (max|dY|, 1/scale) of the current dY's FP16 split
};

// what the weight packs depend on besides the parameters: re-pack when it changes
inline int pack_key(const fg_ctx* c) { return c->conv_impl | (c->mma_f16 << 4); }
int convl_dalloc(ConvLEnv& e, float** p, size_t elems);  // zero-filled device buffer, owned by *e.allocs
int convl_alloc(ConvLEnv& e, ConvL& L);
int convl_pack(fg_ctx* c, ConvL& L, const float* P);
int convl_fwd(ConvLEnv& e, ConvL& L, const float* in, const float* P, float* out, int B);
// G (may be null): dW += wgrad, db += colsum(dy).  din (may be null) = dgrad.
int convl_bwd(ConvLEnv& e, ConvL& L, const float* in, const float* dy, float* G, float* din, int B);
