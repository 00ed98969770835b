// Layer-level dispatch of the layer types in fg_internal.h (TcOp, ConvL, UpsL, ConvLEnv): weight packs, tensor-core
// operand splits and the forward / backward dispatch over the wgmma, bandwidth-shaped and fp32 FFMA kernels.  ConvL
// serves the coarse-to-fine and --scale 16 nets; UpsL serves G's upsampled layers of the 32x32 and --scale 16 generators.
#pragma once
#include <vector>

#include "fg_internal.h"

// option "mma_f16": tensor-core operands in the 3xFP16 split (only with the phase-collapsed kernels)
inline bool tc_f16(const fg_ctx* c) { return c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED; }

// The ONE elementwise producer launched inside the scope also reduces max|output| into `pair` (with the FP16 split) and
// sets *done, so that the consuming layer skips its own read pass.  The pair's max word must be zero (ScalePairs::reset).
struct AmaxInto {
  fg_ctx* c;
  AmaxInto(fg_ctx* c_, TcOp& op) : AmaxInto(c_, op.s, &op.amax_ready) {}
  AmaxInto(fg_ctx* c_, float* pair, bool* done) : c(c_) {
    if (tc_f16(c)) {
      c->amax_out = reinterpret_cast<unsigned*>(pair);
      c->amax_done = done;
    }
  }
  ~AmaxInto() { c->amax_out = nullptr; }
};

// host side of a producer's launch: the word it reduces max|output| into (amax_commit, k_f16split.cuh), or null; says
// so in *c->amax_done
inline unsigned* take_amax(fg_ctx* c) {
  unsigned* p = c->amax_out;
  if (p) *c->amax_done = true;
  return p;
}

// the split of x (n elements) into op, in the format `f16` chooses, minus whatever the producer already did
int tc_op_split(fg_ctx* c, TcOp& op, const float* x, int64_t n, bool f16);

// what the weight packs depend on besides the parameters: re-pack when it changes
inline int pack_key(const fg_ctx* c) { return c->conv_impl | (c->mma_f16 << 4); }
int convl_dalloc(ConvLEnv& e, float** p, size_t elems);  // zero-filled device buffer, owned by *e.allocs
int convl_alloc(ConvLEnv& e, ConvL& L);
// the buffers of L's input operand only (x.s unless set, x's split, xpad): what a copy of the layer that shares its
// weight packs needs for a forward of its own (gen_alloc_fwd)
int convl_alloc_x(ConvLEnv& e, ConvL& L);
bool convl_tc_fwd(const fg_ctx* c, const ConvL& L);  // the forward runs on the tensor cores (it reads the input's split)
bool convl_tc_bwd(const fg_ctx* c, const ConvL& L);  // ... and so does the data gradient
int convl_pack(fg_ctx* c, ConvL& L, const float* P);
int convl_fwd(ConvLEnv& e, ConvL& L, const float* in, const float* P, float* out, int B);
bool convl_tc_wgrad(const fg_ctx* c, const ConvL& L);  // the weight gradient runs on the tensor cores (reads the splits)
// G (may be null): dW += wgrad, db += colsum(dy).  din (may be null) = dgrad.  The flags of e.dy say what dY's producer
// already did (split into L's dY split, max|dY| into L.sdy, bias gradient added); they are cleared.  wgrad_side: the
// weight gradient of a layer without pad_out / pad_dy goes to the wgrad stream (OnWgradStream); the caller keeps
// what it reads (in, dy or L's splits) unchanged until wgrad_join.
int convl_bwd(ConvLEnv& e, ConvL& L, const float* in, const float* dy, float* G, float* din, int B, bool wgrad_side = false);

// option "bwd_streams": whether a backward on e may put weight gradients on c->wgrad_stream.  Timing runs (per-launch
// timers on one stream would misattribute the overlap), debug_keep runs and data-parallel steps stay on one stream.
bool wgrad_async(const fg_ctx* c, const ConvLEnv& e);
// While one lives (with `on`), launches go to c->wgrad_stream, after everything enqueued on c->stream so far, with that
// stream's own copy of each workspace a weight gradient writes (c->wgrad_ws, e.ws_w).  r: the fork's error, if any.
struct OnWgradStream {
  ConvLEnv& e;
  bool on;
  int r = FG_OK;
  OnWgradStream(ConvLEnv& e, bool on);
  ~OnWgradStream();
};
// c->stream waits for every launch made on c->wgrad_stream so far (nothing to do when none was made since the last join)
int wgrad_join(ConvLEnv& e);

bool upsl_tc(const fg_ctx* c, const UpsL& U);  // the layer runs on the tensor cores
int upsl_alloc(ConvLEnv& e, UpsL& U);
int upsl_alloc_x(ConvLEnv& e, UpsL& U);  // the same share of upsl_alloc (x's split, x.s unless set)
int upsl_pack(fg_ctx* c, UpsL& U, const float* P);
// *parts (optional, in: want BatchNorm partials; out: how many tiles wrote one into c->bn_parts, 0 = none)
int upsl_fwd(ConvLEnv& e, UpsL& U, const float* h, const float* P, float* z, int B, int* parts = nullptr);
// G: dW += wgrad (the bias gradient is the producer's: k_bn_prelu_bwd_apply's dbias); dh = dgrad; dy: the operand dz is
// split into.  *pooled: dh already is the gradient of the LOW-RES input (the tensor-core dgrad folds in the 2x2 sum of
// the upsample backward); otherwise dh is the full-resolution gradient the consumer still sums 2x2.
int upsl_bwd(ConvLEnv& e, UpsL& U, TcOp& dy, const float* h, const float* dz, float* G, float* dh, int B, bool* pooled,
             bool wgrad_side = false);

// ---- gen.cu: UpsGen on the owner's layer scratch (ConvLEnv) and parameters (NetPair: PG, gG, bnG, G_pack) ----
int gen_alloc(ConvLEnv& e, UpsGen& G, const GenDesc& d);
// a forward-only instance F of an allocated G (F.owner): G's weight packs, its own input operands, scale pairs,
// activations and batch statistics for batches up to e.maxB
int gen_alloc_fwd(ConvLEnv& e, UpsGen& F, UpsGen& G);
int gen_pack(fg_ctx* c, UpsGen& G, NetPair& p);  // unless p.G_pack is the current pack_key()
// noise: device [B][100] -> G.y (NHWC [B][S][S][C]).  training: batch statistics + running statistics update
int gen_forward(ConvLEnv& e, UpsGen& G, NetPair& p, const float* noise, int B, bool training);
// dy: NHWC [B][S][S][C] of the last (training-mode) forward; accumulates into p.gG; dnoise (device [B][100]) may be null
int gen_backward(ConvLEnv& e, UpsGen& G, NetPair& p, const float* dy, float* dnoise);
void gen_debug_rows(const UpsGen& G, std::vector<DebugTensor>& rows);  // "G.*" of fg_*debug_tensor
