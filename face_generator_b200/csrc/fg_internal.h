// Internal declarations shared by the translation units of libfg_b200.so.
// Everything on the device is NHWC fp32; the NCHW reference layouts exist only at the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <deque>
#include <functional>
#include <initializer_list>
#include <map>
#include <string>
#include <vector>

#include "fg_b200.h"

void fg_set_error(const char* fmt, ...);

#define FG_CUDA(call)                                                                               \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess) {                                                                       \
      fg_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));          \
      return FG_ERR_CUDA;                                                                           \
    }                                                                                               \
  } while (0)
#define FG_TRY(call)                  \
  do {                                \
    int r__ = (call);                 \
    if (r__ != FG_OK) return r__;     \
  } while (0)
#define FG_REQUIRE(cond, ...)         \
  do {                                \
    if (!(cond)) {                    \
      fg_set_error(__VA_ARGS__);      \
      return FG_ERR_INVALID;          \
    }                                 \
  } while (0)
// after every kernel launch on context c: count it and surface a launch error
#define LAUNCH_CHECK(c)                 \
  do {                                  \
    (c)->launches++;                    \
    FG_CUDA(cudaGetLastError());        \
  } while (0)
// grid of a grid-stride kernel over n elements: at most 16 blocks per SM of the H100's 132, at least 1
inline int grid_for(int64_t n, int block, int cap = 132 * 16) {
  int64_t g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}
#define GRID_STRIDE(i, n) \
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

constexpr int kMaskPerSample = 1984;  // 64+128+256+512 SpatialDropout + 512+512 Dropout keep flags
constexpr int kNoiseDim = 100;
constexpr int kSmallMaxParts = 2048;  // partial rows of the small-channel wgrad workspace
constexpr int kGradTail = 8;           // extra floats behind each flat gradient (DP-reduced scalars)
constexpr int kOptRedRows = 132 * 2;  // blocks of the penalty-loss reduction

// Geometry of one stride-1 "same" convolution seen as a sum over taps of shifted GEMMs.
// Output pixels p = (b,y,x) in [0,B)x[0,H)x[0,W); the stored input is [B][H/ups][W/ups][Cin]
// (ups = 2 folds nn.SpatialUpSamplingNearest(2) into the addressing).  Linear layers are k=1,H=W=1.
struct ConvGeom {
  int B, H, W, Cin, Cout, k, ups;
};

// Flat parameter layouts (getParameters() order), float offsets.
struct GLayout {
  int64_t L1W, L1b, a1, C1W, C1b, g1, be1, a2, C2W, C2b, g2, be2, a3, C3W, C3b, total;
};
GLayout make_g_layout(int C, int side);  // the generator of models.lua at side 32 (upsampling32) or 16 (upsampling16)

struct DeviceStats {  // lives in device memory; mirrored to fg_step_stats
  float loss_D, loss_G;
  int conf[4];
  int trained_D;
  int t_D, t_G;
  float acc_D;
  // gate state
  int acc_count, acc_head;
  float step_D, step_G;  // Adam step sizes prepared by adam_prep
  int do_train_D, do_train_G;
};
constexpr int kAccHistMax = 1024;
// the most D or G iterations one train step runs (train.lua --D_iterations / --G_iterations); c->seed_dev holds one
// stream root per iteration (k_seed_roots)
constexpr int kMaxIters = 16;
constexpr int kBnState = 768;  // running mean / var of G's two BatchNorm layers: [mean1 256][var1 256][mean2 128][var2 128]

// A captured train step (net_graph_run) and the key it was captured under
struct StepGraph {
  std::vector<uint8_t> key;
  cudaGraphExec_t exec = nullptr;
  int64_t launches = 0;
  bool failed = false;
};

// The trainable state of one G/D pair (the 32x32 nets, the coarse-to-fine nets, the --scale 16 nets)
struct NetPair {
  int64_t nG = 0, nD = 0;
  float *PG = nullptr, *PD = nullptr, *gG = nullptr, *gD = nullptr;  // flat parameters and gradients
  float *tailG = nullptr, *tailD = nullptr;  // the 8 DP-reduced scalars of each gradient: g + n, or elsewhere (fg_bind_params)
  float *mG = nullptr, *vG = nullptr, *mD = nullptr, *vD = nullptr;  // optimizer moments
  float* bnG = nullptr;  // [kBnState] G's BatchNorm running statistics; null when G has no BatchNorm
  DeviceStats* dstats = nullptr;
  DeviceStats* hstats = nullptr;  // pinned mirror
  float* acc_hist = nullptr;      // [kAccHistMax]
  // the pack_key() (convl.h) each half's weight packs were made under; -1: stale, the parameters changed since
  int G_pack = -1, D_pack = -1;
  std::vector<StepGraph> graphs;
  const char* optim_timer[2] = {nullptr, nullptr};  // ScopedTimer names of the G / D optimizer update (none: untimed)
  // option "debug_keep" (tests): the D iteration's tensors that the G iteration's D forward overwrites, copied by the
  // loop body (pair_train_step) and read back as the "Dstep.*" debug tensors.  The trainer fills the table at alloc.
  struct Keep {
    const char* name;       // "Dstep.<tensor>"
    const float* src;
    int64_t per;            // floats per sample
    float* copy = nullptr;  // maxB * per floats, allocated by the first kept step
  };
  std::vector<Keep> keep;
  int keep_B = 0;
};

// ---- layer types (dispatch in convl.cu) ------------------------------------------------------------------
// A block of device (max|x|, 1/scale) pairs: the power-of-two scales of one net's FP16-split operands (option mma_f16).
// The owner takes one pair per operand at alloc and resets the block at the start of each of its passes.
struct ScalePairs {
  float* base = nullptr;
  int n = 0, used = 0;
  int alloc(fg_ctx* c, std::vector<void*>& allocs, int pairs);
  int take(float** pair);  // the next pair; an error when the block is full
  // with the FP16 split only: zero the max words, which producers reduce into by atomicMax (AmaxInto).  The inverse
  // scales stay: the weight gradients of a later pass still read them.
  int reset(fg_ctx* c) const;
};

// One tensor-core operand: the hi/lo split of a tensor and its device (max|x|, 1/scale) pair.  Each buffer is sized for
// the 3xTF32 split; the 3xFP16 split uses its first half.  A producer kernel that already did part of the work says so:
//   split_ready  it wrote the TF32 split into hi/lo (3xTF32 path)
//   amax_ready   it reduced max|x| into s[0] (3xFP16 path; AmaxInto in convl.h)
//   bias_ready   it added the bias gradient (the column sums of a dY) into the gradient (ConvLEnv::dy only)
// The consuming layer then skips that pass and clears the flag.
struct TcOp {
  float *hi = nullptr, *lo = nullptr;
  float* s = nullptr;
  bool split_ready = false, amax_ready = false, bias_ready = false;
};
struct ConvL {  // NHWC, stride 1, "same" padding (a strided layer runs at stride 1 and is subsampled by its net)
  int Cin = 0, Cout = 0, k = 1, H = 1;
  int64_t w_off = 0, b_off = 0;
  int cA = 0, cS = 0;  // Linear after View([C][H][W]): column j=c*S+s of the reference <-> our NHWC column s*A+c
  int nA = 0, nS = 0;  // Linear before View([C][H][W]): the same permutation on the output rows (weights, bias, gradients)
  float *Wp = nullptr, *Wpd = nullptr;                                            // fp32 packs [t][n][c], [t'][c][n]
  float* bp = nullptr;                                                            // bias in our row order (nA != 0)
  float *Wf_hi = nullptr, *Wf_lo = nullptr, *Wd_hi = nullptr, *Wd_lo = nullptr;   // TF32 splits of the packs
  TcOp x;                    // split of the input (fwd -> wgrad); x.s may be set before convl_alloc
  float* sdy = nullptr;      // (max|dY|, 1/scale) of this layer's dY split; nullptr: the shared ConvLEnv::dy.s
  // this layer's own dY split (a weight gradient on the wgrad stream still reads it while the next layer splits its
  // dY); nullptr: the shared ConvLEnv::dy.hi / lo
  float *dy_hi = nullptr, *dy_lo = nullptr;
  // kpad (Linear only): K zero-padded Cin -> kpad so that the layer runs on the tensor cores (xpad: [B][kpad] input,
  // Wpad: [Cout][kpad] weights, both with zero pad columns); its weight gradient needs Cout * (kpad + Cin) floats of ws
  int kpad = 0;
  float *xpad = nullptr, *Wpad = nullptr;
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
  ConvGeom geom_k(int B) const { return ConvGeom{B, H, H, kpad ? kpad : Cin, Cout, k, 1}; }  // the tensor-core shape
  ConvGeom geom_d(int B) const { return ConvGeom{B, H, H, Cout, Cin, k, 1}; }
};

struct UpsL {  // nn.SpatialUpSamplingNearest(2) -> 5x5 "same" convolution; H = output side
  int Cin = 0, Cout = 0, H = 0;
  int64_t w_off = 0, b_off = 0;
  float *Wp = nullptr, *Wpd = nullptr;                                            // fp32 tap-major packs (FFMA path)
  float *Wf_hi = nullptr, *Wf_lo = nullptr, *Wd_hi = nullptr, *Wd_lo = nullptr;   // phase-collapsed packs [36][..][..]
  float *Wx_hi = nullptr, *Wx_lo = nullptr;                                       // dense forward pack [25][n][c] (conv_impl 1)
  TcOp x;  // split of the low-res input (fwd -> wgrad); x.s may be set before upsl_alloc to keep the pair elsewhere
  // tb: timer of the merged weight-and-data-gradient launch (tc_conv_bwd_ups, option bwd_merge); nullptr: never merged
  const char *tf = "", *td = "", *tw = "", *tb = nullptr;
  ConvGeom geom(int B) const { return ConvGeom{B, H, H, Cin, Cout, 5, 2}; }
};

// what a layer needs from the net that owns it: the allocation list and the shared scratch buffers
struct ConvLEnv {
  fg_ctx* c = nullptr;
  int maxB = 0;
  std::vector<void*>* allocs = nullptr;
  float *ga = nullptr;  // padded forward output (pad_out layers): maxB * H*H * pad_out floats
  TcOp dy;              // split of the current dY (largest layer output); dy.s: (max|dY|, 1/scale) of its FP16 split
  TcOp pad;             // channel-padded split of dY (pad_out / pad_dy layers); scaled by dy.s
  float* ws = nullptr;  // packed weight-gradient workspace (largest layer)
  // the same for the weight gradients on fg_ctx::wgrad_stream; nullptr: a backward on this scratch stays on one stream
  float* ws_w = nullptr;
};

// What differs between the generator sizes, as data: the generator code never asks which net it serves
struct GenDesc {
  int side;            // 32 or 16; every size follows from it
  const char* prefix;  // of every timer name: "" keeps the 32x32 names that bench.py and profiles/ read
  int l1_kpad;         // ConvL::kpad of G.L1 (0: no padding, G.L1 stays on the FFMA kernels)
  bool bwd_merge;      // G.C1 / G.C2 name a merged-launch timer (UpsL::tb), so option bwd_merge may merge them
};

// The generator of models.lua at side S (create_G_decoder_upsampling32 / 16; gen.cu): Linear(100 -> 128 (S/4)^2) View
// PReLU | Up2 conv(128->256,5) BN PReLU | Up2 conv(256->128,5) BN PReLU | conv(128->C,3) Sigmoid
struct UpsGen {
  int S = 32, C = 3;
  GLayout gl;
  ConvL GL1, GC3;
  UpsL GU[2];                          // G.C1, G.C2
  ScalePairs pairs;                    // the scale pairs of every FP16 operand below
  float* sdz[2] = {nullptr, nullptr};  // ... among them those of G.C1 / G.C2's dz
  // activations and gradients (NHWC)
  float *noise = nullptr, *z0 = nullptr, *h0 = nullptr, *z1 = nullptr, *h1 = nullptr, *z2 = nullptr, *h2 = nullptr,
        *z3 = nullptr, *y = nullptr;
  float *dz3 = nullptr, *dfull = nullptr, *dz2 = nullptr, *dz1 = nullptr, *dz0 = nullptr;
  float *bn_mean[2] = {nullptr, nullptr}, *bn_istd[2] = {nullptr, nullptr}, *bn_mg = nullptr;
  int B = 0;
  bool train = true, valid = false;
  UpsGen* owner = nullptr;  // a forward-only instance (gen_alloc_fwd): the instance whose weight packs it reads
  std::deque<std::string> names;  // prefixed timer names (stable storage: the layers point into it)
  const char *t_bn2_finalize = nullptr, *t_bn2_stats = nullptr, *t_bn2_apply = nullptr, *t_bn2_bwd_reduce = nullptr,
             *t_bn2_bwd_apply = nullptr;
};

struct TimerRec {
  double ms = 0;
  int64_t launches = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
};

// the staging buffers of the stacked inputs of a multi-iteration step: one device buffer per input kind, grown on
// demand (the old buffer is released, so a grown buffer gets a new address and with it a new graph key)
struct IterStage {
  float* p[8] = {};
  size_t cap[8] = {};
  int reserve(fg_ctx* c, std::vector<void*>& allocs, int k, size_t n);
  // *out = the n floats at p on the device: p itself (device memory or null), else buffer k (at least `cap_n` floats)
  // after an async copy
  int in(fg_ctx* c, std::vector<void*>& allocs, int k, const float* p, size_t n, size_t cap_n, const float** out);
};

struct Net32;  // the 32x32 nets (nets.cu)

// What every net on one device stream shares: the stream, the options, the data-parallel state and the workspaces of
// the kernels.  Each net owns its own parameters, activations and layer scratch.
struct JpegEncScratch;
struct fg_ctx {
  int device = 0, maxB = 0, C = 3;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  int64_t launches = 0;
  int conv_impl = FG_CONV_TC_COLLAPSED;  // default: wgmma path; FG_CONV_SIMT is the fp32 FFMA cross-check
  int sm_count = 132;
  // OPT.D_optmethod / OPT.G_optmethod (train.lua:38-39): FG_OPT_ADAM | FG_OPT_ADAGRAD | FG_OPT_SGD, and SGD momentum
  int opt_D = 0, opt_G = 0;
  float sgd_mom_D = 0.f, sgd_mom_G = 0.f;
  std::vector<void*> allocs;  // the workspaces below, allocated by fg_create
  Net32* n32 = nullptr;       // allocated by fg_create too, freed by fg_destroy before the workspaces
  float* small_ws = nullptr;  // per-block partials of the small-channel wgrad (k_conv_small.cu)
  // Cross-block sums are never accumulated with float / double atomics, whose order varies from run to run: split-K
  // weight gradients write one partial per split into splitk_ws and k_splitk_reduce adds them in split order; the
  // reduction kernels write one row of partials per block into red_ws and the last block to finish (red_ticket)
  // adds the rows in block order (k_ordered.cuh).  A step is bit-reproducible given its inputs and seed.
  float* splitk_ws = nullptr;
  size_t splitk_ws_elems = 0;
  double* red_ws = nullptr;
  size_t red_ws_elems = 0;
  double* red_ws_opt = nullptr;  // [kOptRedRows]: the penalty-loss sum of the optimizer, which may run on comm_stream
  unsigned* red_ticket = nullptr;  // [0]: red_ws, [1]: red_ws_opt
  // workspaces of the BatchNorm kernels, shared by the generators on this ctx's stream
  double* bn_slice_acc = nullptr;  // workspace of k_bn_finalize_parts: 32 slices x 4 x 256 doubles + tickets
  float* bn_parts = nullptr;  // [m-tile][3][C] BatchNorm partials written by the tensor-core conv epilogue
  int edge_impl = 1;          // option "edge_impl": 0 = the round-1 small-channel kernels (k_conv_small.cu) for G.C3 / D.C1
  int bn_epilogue = 1;        // option "bn_epilogue": 0 = separate statistics pass over z (the round-1 path)
  int mma_f16 = 1;            // option "mma_f16": 1 (default) = tensor-core operands in the 3xFP16 split (f16 MMAs); 0 = 3xTF32
  float* lop_sx = nullptr;  // (max|x|, 1/scale) pair of the L-op convolutions' FP16-split input (lop.cu) ...
  float* lop_sy = nullptr;  // ... and of their dY
  unsigned* amax_out = nullptr;  // when set (AmaxInto, convl.h), the next elementwise producer also reduces max|output| there ...
  bool* amax_done = nullptr;     // ... and sets *amax_done (a TcOp's amax_ready): its consumer skips its own reduction
  double* bn_acc = nullptr;  // [4][256] double accumulators (sum, sumsq / sum g, sum g xhat)
  float* io_dev = nullptr;  // device staging for NCHW images / misc
  size_t io_dev_elems = 0;
  JpegEncScratch* jpeg_enc = nullptr;  // fg_jpeg_encode's chunk buffers (jpeg_enc.cu), made on first use
  // option "jpeg_route" (tests only): the entropy coder of every JPEG encode on this ctx; 0 (default) = by the blocks
  // per file, 1 = one CTA per file, 2 = many CTAs per file.  The bytes are the same.
  int jpeg_route = 0;
  float* scratch[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t scratch_elems[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // data parallel
  void* nccl_comm = nullptr;
  int world = 1, rank = 0;
  // option "dp_overlap" (default 1): D's all-reduce + accuracy gate + optimizer run on comm_stream while the compute
  // stream already runs the G step's G forward (which only needs G's parameters); joined before D is used again
  int dp_overlap = 1;
  // SMs the persistent convolution kernels leave free while a collective, or the D iterations (step_body), run next
  // to them
  int reserve_sms = 0;
  // the convolution kernel launched last (fg_get_option "last_conv_*", include/fg_b200.h): FG_KERNEL_*, its tile, its
  // operand format (0 fp32 FFMA, 1 3xTF32, 2 3xFP16) and its K splits.  Set by the launchers where they choose the
  // kernel (note_conv), cleared on entry to every fg_conv2d_* / fg_scu_* / fg_linear_* call.  Host integers only.
  int last_conv_kind = 0, last_conv_tile_m = 0, last_conv_tile_n = 0, last_conv_format = 0, last_conv_splits = 0;
  // option "bwd_merge": the weight and data gradients of G's upsampled layers run as one persistent launch
  // (k_conv_tc.cu tc_conv_bwd_ups).  1 (default): where its schedule estimate beats two launches (tc_bwd_pair_pays:
  // G.C2 at batch 256, not G.C1); 2: wherever the shapes allow it; 0: two launches.  Option "bwd_merge_ctas"
  // (0 = one per SM) caps the CTAs of the merged launch.
  int bwd_merge = 1, bwd_merge_ctas = 0;
  int* bwd_claim = nullptr;  // the work-item counter of the merged launch
  // option "use_graph" (default 1): fg_train_step replays a captured CUDA graph of the step (launch overhead of ~200
  // kernels); keyed on everything a captured step bakes in, the seed is read from device memory
  int use_graph = 1, graph_epoch = 0;
  int64_t graph_launches = 0;  // steps run as a launch of a captured graph (fg_get_option "step_graph_launches")
  uint64_t* seed_dev = nullptr;
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // with one GPU the loop body (step_body) runs the first G iteration's generator forward on side_stream, next to the
  // D iterations.  side_ws holds a second copy of each workspace above that the generator forward's kernels use;
  // ctx_swap_side exchanges it and the stream with the context's own.
  cudaStream_t side_stream = nullptr;
  struct Workspaces {
    double* red_ws = nullptr;
    unsigned* red_ticket = nullptr;
    double *bn_acc = nullptr, *bn_slice_acc = nullptr;
    float* bn_parts = nullptr;
  } side_ws;
  // option "bwd_streams" (default 1): the backward of the 32x32 D and of G (D32::backward, gen_backward) enqueues the
  // weight gradients that nothing downstream reads before the optimizer on wgrad_stream, next to the data-gradient
  // chain on `stream` (OnWgradStream, convl.h); 0: one stream, in layer order.  wgrad_ws holds the stream's own copy of
  // each workspace a weight gradient writes; wgrad_forked: launches went there since the last wgrad_join.
  int bwd_streams = 1;
  cudaStream_t wgrad_stream = nullptr;
  cudaEvent_t ev_wfork = nullptr, ev_wjoin = nullptr;
  bool wgrad_forked = false;
  struct WgradWorkspaces {
    float* splitk_ws = nullptr;
    double* red_ws = nullptr;
    unsigned* red_ticket = nullptr;
    float* small_ws = nullptr;
  } wgrad_ws;
  // debug (tests): "debug_keep" = 1 keeps a copy of the D step's pre-activations of every train step (NetPair::keep),
  // which the G step's D forward overwrites (the strict gradient-parity tests read PReLU branch decisions from them)
  bool debug_keep = false;
  // timing
  cudaEvent_t events[16] = {};
  bool timing = false;
  std::map<std::string, TimerRec> timers;
};

// record the convolution kernel a launcher is about to run (fg_ctx::last_conv_*)
inline void note_conv(fg_ctx* c, int kind, int tile_m, int tile_n, int format, int splits) {
  c->last_conv_kind = kind;
  c->last_conv_tile_m = tile_m;
  c->last_conv_tile_n = tile_n;
  c->last_conv_format = format;
  c->last_conv_splits = splits;
}

struct ScopedTimer {
  fg_ctx* c;
  TimerRec* rec = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  ScopedTimer(fg_ctx* c_, const char* name) : c(c_) {  // name == nullptr: not timed
    if (c->timing && name) {
      rec = &c->timers[name];
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
      cudaEventRecord(e0, c->stream);
    }
  }
  ~ScopedTimer() {
    if (rec) {
      cudaEventRecord(e1, c->stream);
      rec->pending.emplace_back(e0, e1);
    }
  }
};

// ---- k_elem.cu -------------------------------------------------------------------------------------
int k_fill(fg_ctx* c, float* p, float v, int64_t n);
int k_nchw_to_nhwc(fg_ctx* c, const float* src, float* dst, int B, int C, int HW);
int k_nhwc_to_nchw(fg_ctx* c, const float* src, float* dst, int B, int C, int HW);
// weight packing: flat W[N][Cc][KK] -> fwd pack [t][n'][c'] and (optional) dgrad pack [KK-1-t][c'][n'].
// (nA,nS)/(cA,cS): index permutation j=a*S+s -> j'=s*A+a on rows / columns (0,0 = identity).
int k_pack_weights(fg_ctx* c, const float* W, float* Wp, float* Wpd, int N, int Cc, int KK, int nA, int nS, int cA,
                   int cS);
// grads: dW[n][c][t] += scale * dWp[t][n'][c']
int k_unpack_wgrad(fg_ctx* c, const float* dWp, float* dW, int N, int Cc, int KK, int nA, int nS, int cA, int cS);
int k_colsum_add(fg_ctx* c, const float* X, float* out, int64_t P, int N, int nA, int nS);  // out[perm^-1(n)] += sum_p X[p][n]
int k_prelu_fwd(fg_ctx* c, const float* z, const float* slope, float* h, int64_t n);
// dz = pool?(dh) * (z>0?1:a); *dslope += sum_{z<=0} dh*z.  pool: dh is [B][2H][2W][C] summed 2x2.
int k_prelu_bwd(fg_ctx* c, const float* dh, const float* z, const float* slope, float* dz, float* dslope, int B, int H,
                int W, int C, int pool);
int k_bn_stats(fg_ctx* c, const float* z, double* acc2C, int64_t P, int C);
bool k_bn4_ok(int C);  // k_bn.cu: float4, multi-row versions of the two BatchNorm reductions
int k_bn_stats4(fg_ctx* c, const float* z, double* acc, int64_t P, int C);
int k_bn_bwd_reduce4(fg_ctx* c, const float* dh, const float* z, const float* mean, const float* istd, const float* gamma,
                     const float* beta, const float* slope, double* acc, float* dslope, int64_t P, int C);
int k_bn_finalize(fg_ctx* c, double* acc2C, float* mean, float* istd, float* run_mean, float* run_var, int64_t P,
                  int C);
// statistics from the conv epilogue's per-tile partials (sum z, sum z^2, squared deviations from the tile mean) of a
// convolution with nphase output phases
int k_bn_finalize_parts(fg_ctx* c, const float* part, int nparts, int nphase, float* mean, float* istd, float* run_mean,
                        float* run_var, int64_t P, int C);
int k_bn_eval_prep(fg_ctx* c, const float* run_mean, const float* run_var, float* mean, float* istd, int C);
int k_bn_prelu_apply(fg_ctx* c, const float* z, const float* mean, const float* istd, const float* gamma,
                     const float* beta, const float* slope, float* h, int64_t P, int C, float* hi = nullptr,
                     float* lo = nullptr);  // h may be nullptr when only the TF32 hi/lo split is wanted
int k_bn_prelu_bwd_reduce(fg_ctx* c, const float* dh, const float* z, const float* mean, const float* istd,
                          const float* gamma, const float* beta, const float* slope, double* acc2C, float* dslope,
                          int B, int H, int W, int C, int pool);
int k_bn_bwd_finalize(fg_ctx* c, double* acc2C, float* mg2C, float* dgamma, float* dbeta, int64_t P, int C);
int k_bn_prelu_bwd_apply(fg_ctx* c, const float* dh, const float* z, const float* mean, const float* istd,
                         const float* gamma, const float* beta, const float* slope, const float* mg2C, float* dz,
                         int B, int H, int W, int C, int pool, float* hi = nullptr, float* lo = nullptr,
                         float* dbias = nullptr);  // dbias: += column sums of dz (bias gradient of the conv in front)
int k_sigmoid_fwd(fg_ctx* c, const float* z, float* y, int64_t n);
int k_sigmoid_bwd(fg_ctx* c, const float* dy, const float* y, float* dz, int64_t n);
int k_masks_generate(fg_ctx* c, float* masks, int B, uint64_t seed, float p_spatial, float p_drop,
                     const uint64_t* seed_dev = nullptr);  // seed_dev: effective seed = *seed_dev * 2 + seed
int k_set_u64(fg_ctx* c, uint64_t* dst, uint64_t v);
// roots[j] = 2^60 | roots[0] << 8 | j for 1 <= j < n: the stream root of iteration j of a multi-iteration step
// (fg_b200.h, "Several D and G iterations per call"); roots[0] is the step seed
int k_seed_roots(fg_ctx* c, uint64_t* roots, int n);
// hi / lo (optional): also emit the TF32 split of the result (16-byte aligned buffers of the output's size)
int k_d_act_pool_fwd(fg_ctx* c, const float* z, const float* slope, const float* masks, int moff, float eval_scale,
                     float* p, int B, int H, int W, int C, float* hi = nullptr, float* lo = nullptr);
int k_d_act_pool_bwd(fg_ctx* c, const float* dp, const float* z, const float* slope, const float* masks, int moff,
                     float eval_scale, float* dz, float* dslope, int B, int H, int W, int C, float* hi = nullptr,
                     float* lo = nullptr, float* dbias = nullptr);  // dbias: += column sums of dz (conv bias gradient)
int k_lin_act_drop_fwd(fg_ctx* c, const float* z, const float* slope, const float* masks, int moff, float scale,
                       float* h, int B, int N);
int k_lin_act_drop_bwd(fg_ctx* c, const float* dh, const float* z, const float* slope, const float* masks, int moff,
                       float scale, float* dz, float* dslope, int B, int N);
// out=sigmoid(logit); loss (mean BCE) -> *loss_out; dlogit = bce_grad*y(1-y); targets: first n_ones are 1.
// conf (may be null) gets [pred1&t1, pred0&t1, pred1&t0, pred0&t0] as floats in tail4 (for the DP allreduce)
int k_sigmoid_bce(fg_ctx* c, const float* logit, float* out, float* dlogit, float* loss_out, float* tail4, int B,
                  int n_ones);
int k_bce_fwd(fg_ctx* c, const float* x, const float* t, int n, float* loss_out);
int k_bce_bwd(fg_ctx* c, const float* x, const float* t, int n, float* dx);
int k_sigmoid_grad_mul(fg_ctx* c, const float* dout, const float* out, float* dlogit, int n);
// optimizer
int k_penalty_loss(fg_ctx* c, const float* p, int64_t n, float l1, float l2, float* loss_inout);
// accumulate: conf and trained_D add to the values of the earlier D iterations of the same step instead of replacing them
int k_gate_and_prep(fg_ctx* c, DeviceStats* st, float* acc_hist, int net, const fg_hyper* h, const float* tail4, int B,
                    float world, bool accumulate = false);
// no gate: t += 1 and the step size of `net` for its update rule (fg_optim_step); the accuracy state is left alone
int k_optim_prep(fg_ctx* c, DeviceStats* st, int net, const fg_hyper* h);
int k_gemv_fwd(fg_ctx* c, const float* x, const float* w, const float* bias, float* out, int B, int K);
int k_gemv_dgrad(fg_ctx* c, const float* dy, const float* w, float* dx, int B, int K);
int k_gemv_wgrad_add(fg_ctx* c, const float* x, const float* dy, float* dw, float* db, int B, int K);
int k_adam(fg_ctx* c, float* p, const float* g, float* m, float* v, int64_t n, float beta1, float beta2, float eps,
           float l1_grad, float l2, float clampv, float grad_scale, const float* step_dev, const int* flag_dev,
           float step_host, float* g_out);
// same pass with the update rule selected: mode FG_OPT_ADAM (as k_adam) | FG_OPT_ADAGRAD (variance in v) |
// FG_OPT_SGD (momentum buffer in m, `mom` = momentum = dampening; *t_dev == 1 marks the first step)
int k_optim_update(fg_ctx* c, int mode, float* p, float* g, float* m, float* v, int64_t n, float beta1, float beta2, float eps,
                   float mom, float l1_grad, float l2, float clampv, float grad_scale, const float* step_dev,
                   const int* flag_dev, const int* t_dev);

// ---- k_conv_simt.cu --------------------------------------------------------------------------------
// out[p][n] = bias[n] + sum_{t,c} in[pix(p,t)][c] * Wp[t][n][c]
int k_conv_simt(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, ConvGeom g);
// dWp[t][n][c] = sum_p dY[p][n] * in[pix(p,t)][c]   (dWp is overwritten)
int k_wgrad_simt(fg_ctx* c, const float* in, const float* dY, float* dWp, ConvGeom g);
// ---- k_conv_small.cu: 3-channel-side convolutions (G.C3, D.C1), bandwidth-shaped --------------------
bool k_small_eligible(const ConvGeom& g);
int k_conv_small(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, ConvGeom g);
int k_wgrad_small(fg_ctx* c, const float* in, const float* dY, float* dWp, ConvGeom g);

// ---- k_conv_edge.cu: the same layers at width 32, weights in registers, TMA / smem staged (the default) ----------
bool k_edge_eligible(const ConvGeom& g);
int k_conv_edge(fg_ctx* c, const float* in, const float* Wp, const float* bias, float* out, ConvGeom g);

// the ordered reductions of one launch need rows x n doubles of red_ws
inline int red_check(fg_ctx* c, int64_t rows, int64_t n) {
  if (rows * n > (int64_t)c->red_ws_elems) {
    fg_set_error("ordered reduction of %lld x %lld partials exceeds its workspace", (long long)rows, (long long)n);
    return FG_ERR_UNSUPPORTED;
  }
  return FG_OK;
}
// out[i] = sum over s in order of parts[s * n + i]  (split-K partials of a weight gradient, k_misc.cu)
int k_splitk_reduce(fg_ctx* c, const float* parts, int splits, int64_t n, float* out);

// ---- k_conv_tc.cu ----------------------------------------------------------------------------------
int tc_init(fg_ctx* c);
void tc_destroy(fg_ctx* c);

// ---- nets.cu: the 32x32 nets of fg_ctx::n32 ---------------------------------------------------------
int net32_alloc(fg_ctx* c, int disc);  // disc: FG_DISC_D32B or a branched D at side 32 (nets_dbr.cu)
void net32_free(fg_ctx* c);
NetPair& net32_pair(fg_ctx* c);  // their trainable state

// ---- dp.cu ------------------------------------------------------------------------------------------
int net_allreduce(fg_ctx* c, float* buf, int64_t n);
int net_broadcast(fg_ctx* c, void* buf, size_t bytes);  // rank 0 -> all
int net_group(bool start);                                // ncclGroupStart / ncclGroupEnd

// ---- netpair.cu: the lifecycle of a NetPair, on the ctx stream.  `net` is FG_NET_G or FG_NET_D (anything else: G) ----
// zero-filled device buffer of n floats (at least one), released by whoever owns `allocs`
int fg_dalloc(fg_ctx* c, std::vector<void*>& allocs, float** p, size_t n);
// parameters, gradients (+ tails), moments, statistics, accuracy history and, with `bn`, BatchNorm running statistics
// initialised as nn.SpatialBatchNormalization does (mean 0, var 1)
int pair_alloc(fg_ctx* c, std::vector<void*>& allocs, NetPair& p, int64_t nG, int64_t nD, bool bn);
void pair_clear_graphs(NetPair& p);
void pair_free(NetPair& p);  // graphs and the pinned mirror; the device buffers belong to `allocs`
int pair_zero_grads(fg_ctx* c, NetPair& p, int net);       // GRAD_PARAMETERS_x:zero() incl. the tail scalars
int pair_allreduce_grads(fg_ctx* c, NetPair& p, int net);  // gradient + tail (one call when contiguous); world 1: nothing
// the accuracy gate (D), t += 1 and the step size of `net` on the pair's own statistics
int pair_gate(fg_ctx* c, NetPair& p, int net, const fg_hyper* h, int B, float world, bool accumulate = false);
int pair_optim(fg_ctx* c, NetPair& p, int net, const fg_hyper* h, float grad_scale);  // penalty -> clamp -> update
// stock optim.adam without a gate: *t_dev += 1, *step_dev = lr sqrt(1 - beta2^t) / (1 - beta1^t) in double, for the
// k_optim_update that follows
int k_adam_prep(fg_ctx* c, int* t_dev, float* step_dev, float lr, float beta1, float beta2);
int pair_broadcast(fg_ctx* c, NetPair& p);  // rank 0's parameters, moments, BatchNorm state, statistics, history
int pair_step_stats(fg_ctx* c, const NetPair& p, fg_step_stats* stats);  // synchronise, then the last step's statistics
int pair_set_params(fg_ctx* c, NetPair& p, int net, const float* src);
int pair_get_params(fg_ctx* c, const NetPair& p, int net, float* dst);
int pair_get_grads(fg_ctx* c, const NetPair& p, int net, float* dst);
int pair_set_adam_state(fg_ctx* c, NetPair& p, int net, const float* m, const float* v, int t);
int pair_get_adam_state(fg_ctx* c, const NetPair& p, int net, float* m, float* v, int* t);
int pair_set_bn_state(fg_ctx* c, NetPair& p, const float* src);
int pair_get_bn_state(fg_ctx* c, const NetPair& p, float* dst);
// Runs `body` (launches on c->stream that read their seed from c->seed_dev) as a train step of pair p: eagerly, or as a
// captured CUDA graph keyed on B, the hyper-parameter struct's bytes, `inputs`, the stream, the communicator,
// graph_epoch, pack_key and the iteration counts nd / ng
int net_graph_run(fg_ctx* c, NetPair& p, int B, const void* hyper, size_t hyper_bytes, std::initializer_list<const void*> inputs,
                  uint64_t seed, const std::function<int()>& body, int nd = 1, int ng = 1);

// ---- the adversarial.lua loop body (adversarial_c2f.lua for the coarse-to-fine nets), netpair.cu ----
// the checks of a train-step entry `what`, made before it stages anything: the iteration counts (1 <= nd, ng <=
// kMaxIters, else FG_ERR_UNSUPPORTED), the feeding dataset d when `fed`, the inputs (`inputs`: none is null) and the batch
int step_check(fg_ctx* c, const char* what, int B, int nd, int ng, bool inputs, const fg_dataset* d = nullptr, bool fed = false);
// What one trainer contributes to the loop body: the calls on its nets and its D's output buffers.  It holds its own
// inputs (device pointers, stacked per iteration).
struct StepNets {
  StepNets(fg_ctx* c, NetPair& pair, const fg_hyper* h, int B, float* logit, float* out, float* dlogit, float* masks,
           int64_t mask, bool gate, bool overlap)
      : c(c), pair(&pair), h(h), B(B), logit(logit), out(out), dlogit(dlogit), masks(masks), mask(mask), gate(gate),
        overlap(overlap) {}
  fg_ctx* c;
  NetPair* pair;
  const fg_hyper* h;
  int B;
  float *logit, *out, *dlogit;  // D's output buffers
  float* masks;                 // D's dropout keep flags, `mask` floats per sample
  int64_t mask;
  bool gate;     // the accuracy gate decides whether D trains; false: it always does (adversarial_c2f.lua)
  bool overlap;  // option dp_overlap may run D's all-reduce, gate and optimizer next to the following G forward
  // the D iterations take their fakes from a generator of their own, so the first G iteration's generator forward
  // may run next to the last D iteration's D forward, backward and update (step_body)
  virtual bool g_side() const { return false; }
  // G in training mode: the B/2 fakes of D iteration j (d_iter), or the B samples of G iteration j; with the
  // condition rows D reads next, if any
  virtual int g_forward(int j, bool d_iter) = 0;
  virtual int d_input(int j) = 0;                              // D's input of D iteration j: the real half, then the fakes
  virtual int draw_masks(int kind, const uint64_t* root) = 0;  // D's keep flags of kind 1 (D iteration) or 2 (G iteration)
  virtual int d_forward(bool on_g) = 0;                        // D in training mode on its input, or on G's output
  virtual int d_backward(bool want_wgrad, bool want_dx) = 0;   // from dlogit
  virtual int g_backward() = 0;                                // from D's input gradient
};
// c->stream and the workspaces in c->side_ws change places with c->side_stream and the context's own (twice: back)
void ctx_swap_side(fg_ctx* c);
// nd D iterations, then ng G iterations, then the statistics to `stats` (may be null).  masksD / masksG (may be null:
// drawn from the stream root of each iteration) are stacked per iteration; feed (may be null) runs first inside the
// step, after the stream roots are set: a device-fed step draws its inputs there.  The step is keyed (net_graph_run) on
// `inputs`, which name every input pointer and what the feed reads.
int pair_train_step(StepNets& s, int nd, int ng, const float* masksD, const float* masksG, uint64_t seed,
                    std::initializer_list<const void*> inputs, const std::function<int()>* feed, fg_step_stats* stats);
// the "Dstep.*" rows of a debug-tensor table
struct DebugTensor;
void pair_keep_rows(const NetPair& p, std::vector<DebugTensor>& ents);

// ---- nets_ae.cu: the elementwise layers of the autoencoder (nn.ReLU, nn.Tanh + nn.Dropout, nn.AbsCriterion).  Each is
// a producer in AmaxInto's sense (convl.h). ----
int k_relu_fwd(fg_ctx* c, const float* z, float* h, int64_t n);
int k_relu_bwd(fg_ctx* c, const float* dh, const float* z, float* dz, int64_t n);  // dz = dh [z > 0]
// code = tanh(z), h (may be null) = Dropout(code): keep flags given (masks_in), drawn with probability 1 - p from
// *seed_dev, or none (both null: h = code); flags_out (may be null) receives the flags used
int k_tanh_dropout_fwd(fg_ctx* c, const float* z, const float* masks_in, const uint64_t* seed_dev, float p, float* code, float* h,
                       float* flags_out, int64_t n);
int k_tanh_dropout_bwd(fg_ctx* c, const float* dh, const float* masks, float p, const float* code, float* dz, int64_t n);
// mean |y - t| -> *loss and its gradient -> dz, with y = sigmoid(z) (also stored) and dz taken through Sigmoid.backward
// when `sigmoid`, else y = z; y, dz and loss may each be null
int k_abs_criterion(fg_ctx* c, bool sigmoid, const float* z, const float* t, float* y, float* dz, int64_t n, float* loss);

// ---- capi.cu: host or device pointers at the C ABI ----
bool fg_is_dev(const void* p);
// device pointer holding n floats of p: p itself when it is device memory, else `staging` after an async copy
int fg_to_dev(fg_ctx* c, const float* p, size_t n, float* staging, const float** out);
// n floats from a device buffer to a user pointer (host: synchronised, so valid on return; dst == src: nothing)
int fg_to_user(fg_ctx* c, float* dst, const float* src_dev, size_t n);
// the fg_*debug_tensor contract over a table of named device tensors (per * B floats each; p == nullptr: not produced
// yet): dst == nullptr -> the element count; -2: dst too small; -1 + fg_last_error: unknown or not produced
struct DebugTensor {
  const char* name;
  const float* p;
  int64_t per;
  int B;
};
int64_t debug_tensor_copy(fg_ctx* c, const char* what, const DebugTensor* ents, size_t n_ents, const char* name, float* dst,
                          int64_t max_elems);

// ---- dataset.cu / jpeg.cu: the device-resident dataset ----
struct JpegScratch;                     // fg_dataset_upload_jpeg's chunk buffers (jpeg.cu), made on first use
void jpeg_scratch_free(JpegScratch* s);
struct JpegEncScratch;                  // fg_dataset_encode_jpeg / fg_dataset_jpeg_roundtrip's chunk buffers (jpeg_enc.cu)
void jpeg_enc_scratch_free(JpegEncScratch* s);
struct fg_dataset {
  fg_ctx* c = nullptr;
  int64_t N = 0;
  int Cs = 3, Hs = 64, Ws = 64;
  uint8_t* data = nullptr;  // [N][Cs][Hs][Ws]
  int32_t* idx = nullptr;   // [maxB] staging for host index lists / drawn indices
  JpegScratch* jpeg = nullptr;
  JpegEncScratch* jpeg_enc = nullptr;
};
// ---- dataset.cu: inputs of the device-fed --scale 16 / coarse-to-fine steps (launches on the ctx stream) ----
// root (optional): the stream is *root * kinds + seed, read on the device (a captured step replays with a new seed)
int dataset_check_feed(const fg_dataset* d, const fg_ctx* c, const char* what);  // same ctx, compatible channels
// out [B][C][size][size] (device) = gather at `size` of B indices drawn from stream `seed` (fg_dataset_draw)
int dataset_draw_gather(fg_dataset* d, uint64_t seed, int B, int size, float* out_dev, const uint64_t* root = nullptr,
                        uint64_t kinds = 0);
// fine / coarse / diff [B][C][S][S] (device, any may be null) = fg_dataset_gather_c2f_sized of B indices drawn from `seed`
int dataset_draw_gather_c2f(fg_dataset* d, uint64_t seed, int B, int fine_size, int coarse_size, float* fine, float* coarse,
                            float* diff, const uint64_t* root = nullptr, uint64_t kinds = 0);
// fg_noise_uniform into device memory
int noise_uniform_dev(fg_ctx* c, uint64_t seed, int64_t n, float* out_dev, const uint64_t* root = nullptr, uint64_t kinds = 0);
