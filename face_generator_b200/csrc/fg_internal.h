// Internal declarations shared by the translation units of libfg_b200.so.
// Everything on the device is NHWC fp32; the NCHW reference layouts exist only at the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <functional>
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

constexpr int kMaskPerSample = 1984;  // 64+128+256+512 SpatialDropout + 512+512 Dropout keep flags
constexpr int kNoiseDim = 100;
constexpr int kSmallMaxParts = 2048;  // partial rows of the small-channel wgrad workspace
constexpr int kGradTail = 8;
constexpr int kOptRedRows = 132 * 2;  // blocks of the penalty-loss reduction          // extra floats behind each flat gradient (DP-reduced scalars)

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
struct DLayout {
  int64_t cW[4], cb[4], ca[4], L1W, L1b, a5, L2W, L2b, a6, L3W, L3b, total;
};
GLayout make_g_layout(int C);
DLayout make_d_layout(int C);

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

struct TimerRec {
  double ms = 0;
  int64_t launches = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
};

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
  GLayout gl;
  DLayout dl;
  std::vector<void*> allocs;  // every cudaMalloc of net_alloc(), released by net_free()
  // flat buffers (owned)
  float *PG = nullptr, *PD = nullptr, *gG = nullptr, *gD = nullptr;
  // the library's own allocations (PG.. point here unless fg_bind_params borrowed caller-owned buffers) and the 8
  // DP-reduced scalars behind each gradient: contiguous with the own gradient buffer, separate for a bound one
  float *ownPG = nullptr, *ownPD = nullptr, *ownGG = nullptr, *ownGD = nullptr;
  float *tailG = nullptr, *tailD = nullptr, *tail_sep = nullptr;
  float *mG = nullptr, *vG = nullptr, *mD = nullptr, *vD = nullptr;
  float* bnG = nullptr;  // [768] running stats
  DeviceStats* dstats = nullptr;
  float* acc_hist = nullptr;  // [kAccHistMax]
  DeviceStats* hstats = nullptr;  // pinned mirror
  // packed weights (forward packs [tap][n][c], dgrad packs [tap'][c][n])
  float *G_L1p = nullptr, *G_L1pd = nullptr, *G_C1p = nullptr, *G_C1pd = nullptr, *G_C2p = nullptr, *G_C2pd = nullptr,
        *G_C3p = nullptr, *G_C3pd = nullptr;
  float *D_cp[4] = {nullptr, nullptr, nullptr, nullptr}, *D_cpd[4] = {nullptr, nullptr, nullptr, nullptr};
  float *D_L1p = nullptr, *D_L1pd = nullptr, *D_L2pd = nullptr, *D_L3pd = nullptr;
  bool G_packed = false, D_packed = false;
  float* small_ws = nullptr;  // per-block partials of the small-channel wgrad (k_conv_small.cu)
  float* wgrad_ws = nullptr;  // packed weight-gradient workspace (largest layer)
  size_t wgrad_ws_elems = 0;
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
  // G activations (NHWC)
  int G_B = 0;
  bool G_train = true, G_fwd_valid = false;
  float *G_noise = nullptr, *G_z0 = nullptr, *G_h0 = nullptr, *G_z1 = nullptr, *G_h1 = nullptr, *G_z2 = nullptr,
        *G_h2 = nullptr, *G_z3 = nullptr, *G_y = nullptr;
  double* bn_slice_acc = nullptr;  // workspace of k_bn_finalize_parts: 32 slices x 2 x 256 doubles + tickets
  float* bn_parts = nullptr;  // [m-tile][2][C] BatchNorm partials written by the tensor-core conv epilogue
  int edge_impl = 1;          // option "edge_impl": 0 = the round-1 small-channel kernels (k_conv_small.cu) for G.C3 / D.C1
  int bn_epilogue = 1;        // option "bn_epilogue": 0 = separate statistics pass over z (the round-1 path)
  int mma_f16 = 1;            // option "mma_f16": 1 (default) = tensor-core operands in the 3xFP16 split (f16 MMAs); 0 = 3xTF32
  float* amax_slot = nullptr; // [32] (max|x|, 1/scale) pairs on the device: power-of-two scales of the FP16-split operands
  unsigned* amax_out = nullptr;  // when set (nets.cu AmaxInto), the next elementwise producer also reduces max|output| there ...
  int amax_id = 0;               // ... and marks amax_valid[amax_id]: split_h_scaled then skips its own reduction pass
  bool amax_valid[32] = {};
  double* bn_acc = nullptr;  // [4][256] double accumulators (sum, sumsq / sum g, sum g xhat)
  float *bn_mean1 = nullptr, *bn_istd1 = nullptr, *bn_mean2 = nullptr, *bn_istd2 = nullptr, *bn_mg = nullptr;
  float *G_dz3 = nullptr, *G_dfull = nullptr, *G_dz2 = nullptr, *G_dz1 = nullptr, *G_dz0 = nullptr;
  // D activations (NHWC)
  int D_B = 0;
  bool D_train = true, D_fwd_valid = false;
  float *D_x = nullptr, *D_z[4] = {nullptr, nullptr, nullptr, nullptr}, *D_p[4] = {nullptr, nullptr, nullptr, nullptr};
  float *D_zl1 = nullptr, *D_hl1 = nullptr, *D_zl2 = nullptr, *D_hl2 = nullptr, *D_logit = nullptr, *D_out = nullptr;
  float* D_masks = nullptr;
  float D_drop_scale = 2.0f, D_spatial_eval = 0.8f;  // 1/(1-p_drop), 1-p_spatial of the last forward
  float *D_dlogit = nullptr, *D_dh = nullptr, *D_dzl = nullptr, *D_dz = nullptr, *D_dp = nullptr, *D_dx = nullptr;
  float* D_targets = nullptr;
  // staging
  float* stage_pinned = nullptr;
  size_t stage_pinned_bytes = 0;
  float* io_dev = nullptr;  // device staging for NCHW images / misc
  size_t io_dev_elems = 0;
  float* io_dev2 = nullptr;
  float *in_real = nullptr, *in_noiseD = nullptr, *in_noiseG = nullptr, *in_masksD = nullptr, *in_masksG = nullptr;
  float* scratch[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t scratch_elems[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // data parallel
  void* nccl_comm = nullptr;
  int world = 1, rank = 0;
  // option "dp_overlap" (default 1): D's all-reduce + accuracy gate + optimizer run on comm_stream while the compute
  // stream already runs the G step's G forward (which only needs G's parameters); joined before D is used again
  int dp_overlap = 1;
  int reserve_sms = 0;  // SMs the persistent convolution kernels leave free while a collective runs next to them
  // option "use_graph" (default 1): fg_train_step replays a captured CUDA graph of the step (launch overhead of ~200
  // kernels); keyed on everything a captured step bakes in, the seed is read from device memory
  int use_graph = 1, graph_epoch = 0;
  uint64_t* seed_dev = nullptr;
  struct StepGraph {
    std::vector<uint8_t> key;
    cudaGraphExec_t exec = nullptr;
    int64_t launches = 0;
    bool failed = false;
  };
  std::vector<StepGraph> graphs;
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // debug (tests): "debug_keep" = 1 keeps a copy of the D step's pre-activations of fg_train_step, which the G
  // step's D forward overwrites (the strict gradient-parity tests read PReLU branch decisions from them)
  bool debug_keep = false;
  int keep_B = 0;
  float* keep_D[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // D_z[0..3], D_zl1, D_zl2, D_logit, D_out
  // timing
  cudaEvent_t events[16] = {};
  bool timing = false;
  std::map<std::string, TimerRec> timers;
  // tensor-core path: TF32 hi/lo splits of activations / gradients / packed weights (k_conv_tc.cu)
  struct TcBufs {
    float *G_h0_hi = nullptr, *G_h0_lo = nullptr, *G_h1_hi = nullptr, *G_h1_lo = nullptr;  // conv inputs (fwd -> wgrad)
    // G.L1 (nn.Linear 100 -> 8192, models.lua:59) as a 1x1 convolution with K padded 100 -> 128: zero-padded noise
    // [B][128] and its split, packed weights [8192'][128] (rows permuted for the View) and their split
    float *G_xpad = nullptr, *G_x_hi = nullptr, *G_x_lo = nullptr, *G_L1pad = nullptr, *G_L1w_hi = nullptr, *G_L1w_lo = nullptr;
    float *dy_hi = nullptr, *dy_lo = nullptr;                                             // current dY (dgrad + wgrad)
    float *G_Wf_hi[2] = {nullptr, nullptr}, *G_Wf_lo[2] = {nullptr, nullptr};  // C1,C2 collapsed fwd [36][n][c]
    float *G_Wd_hi[2] = {nullptr, nullptr}, *G_Wd_lo[2] = {nullptr, nullptr};  // collapsed dgrad [36][c][n]
    float *G_Wx_hi[2] = {nullptr, nullptr}, *G_Wx_lo[2] = {nullptr, nullptr};  // dense fwd [25][n][c]
    float *D_p_hi[3] = {nullptr, nullptr, nullptr}, *D_p_lo[3] = {nullptr, nullptr, nullptr};  // pooled inputs of c2..c4
    float *D_Wf_hi[4] = {nullptr, nullptr, nullptr, nullptr}, *D_Wf_lo[4] = {nullptr, nullptr, nullptr, nullptr};
    float *D_Wd_hi[4] = {nullptr, nullptr, nullptr, nullptr}, *D_Wd_lo[4] = {nullptr, nullptr, nullptr, nullptr};
    // D's Linear layers: [0] L1 fwd [512][2048'], [1] L1 dgrad [2048'][512], [2] L2 fwd, [3] L2 dgrad
    float *D_Lw_hi[4] = {nullptr, nullptr, nullptr, nullptr}, *D_Lw_lo[4] = {nullptr, nullptr, nullptr, nullptr};
    float *D_lin_hi[2] = {nullptr, nullptr}, *D_lin_lo[2] = {nullptr, nullptr};  // splits of p4 / hl1 kept for wgrad
    // 3xFP16 split twins (option mma_f16) of the K-major operands: n halves = n/2 floats per buffer
    float *G_h0_hh = nullptr, *G_h0_hl = nullptr, *G_h1_hh = nullptr, *G_h1_hl = nullptr, *dy_hh = nullptr, *dy_hl = nullptr;
    float *G_Wf_hh[2] = {nullptr, nullptr}, *G_Wf_hl[2] = {nullptr, nullptr}, *G_Wd_hh[2] = {nullptr, nullptr},
          *G_Wd_hl[2] = {nullptr, nullptr};
    float *D_p_hh[3] = {nullptr, nullptr, nullptr}, *D_p_hl[3] = {nullptr, nullptr, nullptr};
    float *D_Wf_hh[4] = {nullptr, nullptr, nullptr, nullptr}, *D_Wf_hl[4] = {nullptr, nullptr, nullptr, nullptr};
    float *D_Wd_hh[4] = {nullptr, nullptr, nullptr, nullptr}, *D_Wd_hl[4] = {nullptr, nullptr, nullptr, nullptr};
    float *G_x_hh = nullptr, *G_x_hl = nullptr, *G_L1w_hh = nullptr, *G_L1w_hl = nullptr;
    float *D_lin_hh[2] = {nullptr, nullptr}, *D_lin_hl[2] = {nullptr, nullptr};
    float *D_Lw_hh[4] = {nullptr, nullptr, nullptr, nullptr}, *D_Lw_hl[4] = {nullptr, nullptr, nullptr, nullptr};
  } tcb;
};

struct ScopedTimer {
  fg_ctx* c;
  TimerRec* rec = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  ScopedTimer(fg_ctx* c_, const char* name) : c(c_) {
    if (c->timing) {
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
int k_bn_finalize_parts(fg_ctx* c, const float* part, int nparts, float* mean, float* istd, float* run_mean, float* run_var,
                        int64_t P, int C);  // statistics from the conv epilogue's per-tile partials
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
int k_gate_and_prep(fg_ctx* c, int net, const fg_hyper* h, const float* tail4, int B, float world);
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

// ---- nets.cu ---------------------------------------------------------------------------------------
int net_alloc(fg_ctx* c);
void net_free(fg_ctx* c);
int net_pack_G(fg_ctx* c);
int net_pack_D(fg_ctx* c);
int net_G_forward(fg_ctx* c, const float* noise_dev, int B, bool training);                 // -> c->G_y (NHWC)
int net_G_backward(fg_ctx* c, const float* dy_nhwc, float* dnoise_dev);                      // accumulates c->gG
int net_D_forward(fg_ctx* c, const float* x_nhwc, int B, bool training, const fg_hyper* h);  // masks in c->D_masks
int net_D_backward(fg_ctx* c, const float* dlogit_dev, bool want_wgrad, bool want_dx);       // -> c->D_dx (NHWC)
int net_optim(fg_ctx* c, int net, const fg_hyper* h, float grad_scale, bool gate);
void net_graphs_clear(fg_ctx* c);
int net_graph_run(fg_ctx* c, std::vector<fg_ctx::StepGraph>& cache, const std::vector<uint8_t>& key, uint64_t seed,
                  const std::function<int()>& body, const std::function<void()>& repack, bool allow_graph);
int net_train_step(fg_ctx* c, const fg_hyper* h, int B, const float* real_nchw_dev, const float* noiseD_dev,
                   const float* noiseG_dev, const float* masksD_dev, const float* masksG_dev, uint64_t seed,
                   bool allow_graph = false);
int net_allreduce(fg_ctx* c, float* buf, int64_t n);
int net_zero_grads(fg_ctx* c, int net);
int net_allreduce_grads(fg_ctx* c, int net);  // flat gradient + its 8 tail scalars (one call when contiguous)
int net_broadcast(fg_ctx* c, void* buf, size_t bytes);  // rank 0 -> all (dp.cu)
int net_group(bool start);                                // ncclGroupStart / ncclGroupEnd
