// The 32x32 nets of train.lua and their C entry points: G (models.lua:57-81; gen.cu), D (models.lua:382-416) and their
// part of the adversarial.lua loop body (adversarial.lua:54-300; the loop itself is pair_train_step in netpair.cu) on
// one stream.  Kernels live in k_elem.cu / k_conv_simt.cu / k_conv_tc.cu.
#include <algorithm>

#include "convl.h"
#include "fg_internal.h"
#include "k_conv_tc.h"

namespace {
// Flat parameter layout of D (getParameters() order), float offsets
struct DLayout {
  int64_t cW[4], cb[4], ca[4], L1W, L1b, a5, L2W, L2b, a6, L3W, L3b, total;
};

DLayout make_d_layout(int C) {
  DLayout L;
  const int cin[4] = {C, 64, 128, 256}, cout[4] = {64, 128, 256, 512};
  int64_t o = 0;
  for (int i = 0; i < 4; ++i) {
    L.cW[i] = o; o += (int64_t)cout[i] * cin[i] * 9;
    L.cb[i] = o; o += cout[i];
    L.ca[i] = o; o += 1;
  }
  L.L1W = o; o += 512 * 2048;
  L.L1b = o; o += 512;
  L.a5 = o; o += 1;
  L.L2W = o; o += 512 * 512;
  L.L2b = o; o += 512;
  L.a6 = o; o += 1;
  L.L3W = o; o += 512;
  L.L3b = o; o += 1;
  L.total = o;
  return L;
}

const int kDcin[4] = {0 /*C*/, 64, 128, 256}, kDcout[4] = {64, 128, 256, 512}, kDhw[4] = {32, 16, 8, 4};
const int kDmoff[4] = {0, 64, 192, 448};
inline int dcin(const fg_ctx* c, int i) { return i == 0 ? c->C : kDcin[i]; }
}  // namespace

struct Net32 {
  fg_ctx* c = nullptr;
  NetPair net;
  // the library's own allocations (net.PG.. point here unless fg_bind_params borrowed caller-owned buffers) and the 8
  // DP-reduced scalars behind a bound gradient (behind the own gradient buffer they are contiguous with it)
  float *ownPG = nullptr, *ownPD = nullptr, *ownGG = nullptr, *ownGD = nullptr;
  float* tail_sep = nullptr;
  UpsGen G;
  // the layers of D (D.L3 runs on the GEMV kernels); D's FP16 scale pairs, env.dy's included, live in D_pairs
  DLayout dl;
  ConvL Dc[4], DL1, DL2;
  ScalePairs D_pairs;
  // D activations (NHWC)
  int D_B = 0;
  bool D_train = true, D_fwd_valid = false;
  float *D_x = nullptr, *D_z[4] = {nullptr, nullptr, nullptr, nullptr}, *D_p[4] = {nullptr, nullptr, nullptr, nullptr};
  float *D_zl1 = nullptr, *D_hl1 = nullptr, *D_zl2 = nullptr, *D_hl2 = nullptr, *D_logit = nullptr, *D_out = nullptr;
  float* D_masks = nullptr;
  float D_drop_scale = 2.0f, D_spatial_eval = 0.8f;  // 1/(1-p_drop), 1-p_spatial of the last forward
  float *D_dlogit = nullptr, *D_dh = nullptr, *D_dzl = nullptr, *D_dz = nullptr, *D_dp = nullptr, *D_dx = nullptr;
  float* D_targets = nullptr;
  // option "debug_keep" (tests): the backward reuses D_dh / D_dzl / D_dp / D_dz across layers, so D_backward copies
  // each one as a kernel wrote it ("Dbwd.*" debug tensors, the last D backward; Keep::src is unused here)
  std::vector<NetPair::Keep> bwd_keep;
  int bwd_keep_B = 0;
  // staging
  float* io_dev2 = nullptr;
  float *in_noiseD = nullptr, *in_noiseG = nullptr;
  IterStage iter_stage;  // the inputs of the host-fed and device-fed train steps, stacked per iteration
  std::vector<void*> allocs;
  // the scratch G's and D's layers share: env.dy is the split of the current dY, env.ws the packed weight-gradient
  // workspace (largest layer)
  ConvLEnv env;
};

namespace {
int dalloc(Net32* n, float** p, size_t elems) { return fg_dalloc(n->c, n->allocs, p, elems); }

int n32_alloc(Net32* n) {
  fg_ctx* c = n->c;
  const size_t B = c->maxB, C = c->C;
  n->dl = make_d_layout(c->C);
  NetPair& p = n->net;
  FG_TRY(pair_alloc(c, n->allocs, p, make_g_layout(c->C, 32).total, n->dl.total, true));
  p.optim_timer[0] = "hbm.optim.G";
  p.optim_timer[1] = "hbm.optim.D";
  n->ownPG = p.PG; n->ownPD = p.PD; n->ownGG = p.gG; n->ownGD = p.gD;
  FG_TRY(dalloc(n, &n->tail_sep, 2 * kGradTail));
  // the largest weight gradient: D.C4 / G's collapsed 5x5 layers; G.L1 on the tensor cores needs 8192 x (128 + 100)
  FG_TRY(dalloc(n, &n->env.ws, std::max<size_t>(9 * 512 * 256, 8192 * (128 + kNoiseDim))));
  // D activations
  FG_TRY(dalloc(n, &n->D_x, B * 1024 * C));
  for (int i = 0; i < 4; ++i) {
    const size_t e = B * (size_t)kDhw[i] * kDhw[i] * kDcout[i];
    FG_TRY(dalloc(n, &n->D_z[i], e));
    FG_TRY(dalloc(n, &n->D_p[i], e / 4));
  }
  FG_TRY(dalloc(n, &n->D_zl1, B * 512));
  FG_TRY(dalloc(n, &n->D_hl1, B * 512));
  FG_TRY(dalloc(n, &n->D_zl2, B * 512));
  FG_TRY(dalloc(n, &n->D_hl2, B * 512));
  FG_TRY(dalloc(n, &n->D_logit, B));
  FG_TRY(dalloc(n, &n->D_out, B));
  FG_TRY(dalloc(n, &n->D_masks, B * kMaskPerSample));
  FG_TRY(dalloc(n, &n->D_dlogit, B));
  FG_TRY(dalloc(n, &n->D_dh, B * 512));
  FG_TRY(dalloc(n, &n->D_dzl, B * 512));
  FG_TRY(dalloc(n, &n->D_dz, B * 65536));
  FG_TRY(dalloc(n, &n->D_dp, B * 16384));
  FG_TRY(dalloc(n, &n->D_dx, B * 1024 * C));
  FG_TRY(dalloc(n, &n->D_targets, B));
  FG_TRY(dalloc(n, &n->io_dev2, c->io_dev_elems));
  {  // the layers (convl.h) and the scratch they share
    ConvLEnv& e = n->env;
    e.c = c;
    e.maxB = c->maxB;
    e.allocs = &n->allocs;
    FG_TRY(dalloc(n, &e.dy.hi, B * 131072));
    FG_TRY(dalloc(n, &e.dy.lo, B * 131072));
    static const GenDesc g32{32, "", 128, true};  // G.L1 padded to K = 128 for the tensor cores; G.C1 / G.C2 may merge
    FG_TRY(gen_alloc(e, n->G, g32));
    ScalePairs& sp = n->D_pairs;  // every FP16-split operand of D gets its own scale pair
    FG_TRY(sp.alloc(c, n->allocs, 1 + 2 * 6));
    FG_TRY(sp.take(&e.dy.s));
    const DLayout& dl = n->dl;
    auto conv = [&](ConvL& L, int Cin, int Cout, int k, int H, int64_t w_off, int64_t b_off, const char* tf, const char* td,
                    const char* tw) {
      L.Cin = Cin; L.Cout = Cout; L.k = k; L.H = H;
      L.w_off = w_off; L.b_off = b_off;
      L.tf = tf; L.td = td; L.tw = tw;
    };
    static const char* tf[4] = {"D.C1.fwd", "D.C2.fwd", "D.C3.fwd", "D.C4.fwd"};
    static const char* td[4] = {"D.C1.dgrad", "D.C2.dgrad", "D.C3.dgrad", "D.C4.dgrad"};
    static const char* tw[4] = {"D.C1.wgrad", "D.C2.wgrad", "D.C3.wgrad", "D.C4.wgrad"};
    for (int i = 0; i < 4; ++i) conv(n->Dc[i], dcin(c, i), kDcout[i], 3, kDhw[i], dl.cW[i], dl.cb[i], tf[i], td[i], tw[i]);
    conv(n->DL1, 2048, 512, 1, 1, dl.L1W, dl.L1b, "D.L1.fwd", "D.L1.dgrad", "D.L1.wgrad");
    n->DL1.cA = 512; n->DL1.cS = 4;  // View(2048) flattens [512][2][2] in (c,h,w) order; ours is NHWC (h,w,c)
    conv(n->DL2, 512, 512, 1, 1, dl.L2W, dl.L2b, "D.L2.fwd", "D.L2.dgrad", "D.L2.wgrad");
    for (ConvL* L : {&n->Dc[0], &n->Dc[1], &n->Dc[2], &n->Dc[3], &n->DL1, &n->DL2}) {
      FG_TRY(sp.take(&L->x.s));
      FG_TRY(sp.take(&L->sdy));
      FG_TRY(convl_alloc(e, *L));
    }
  }
  FG_TRY(dalloc(n, &n->in_noiseD, B * kNoiseDim));
  FG_TRY(dalloc(n, &n->in_noiseG, B * kNoiseDim));
  p.keep = {{"Dstep.z1", n->D_z[0], 65536}, {"Dstep.z2", n->D_z[1], 32768}, {"Dstep.z3", n->D_z[2], 16384},
            {"Dstep.z4", n->D_z[3], 8192},  {"Dstep.zl1", n->D_zl1, 512},    {"Dstep.zl2", n->D_zl2, 512},
            {"Dstep.logit", n->D_logit, 1}, {"Dstep.out", n->D_out, 1}};
  n->bwd_keep = {{"Dbwd.dh3", nullptr, 512},    {"Dbwd.dzl2", nullptr, 512},  {"Dbwd.dh2", nullptr, 512},
                 {"Dbwd.dzl1", nullptr, 512},   {"Dbwd.dp4", nullptr, 2048},  {"Dbwd.dz4", nullptr, 8192},
                 {"Dbwd.dp3", nullptr, 4096},   {"Dbwd.dz3", nullptr, 16384}, {"Dbwd.dp2", nullptr, 8192},
                 {"Dbwd.dz2", nullptr, 32768},  {"Dbwd.dp1", nullptr, 16384}, {"Dbwd.dz1", nullptr, 65536}};
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int pack_D(Net32* n) {
  fg_ctx* c = n->c;
  if (n->net.D_pack == pack_key(c)) return FG_OK;
  for (int i = 0; i < 4; ++i) FG_TRY(convl_pack(c, n->Dc[i], n->net.PD));
  FG_TRY(convl_pack(c, n->DL1, n->net.PD));
  FG_TRY(convl_pack(c, n->DL2, n->net.PD));
  n->net.D_pack = pack_key(c);
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// D
// ---------------------------------------------------------------------------------------------------
// x: NHWC device [B][32][32][C]; keep flags already in D_masks when training
int D_forward(Net32* n, const float* x, int B, bool training, const fg_hyper* h) {
  fg_ctx* c = n->c;
  FG_REQUIRE(B >= 1 && B <= c->maxB, "D forward: batch %d out of range [1,%d]", B, c->maxB);
  FG_TRY(pack_D(n));
  FG_TRY(n->D_pairs.reset(c));
  const DLayout& L = n->dl;
  float* P = n->net.PD;
  if (x != n->D_x)
    FG_CUDA(cudaMemcpyAsync(n->D_x, x, sizeof(float) * (size_t)B * 1024 * c->C, cudaMemcpyDeviceToDevice, c->stream));
  n->D_B = B;
  n->D_train = training;
  const float* masks = training ? n->D_masks : nullptr;
  const float* cur = n->D_x;
  for (int i = 0; i < 4; ++i) {
    const int H = kDhw[i];
    FG_TRY(convl_fwd(n->env, n->Dc[i], cur, P, n->D_z[i], B));
    // the pooled activation is the next layer's tensor-core operand: its TF32 split (or max|p|) comes out of the same kernel
    TcOp& nx = (i < 3 ? n->Dc[i + 1] : n->DL1).x;
    nx.split_ready = convl_tc_fwd(c, i < 3 ? n->Dc[i + 1] : n->DL1) && !tc_f16(c);
    {
      AmaxInto am(c, nx);
      FG_TRY(k_d_act_pool_fwd(c, n->D_z[i], P + L.ca[i], masks, kDmoff[i], 1.0f - h->p_spatial, n->D_p[i], B, H, H,
                              kDcout[i], nx.split_ready ? nx.hi : nullptr, nx.split_ready ? nx.lo : nullptr));
    }
    cur = n->D_p[i];
  }
  const float scale = 1.0f / (1.0f - h->p_drop);
  n->D_drop_scale = scale;
  n->D_spatial_eval = 1.0f - h->p_spatial;
  FG_TRY(convl_fwd(n->env, n->DL1, n->D_p[3], P, n->D_zl1, B));
  {
    AmaxInto am(c, n->DL2.x);
    FG_TRY(k_lin_act_drop_fwd(c, n->D_zl1, P + L.a5, masks, 960, scale, n->D_hl1, B, 512));
  }
  FG_TRY(convl_fwd(n->env, n->DL2, n->D_hl1, P, n->D_zl2, B));
  FG_TRY(k_lin_act_drop_fwd(c, n->D_zl2, P + L.a6, masks, 1472, scale, n->D_hl2, B, 512));
  {
    ScopedTimer tm(c, "D.L3.fwd");
    FG_TRY(k_gemv_fwd(c, n->D_hl2, P + L.L3W, P + L.L3b, n->D_logit, B, 512));
  }
  n->D_fwd_valid = true;
  return FG_OK;
}

// option "debug_keep": bwd_keep[k].copy = the first B samples of src, bit for bit (allocated by the first use)
int keep_bwd(Net32* n, int k, const float* src, int B) {
  fg_ctx* c = n->c;
  if (!c->debug_keep) return FG_OK;
  NetPair::Keep& e = n->bwd_keep[k];
  if (!e.copy) FG_CUDA(cudaMalloc((void**)&e.copy, sizeof(float) * c->maxB * e.per));
  FG_CUDA(cudaMemcpyAsync(e.copy, src, sizeof(float) * B * e.per, cudaMemcpyDeviceToDevice, c->stream));
  n->bwd_keep_B = B;
  return FG_OK;
}

// dlogit [B]; want_dx: the image gradient into D_dx (NHWC)
int D_backward(Net32* n, const float* dlogit, bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  if (!n->D_fwd_valid) {
    fg_set_error("D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const DLayout& L = n->dl;
  float *P = n->net.PD, *G = n->net.gD;
  const int B = n->D_B;
  const float* masks = n->D_train ? n->D_masks : nullptr;
  const float scale = n->D_drop_scale, eval_scale = n->D_spatial_eval;
  FG_TRY(n->D_pairs.reset(c));
  // L3
  if (want_wgrad) {
    ScopedTimer tm(c, "D.L3.wgrad");
    FG_TRY(k_gemv_wgrad_add(c, n->D_hl2, dlogit, G + L.L3W, G + L.L3b, B, 512));
  }
  {
    ScopedTimer tm(c, "D.L3.dgrad");
    FG_TRY(k_gemv_dgrad(c, dlogit, P + L.L3W, n->D_dh, B, 512));
  }
  FG_TRY(keep_bwd(n, 0, n->D_dh, B));
  TcOp& dy = n->env.dy;  // the producers below say in its flags what they already did for the layer that follows
  float* GD = want_wgrad ? G : nullptr;
  {
    AmaxInto am(c, n->DL2.sdy, &dy.amax_ready);
    FG_TRY(k_lin_act_drop_bwd(c, n->D_dh, n->D_zl2, P + L.a6, masks, 1472, scale, n->D_dzl, want_wgrad ? G + L.a6 : nullptr, B,
                              512));
  }
  FG_TRY(keep_bwd(n, 1, n->D_dzl, B));
  FG_TRY(convl_bwd(n->env, n->DL2, n->D_hl1, n->D_dzl, GD, n->D_dh, B));
  FG_TRY(keep_bwd(n, 2, n->D_dh, B));
  {
    AmaxInto am(c, n->DL1.sdy, &dy.amax_ready);
    FG_TRY(k_lin_act_drop_bwd(c, n->D_dh, n->D_zl1, P + L.a5, masks, 960, scale, n->D_dzl, want_wgrad ? G + L.a5 : nullptr, B,
                              512));
  }
  FG_TRY(keep_bwd(n, 3, n->D_dzl, B));
  FG_TRY(convl_bwd(n->env, n->DL1, n->D_p[3], n->D_dzl, GD, n->D_dp, B));
  for (int i = 3; i >= 0; --i) {
    const int H = kDhw[i];
    FG_TRY(keep_bwd(n, 4 + 2 * (3 - i), n->D_dp, B));  // "Dbwd.dp<i+1>": the input of layer i's act/pool backward
    // dz and, for the tensor-core layers, its TF32 split in one pass, + the conv bias gradient (column sums of dz)
    dy.split_ready = convl_tc_bwd(c, n->Dc[i]) && !tc_f16(c);
    dy.bias_ready = want_wgrad;
    {
      AmaxInto am(c, n->Dc[i].sdy, &dy.amax_ready);
      FG_TRY(k_d_act_pool_bwd(c, n->D_dp, n->D_z[i], P + L.ca[i], masks, kDmoff[i], eval_scale, n->D_dz,
                              want_wgrad ? G + L.ca[i] : nullptr, B, H, H, kDcout[i], dy.split_ready ? dy.hi : nullptr,
                              dy.split_ready ? dy.lo : nullptr, want_wgrad ? G + L.cb[i] : nullptr));
    }
    FG_TRY(keep_bwd(n, 5 + 2 * (3 - i), n->D_dz, B));
    float* din = i > 0 ? n->D_dp : want_dx ? n->D_dx : nullptr;
    FG_TRY(convl_bwd(n->env, n->Dc[i], i == 0 ? n->D_x : n->D_p[i - 1], n->D_dz, GD, din, B));
  }
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// the 32x32 nets in the adversarial.lua loop body (pair_train_step, netpair.cu): real [B/2][C][32][32], noiseD [B/2][100]
// and noiseG [B][100] per iteration
// ---------------------------------------------------------------------------------------------------
struct NetStep final : StepNets {
  Net32* n;
  const float *real, *noiseD, *noiseG;
  NetStep(Net32* n, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG)
      : StepNets(n->c, n->net, h, B, n->D_logit, n->D_out, n->D_dlogit, n->D_masks, kMaskPerSample, true, true), n(n),
        real(real), noiseD(noiseD), noiseG(noiseG) {}
  int g_forward(int j, bool d_iter) override {
    const int rows = d_iter ? B / 2 : B;
    return gen_forward(n->env, n->G, n->net, (d_iter ? noiseD : noiseG) + (size_t)j * rows * kNoiseDim, rows, true);
  }
  int d_input(int j) override {
    const int Bh = B / 2;
    const size_t img = (size_t)c->C * 1024;
    FG_TRY(k_nchw_to_nhwc(c, real + (size_t)j * Bh * img, n->D_x, Bh, c->C, 1024));
    FG_CUDA(cudaMemcpyAsync(n->D_x + Bh * img, n->G.y, sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
    return FG_OK;
  }
  int draw_masks(int kind, const uint64_t* root) override {
    return k_masks_generate(c, n->D_masks, B, kind, h->p_spatial, h->p_drop, root);
  }
  int d_forward(bool on_g) override { return D_forward(n, on_g ? n->G.y : n->D_x, B, true, h); }
  int d_backward(bool want_wgrad, bool want_dx) override { return D_backward(n, n->D_dlogit, want_wgrad, want_dx); }
  int g_backward() override { return gen_backward(n->env, n->G, n->net, n->D_dx, nullptr); }
};
}  // namespace

int net32_alloc(fg_ctx* c) {
  c->n32 = new Net32();
  c->n32->c = c;
  return n32_alloc(c->n32);
}
void net32_free(fg_ctx* c) {
  Net32* n = c->n32;
  if (!n) return;
  pair_free(n->net);
  for (NetPair::Keep& k : n->bwd_keep)
    if (k.copy) cudaFree(k.copy);
  for (void* p : n->allocs) cudaFree(p);
  delete n;
  c->n32 = nullptr;
}
NetPair& net32_pair(fg_ctx* c) { return c->n32->net; }

#define ENTER(c)                                      \
  do {                                                \
    if (!(c)) {                                       \
      fg_set_error("null fg_ctx");                    \
      return FG_ERR_INVALID;                          \
    }                                                 \
    FG_CUDA(cudaSetDevice((c)->device));              \
  } while (0)

namespace {
// d_iters D iterations + g_iters G iterations of the loop body on inputs stacked per iteration, for the entry `what`
int train_step_iters(fg_ctx* c, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                     const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                     fg_step_stats* stats) {
  ENTER(c);
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h && real && noise_D && noise_G));
  Net32* n = c->n32;
  const size_t nd = d_iters, ng = g_iters, Bh = B / 2, M = c->maxB, img = (size_t)c->C * 1024;
  IterStage& s = n->iter_stage;
  const float *r, *zd, *zg, *md, *mg;
  FG_TRY(s.in(c, n->allocs, 0, real, nd * Bh * img, nd * M / 2 * img, &r));
  FG_TRY(s.in(c, n->allocs, 1, noise_D, nd * Bh * kNoiseDim, nd * M / 2 * kNoiseDim, &zd));
  FG_TRY(s.in(c, n->allocs, 2, noise_G, ng * B * kNoiseDim, ng * M * kNoiseDim, &zg));
  FG_TRY(s.in(c, n->allocs, 3, masks_D, nd * B * kMaskPerSample, nd * M * kMaskPerSample, &md));
  FG_TRY(s.in(c, n->allocs, 4, masks_G, ng * B * kMaskPerSample, ng * M * kMaskPerSample, &mg));
  NetStep st(n, h, B, r, zd, zg);
  return pair_train_step(st, d_iters, g_iters, md, mg, seed, {r, zd, zg, md, mg, nullptr}, nullptr, stats);
}

// the same fed on the device: the inputs of D iteration j are gather(draw(4*r_j)) and uniform(4*r_j+1), those of G
// iteration j uniform(4*r_j+2), r_j the stream root of iteration j (fg_b200.h; r_0 = seed).  The draws run inside the
// step (one graph launch per call once captured), each reading its root from c->seed_dev.
int train_step_dataset_iters(fg_ctx* c, fg_dataset* d, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters,
                             uint64_t seed, fg_step_stats* stats) {
  if (!d || !d->c) {
    fg_set_error("null fg_dataset");
    return FG_ERR_INVALID;
  }
  FG_CUDA(cudaSetDevice(d->c->device));
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h, d, true));
  Net32* n = c->n32;
  const int Bh = B / 2;
  const size_t M = c->maxB, img = (size_t)c->C * 1024;
  IterStage& s = n->iter_stage;
  FG_TRY(s.reserve(c, n->allocs, 0, d_iters * M / 2 * img));
  FG_TRY(s.reserve(c, n->allocs, 1, d_iters * M / 2 * kNoiseDim));
  FG_TRY(s.reserve(c, n->allocs, 2, g_iters * M * kNoiseDim));
  float *real = s.p[0], *zd = s.p[1], *zg = s.p[2];
  const std::function<int()> feed = [&]() -> int {
    for (int j = 0; j < d_iters; ++j) {
      FG_TRY(dataset_draw_gather(d, 0, Bh, 32, real + (size_t)j * Bh * img, c->seed_dev + j, 4));
      FG_TRY(noise_uniform_dev(c, 1, (int64_t)Bh * kNoiseDim, zd + (size_t)j * Bh * kNoiseDim, c->seed_dev + j, 4));
    }
    for (int j = 0; j < g_iters; ++j)
      FG_TRY(noise_uniform_dev(c, 2, (int64_t)B * kNoiseDim, zg + (size_t)j * B * kNoiseDim, c->seed_dev + j, 4));
    return FG_OK;
  };
  NetStep st(n, h, B, real, zd, zg);
  return pair_train_step(st, d_iters, g_iters, nullptr, nullptr, seed, {real, zd, zg, nullptr, nullptr, d}, &feed, stats);
}
}  // namespace

extern "C" {

int64_t fg_param_count(int net, int channels) {
  if (channels != 1 && channels != 3) return -1;
  return net == FG_NET_G ? make_g_layout(channels, 32).total : net == FG_NET_D ? make_d_layout(channels).total : -1;
}
int fg_set_params(fg_ctx* c, int net, const float* src) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_set_params(c, c->n32->net, net, src);
}
int fg_get_params(fg_ctx* c, int net, float* dst) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_get_params(c, c->n32->net, net, dst);
}
int fg_get_grads(fg_ctx* c, int net, float* dst) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_get_grads(c, c->n32->net, net, dst);
}
int fg_zero_grads(fg_ctx* c, int net) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_zero_grads(c, c->n32->net, net);
}
// Borrow caller-owned DEVICE buffers as the flat parameter / gradient vectors of `net` (see include/fg_b200.h).
int fg_bind_params(fg_ctx* c, int net, float* params_dev, float* grads_dev) {
  ENTER(c);
  c->graph_epoch++;
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  for (const float* p : {params_dev, grads_dev}) {
    if (!p) continue;
    FG_REQUIRE(fg_is_dev(p), "fg_bind_params: buffers must be DEVICE memory (CudaTensor:data())");
    FG_REQUIRE(reinterpret_cast<uintptr_t>(p) % 16 == 0, "fg_bind_params: buffers must be 16-byte aligned");
  }
  FG_CUDA(cudaStreamSynchronize(c->stream));
  Net32* n = c->n32;
  NetPair& np = n->net;
  const bool d = net == FG_NET_D;
  (d ? np.PD : np.PG) = params_dev ? params_dev : (d ? n->ownPD : n->ownPG);
  float* own_g = d ? n->ownGD : n->ownGG;
  const int64_t len = d ? np.nD : np.nG;
  (d ? np.gD : np.gG) = grads_dev ? grads_dev : own_g;
  (d ? np.tailD : np.tailG) = grads_dev ? n->tail_sep + (d ? kGradTail : 0) : own_g + len;
  np.G_pack = np.D_pack = -1;
  return FG_OK;
}
float* fg_params_ptr(fg_ctx* c, int net) {
  return !c ? nullptr : net == FG_NET_D ? c->n32->net.PD : net == FG_NET_G ? c->n32->net.PG : nullptr;
}
float* fg_grads_ptr(fg_ctx* c, int net) {
  return !c ? nullptr : net == FG_NET_D ? c->n32->net.gD : net == FG_NET_G ? c->n32->net.gG : nullptr;
}

int fg_set_adam_state(fg_ctx* c, int net, const float* m, const float* v, int t) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_set_adam_state(c, c->n32->net, net, m, v, t);
}
int fg_get_adam_state(fg_ctx* c, int net, float* m, float* v, int* t) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_get_adam_state(c, c->n32->net, net, m, v, t);
}
int fg_set_bn_state(fg_ctx* c, const float* src) {
  ENTER(c);
  return pair_set_bn_state(c, c->n32->net, src);
}
int fg_get_bn_state(fg_ctx* c, float* dst) {
  ENTER(c);
  return pair_get_bn_state(c, c->n32->net, dst);
}

// ---- L-net ------------------------------------------------------------------------------------------
int fg_G_forward(fg_ctx* c, const float* noise, int B, int training, float* images_out) {
  ENTER(c);
  FG_REQUIRE(noise && B >= 1 && B <= c->maxB, "fg_G_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  Net32* n = c->n32;
  n->net.G_pack = -1;  // parameters may have been edited through fg_params_ptr()
  const float* nd;
  FG_TRY(fg_to_dev(c, noise, (size_t)B * kNoiseDim, n->in_noiseG, &nd));
  FG_TRY(gen_forward(n->env, n->G, n->net, nd, B, training != 0));
  if (images_out) {
    FG_TRY(k_nhwc_to_nchw(c, n->G.y, c->io_dev, B, c->C, 1024));
    FG_TRY(fg_to_user(c, images_out, c->io_dev, (size_t)B * c->C * 1024));
  }
  return FG_OK;
}
int fg_G_backward(fg_ctx* c, const float* d_images, float* d_noise) {
  ENTER(c);
  FG_REQUIRE(d_images, "fg_G_backward: d_images is null");
  Net32* n = c->n32;
  const int B = n->G.B;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_images, (size_t)B * c->C * 1024, c->io_dev, &dd));
  FG_TRY(k_nchw_to_nhwc(c, dd, n->io_dev2, B, c->C, 1024));
  float* dn = nullptr;
  if (d_noise) dn = fg_is_dev(d_noise) ? d_noise : n->in_noiseD;
  FG_TRY(gen_backward(n->env, n->G, n->net, n->io_dev2, dn));
  if (d_noise && dn != d_noise) FG_TRY(fg_to_user(c, d_noise, dn, (size_t)B * kNoiseDim));
  return FG_OK;
}
int fg_D_forward(fg_ctx* c, const float* images, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(c);
  FG_REQUIRE(images && B >= 1 && B <= c->maxB, "fg_D_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  Net32* n = c->n32;
  n->net.D_pack = -1;
  fg_hyper h;
  fg_hyper_default(&h);
  const float* xd;
  FG_TRY(fg_to_dev(c, images, (size_t)B * c->C * 1024, c->io_dev, &xd));
  FG_TRY(k_nchw_to_nhwc(c, xd, n->D_x, B, c->C, 1024));
  if (training) {
    if (masks) {
      FG_CUDA(cudaMemcpyAsync(n->D_masks, masks, sizeof(float) * (size_t)B * kMaskPerSample, cudaMemcpyDefault, c->stream));
    } else {
      FG_TRY(k_masks_generate(c, n->D_masks, B, seed, h.p_spatial, h.p_drop));
    }
  }
  FG_TRY(D_forward(n, n->D_x, B, training != 0, &h));
  FG_TRY(k_sigmoid_fwd(c, n->D_logit, n->D_out, B));
  if (out) FG_TRY(fg_to_user(c, out, n->D_out, B));
  return FG_OK;
}
int fg_D_backward(fg_ctx* c, const float* d_out, int want_wgrad, float* d_images) {
  ENTER(c);
  FG_REQUIRE(d_out, "fg_D_backward: d_out is null");
  Net32* n = c->n32;
  const int B = n->D_B;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_out, B, n->D_targets, &dd));
  FG_TRY(k_sigmoid_grad_mul(c, dd, n->D_out, n->D_dlogit, B));
  FG_TRY(D_backward(n, n->D_dlogit, want_wgrad != 0, d_images != nullptr));
  if (d_images) {
    FG_TRY(k_nhwc_to_nchw(c, n->D_dx, c->io_dev, B, c->C, 1024));
    FG_TRY(fg_to_user(c, d_images, c->io_dev, (size_t)B * c->C * 1024));
  }
  return FG_OK;
}
int fg_bce_forward(fg_ctx* c, const float* x, const float* t, int n, float* loss_out) {
  ENTER(c);
  FG_REQUIRE(x && t && loss_out && n > 0 && n <= c->maxB, "fg_bce_forward: bad arguments");
  const float *xd, *td;
  FG_TRY(fg_to_dev(c, x, n, c->io_dev, &xd));
  FG_TRY(fg_to_dev(c, t, n, c->n32->io_dev2, &td));
  FG_TRY(k_bce_fwd(c, xd, td, n, c->n32->D_targets));
  return fg_to_user(c, loss_out, c->n32->D_targets, 1);
}
int fg_bce_backward(fg_ctx* c, const float* x, const float* t, int n, float* dx) {
  ENTER(c);
  FG_REQUIRE(x && t && dx && n > 0 && n <= c->maxB, "fg_bce_backward: bad arguments");
  const float *xd, *td;
  FG_TRY(fg_to_dev(c, x, n, c->io_dev, &xd));
  FG_TRY(fg_to_dev(c, t, n, c->n32->io_dev2, &td));
  FG_TRY(k_bce_bwd(c, xd, td, n, c->n32->D_targets));
  return fg_to_user(c, dx, c->n32->D_targets, n);
}
int fg_optim_step(fg_ctx* c, int net, const fg_hyper* h, float grad_scale) {
  ENTER(c);
  FG_REQUIRE(h && (net == FG_NET_G || net == FG_NET_D), "fg_optim_step: bad arguments");
  // no accuracy information at this level: no gate, and the fused steps' accuracy history is not touched
  FG_TRY(k_optim_prep(c, c->n32->net.dstats, net, h));
  return pair_optim(c, c->n32->net, net, h, grad_scale);
}

// ---- L-step -----------------------------------------------------------------------------------------
int fg_train_step(fg_ctx* c, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                  const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  return train_step_iters(c, "fg_train_step", h, B, 1, 1, real, noise_D, noise_G, masks_D, masks_G, seed, stats);
}
int fg_train_step_iters(fg_ctx* c, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                        const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                        fg_step_stats* stats) {
  return train_step_iters(c, "fg_train_step_iters", h, B, d_iters, g_iters, real, noise_D, noise_G, masks_D, masks_G, seed,
                          stats);
}
// One adversarial.lua loop body fed entirely on the device: real half-batch = gather(draw(4*seed)), noise for the
// D step = uniform(4*seed+1), for the G step = uniform(4*seed+2), dropout masks from `seed` as in fg_train_step.
int fg_train_step_dataset(fg_ctx* c, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats) {
  return train_step_dataset_iters(c, d, "fg_train_step_dataset", h, B, 1, 1, seed, stats);
}
int fg_train_step_dataset_iters(fg_ctx* c, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters, uint64_t seed,
                                fg_step_stats* stats) {
  return train_step_dataset_iters(c, d, "fg_train_step_dataset_iters", h, B, d_iters, g_iters, seed, stats);
}

int fg_sample(fg_ctx* c, const float* noise, int N, int chunk, float* images_out) {
  ENTER(c);
  FG_REQUIRE(noise && images_out && N >= 1 && chunk >= 1 && chunk <= c->maxB, "fg_sample: bad arguments (chunk %d, max %d)",
             chunk, c->maxB);
  Net32* n = c->n32;
  const bool out_dev = fg_is_dev(images_out);
  const size_t img = (size_t)c->C * 1024;
  n->net.G_pack = -1;
  for (int s = 0; s < N; s += chunk) {
    const int b = std::min(chunk, N - s);
    const float* nd;
    FG_TRY(fg_to_dev(c, noise + (size_t)s * kNoiseDim, (size_t)b * kNoiseDim, n->in_noiseG, &nd));
    // sample.lua never calls :evaluate() => BatchNorm uses the statistics of each chunk (SURVEY 3.4)
    FG_TRY(gen_forward(n->env, n->G, n->net, nd, b, true));
    float* dst = images_out + (size_t)s * img;
    if (out_dev) {
      FG_TRY(k_nhwc_to_nchw(c, n->G.y, dst, b, c->C, 1024));
    } else {
      FG_TRY(k_nhwc_to_nchw(c, n->G.y, c->io_dev, b, c->C, 1024));
      FG_CUDA(cudaMemcpyAsync(dst, c->io_dev, b * img * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
      if (s + chunk < N) FG_CUDA(cudaStreamSynchronize(c->stream));  // io_dev is reused by the next chunk
    }
  }
  if (!out_dev) FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int64_t fg_debug_tensor(fg_ctx* c, const char* name, float* dst, int64_t max_elems) {
  if (!c || !name) return -1;
  cudaSetDevice(c->device);
  const Net32* n = c->n32;
  const int db = n->D_B;
  std::vector<DebugTensor> ents = {
      {"D.z1", n->D_z[0], 65536, db}, {"D.z2", n->D_z[1], 32768, db}, {"D.z3", n->D_z[2], 16384, db},
      {"D.z4", n->D_z[3], 8192, db}, {"D.p1", n->D_p[0], 16384, db}, {"D.p2", n->D_p[1], 8192, db},
      {"D.p3", n->D_p[2], 4096, db}, {"D.p4", n->D_p[3], 2048, db}, {"D.logit", n->D_logit, 1, db},
      {"D.out", n->D_out, 1, db}, {"D.dx", n->D_dx, 1024 * c->C, db}, {"D.masks", n->D_masks, kMaskPerSample, db},
      {"D.zl1", n->D_zl1, 512, db}, {"D.hl1", n->D_hl1, 512, db}, {"D.zl2", n->D_zl2, 512, db},
      {"D.hl2", n->D_hl2, 512, db}, {"D.dlogit", n->D_dlogit, 1, db}};
  for (const NetPair::Keep& k : n->bwd_keep) ents.push_back({k.name, k.copy, k.per, n->bwd_keep_B});
  pair_keep_rows(n->net, ents);
  gen_debug_rows(n->G, ents);
  return debug_tensor_copy(c, "fg_debug_tensor", ents.data(), ents.size(), name, dst, max_elems);
}

}  // extern "C"
