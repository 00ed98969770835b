// Coarse-to-fine GAN (BASELINE configs[3], train_c2f.lua) on the same kernels as the 32x32 nets:
//   G = models_c2f.lua:113-145 create_G_d : JoinTable{noise[1x32x32], coarse[Cx32x32]} -> SCU(C+1->64,3) PReLU
//       SCU(64->64,3) PReLU SCU(64->128,5) PReLU SCU(128->256,5) PReLU SCU(256->C,7)            (all at 32x32)
//   D = models_c2f.lua:237-278 create_D_c : CAddTable{diff, coarse} -> conv(C->64,3) PReLU conv(64->64,3) PReLU
//       MaxPool2 conv(64->128,3) PReLU conv(128->256,3) PReLU MaxPool2 Dropout View(16384) Linear(512) PReLU
//       Dropout Linear(1) Sigmoid
//   loop = adversarial_c2f.lua:121-187 (fevalD :40-81, fevalG_on_D :85-116, optim.adam)
// cudnn.SpatialConvolutionUpsample with factor 1 (layers/cudnnSpatialConvolutionUpsample.lua:4-28) is a "same"
// convolution whose output view is the identity, so every layer maps onto the tap-GEMM convolution kernels:
// wgmma (3xTF32, chunk-promoted) where the channel counts make a dense contraction (64->64, 64->128,
// 128->256 and the 16384->512 Linear), the bandwidth-shaped small-channel kernels for (C+1)->64 / C->64 and the
// fp32 FFMA tile kernel for the 256->C 7x7 output layer (N = 3 is not a tensor-core shape).
#include <algorithm>
#include <cstring>

#include "convl.h"
#include "fg_internal.h"
#include "k_conv_tc.h"
#include "k_misc.h"

namespace {
constexpr int kC2fMask = 16384 + 512;  // nn.Dropout keep flags per sample: [256][8][8] then [512]
}  // namespace

struct fg_c2f {
  fg_ctx* c = nullptr;
  int maxB = 0, C = 3;
  int64_t nG = 0, nD = 0;
  float *PG = nullptr, *PD = nullptr, *gG = nullptr, *gD = nullptr, *mG = nullptr, *vG = nullptr, *mD = nullptr,
        *vD = nullptr;
  DeviceStats *dstats = nullptr, *hstats = nullptr;
  float* acc_hist = nullptr;
  int64_t Gca[4] = {0, 0, 0, 0}, Dca[4] = {0, 0, 0, 0}, Da5 = 0, DL2W = 0, DL2b = 0;
  ConvL Gc[5], Dc[4], DL1;
  bool G_packed = false, D_packed = false;
  int G_pack_impl = -1, D_pack_impl = -1;
  float *G_x = nullptr, *G_z[5] = {}, *G_h[4] = {};
  float *D_x = nullptr, *D_cond = nullptr, *D_z[4] = {}, *D_h[4] = {}, *D_p2 = nullptr, *D_p4 = nullptr, *D_d4 = nullptr;
  float *D_zl1 = nullptr, *D_al1 = nullptr, *D_hl1 = nullptr, *D_logit = nullptr, *D_out = nullptr, *D_masks = nullptr,
        *D_dlogit = nullptr, *D_dx = nullptr;
  float *ga = nullptr, *gb = nullptr, *dy_hi = nullptr, *dy_lo = nullptr, *ws = nullptr;
  float *pad_hi = nullptr, *pad_lo = nullptr;  // channel-padded TF32 split of dY (ConvL::pad_out / pad_dy)
  float *in_a = nullptr, *in_b = nullptr, *in_c = nullptr, *in_d = nullptr, *in_e = nullptr, *in_m1 = nullptr,
        *in_m2 = nullptr, *io = nullptr;
  int G_B = 0, D_B = 0;
  bool G_valid = false, D_valid = false, D_train = true;
  float D_scale = 2.f;
  std::vector<void*> allocs;
  ConvLEnv env;  // shared scratch of the ConvL layers (filled by c2f_alloc)
  std::vector<fg_ctx::StepGraph> graphs;  // captured train steps
};

namespace {
int dalloc(fg_c2f* n, float** p, size_t elems) { return convl_dalloc(n->env, p, elems); }
inline int to_dev(fg_ctx* c, const float* p, size_t n, float* staging, const float** out) { return fg_to_dev(c, p, n, staging, out); }
inline int to_user(fg_ctx* c, float* dst, const float* src_dev, size_t n) { return fg_to_user(c, dst, src_dev, n); }
inline int convl_alloc(fg_c2f* n, ConvL& L) { return ::convl_alloc(n->env, L); }
inline int convl_fwd(fg_c2f* n, ConvL& L, const float* in, const float* P, float* out, int B) { return ::convl_fwd(n->env, L, in, P, out, B); }
inline int convl_bwd(fg_c2f* n, ConvL& L, const float* in, const float* dy, float* G, float* din, int B) {
  return ::convl_bwd(n->env, L, in, dy, G, din, B);
}

void make_layouts(fg_c2f* n) {
  const int C = n->C;
  {
    const int ci[5] = {C + 1, 64, 64, 128, 256}, co[5] = {64, 64, 128, 256, C}, kk[5] = {3, 3, 5, 5, 7};
    static const char* tf[5] = {"c2f.G.c1.fwd", "c2f.G.c2.fwd", "c2f.G.c3.fwd", "c2f.G.c4.fwd", "c2f.G.c5.fwd"};
    static const char* td[5] = {"c2f.G.c1.dgrad", "c2f.G.c2.dgrad", "c2f.G.c3.dgrad", "c2f.G.c4.dgrad", "c2f.G.c5.dgrad"};
    static const char* tw[5] = {"c2f.G.c1.wgrad", "c2f.G.c2.wgrad", "c2f.G.c3.wgrad", "c2f.G.c4.wgrad", "c2f.G.c5.wgrad"};
    int64_t o = 0;
    for (int i = 0; i < 5; ++i) {
      ConvL& L = n->Gc[i];
      L.Cin = ci[i]; L.Cout = co[i]; L.k = kk[i]; L.H = 32;
      L.w_off = o; o += (int64_t)co[i] * ci[i] * kk[i] * kk[i];
      L.b_off = o; o += co[i];
      if (i < 4) { n->Gca[i] = o; o += 1; }
      L.need_dgrad = i > 0;
      L.tf = tf[i]; L.td = td[i]; L.tw = tw[i];
      if (co[i] <= 4 && ci[i] % 128 == 0) L.pad_out = 64;  // c5: 256 -> C, 7x7
      if (co[i] == 64 && ci[i] % 64 == 0) L.pad_dy = 128;  // c2: 64 -> 64
    }
    n->nG = o;
  }
  {
    const int ci[4] = {C, 64, 64, 128}, co[4] = {64, 64, 128, 256}, hw[4] = {32, 32, 16, 16};
    static const char* tf[4] = {"c2f.D.c1.fwd", "c2f.D.c2.fwd", "c2f.D.c3.fwd", "c2f.D.c4.fwd"};
    static const char* td[4] = {"c2f.D.c1.dgrad", "c2f.D.c2.dgrad", "c2f.D.c3.dgrad", "c2f.D.c4.dgrad"};
    static const char* tw[4] = {"c2f.D.c1.wgrad", "c2f.D.c2.wgrad", "c2f.D.c3.wgrad", "c2f.D.c4.wgrad"};
    int64_t o = 0;
    for (int i = 0; i < 4; ++i) {
      ConvL& L = n->Dc[i];
      L.Cin = ci[i]; L.Cout = co[i]; L.k = 3; L.H = hw[i];
      L.w_off = o; o += (int64_t)co[i] * ci[i] * 9;
      L.b_off = o; o += co[i];
      n->Dca[i] = o; o += 1;
      L.tf = tf[i]; L.td = td[i]; L.tw = tw[i];
      if (co[i] == 64 && ci[i] % 64 == 0) L.pad_dy = 128;  // c2: 64 -> 64
    }
    ConvL& L = n->DL1;
    L.Cin = 16384; L.Cout = 512; L.k = 1; L.H = 1;
    L.cA = 256; L.cS = 64;  // View(16384) flattens [256][8][8]; ours is [8][8][256]
    L.w_off = o; o += (int64_t)512 * 16384;
    L.b_off = o; o += 512;
    L.tf = "c2f.D.L1.fwd"; L.td = "c2f.D.L1.dgrad"; L.tw = "c2f.D.L1.wgrad";
    n->Da5 = o; o += 1;
    n->DL2W = o; o += 512;
    n->DL2b = o; o += 1;
    n->nD = o;
  }
}

int c2f_alloc(fg_c2f* n) {
  const size_t B = n->maxB, C = n->C;
  make_layouts(n);
  n->env.c = n->c;
  n->env.maxB = n->maxB;
  n->env.allocs = &n->allocs;
  FG_TRY(dalloc(n, &n->PG, n->nG));
  FG_TRY(dalloc(n, &n->PD, n->nD));
  FG_TRY(dalloc(n, &n->gG, n->nG + kGradTail));
  FG_TRY(dalloc(n, &n->gD, n->nD + kGradTail));
  FG_TRY(dalloc(n, &n->mG, n->nG));
  FG_TRY(dalloc(n, &n->vG, n->nG));
  FG_TRY(dalloc(n, &n->mD, n->nD));
  FG_TRY(dalloc(n, &n->vD, n->nD));
  float* tmp = nullptr;
  FG_TRY(dalloc(n, &tmp, (sizeof(DeviceStats) + 3) / 4));
  n->dstats = (DeviceStats*)tmp;
  FG_TRY(dalloc(n, &n->acc_hist, kAccHistMax));
  FG_CUDA(cudaMallocHost((void**)&n->hstats, sizeof(DeviceStats)));
  memset(n->hstats, 0, sizeof(DeviceStats));
  for (int i = 0; i < 5; ++i) FG_TRY(convl_alloc(n, n->Gc[i]));
  for (int i = 0; i < 4; ++i) FG_TRY(convl_alloc(n, n->Dc[i]));
  FG_TRY(convl_alloc(n, n->DL1));
  FG_TRY(dalloc(n, &n->G_x, B * 1024 * (C + 1)));
  for (int i = 0; i < 5; ++i) {
    FG_TRY(dalloc(n, &n->G_z[i], B * 1024 * n->Gc[i].Cout));
    if (i < 4) FG_TRY(dalloc(n, &n->G_h[i], B * 1024 * n->Gc[i].Cout));
  }
  FG_TRY(dalloc(n, &n->D_x, B * 1024 * C));
  FG_TRY(dalloc(n, &n->D_cond, B * 1024 * C));
  for (int i = 0; i < 4; ++i) {
    const size_t e = B * (size_t)n->Dc[i].H * n->Dc[i].H * n->Dc[i].Cout;
    FG_TRY(dalloc(n, &n->D_z[i], e));
    FG_TRY(dalloc(n, &n->D_h[i], e));
  }
  FG_TRY(dalloc(n, &n->D_p2, B * 256 * 64));
  FG_TRY(dalloc(n, &n->D_p4, B * 16384));
  FG_TRY(dalloc(n, &n->D_d4, B * 16384));
  FG_TRY(dalloc(n, &n->D_zl1, B * 512));
  FG_TRY(dalloc(n, &n->D_al1, B * 512));
  FG_TRY(dalloc(n, &n->D_hl1, B * 512));
  FG_TRY(dalloc(n, &n->D_logit, B));
  FG_TRY(dalloc(n, &n->D_out, B));
  FG_TRY(dalloc(n, &n->D_dlogit, B));
  FG_TRY(dalloc(n, &n->D_masks, B * kC2fMask));
  FG_TRY(dalloc(n, &n->D_dx, B * 1024 * C));
  const size_t big = B * 1024 * 256;  // largest activation: G conv4 output
  FG_TRY(dalloc(n, &n->ga, big));
  FG_TRY(dalloc(n, &n->gb, big));
  FG_TRY(dalloc(n, &n->dy_hi, big));
  FG_TRY(dalloc(n, &n->dy_lo, big));
  FG_TRY(dalloc(n, &n->pad_hi, big / 2));  // up to 128 padded channels at 32x32
  FG_TRY(dalloc(n, &n->pad_lo, big / 2));
  FG_TRY(dalloc(n, &n->ws, std::max<size_t>((size_t)512 * 16384, (size_t)25 * 256 * 128)));
  n->env.ga = n->ga; n->env.dy_hi = n->dy_hi; n->env.dy_lo = n->dy_lo;
  n->env.pad_hi = n->pad_hi; n->env.pad_lo = n->pad_lo; n->env.ws = n->ws;
  FG_TRY(dalloc(n, &n->in_a, B * 1024 * C));
  FG_TRY(dalloc(n, &n->in_b, B * 1024 * C));
  FG_TRY(dalloc(n, &n->in_c, B * 1024));
  FG_TRY(dalloc(n, &n->in_d, B * 1024 * C));
  FG_TRY(dalloc(n, &n->in_e, B * 1024));
  FG_TRY(dalloc(n, &n->in_m1, B * kC2fMask));
  FG_TRY(dalloc(n, &n->in_m2, B * kC2fMask));
  FG_TRY(dalloc(n, &n->io, B * 1024 * C));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}

// packs are rebuilt after every optimizer step / set_params, and when the ctx's "conv_impl" changed since the last
// pack (the TF32 splits are only produced for the tensor-core implementations)
int pack_G(fg_c2f* n) {
  if (n->G_packed && n->G_pack_impl == pack_key(n->c)) return FG_OK;
  for (int i = 0; i < 5; ++i) FG_TRY(convl_pack(n->c, n->Gc[i], n->PG));
  n->G_packed = true;
  n->G_pack_impl = pack_key(n->c);
  return FG_OK;
}
int pack_D(fg_c2f* n) {
  if (n->D_packed && n->D_pack_impl == pack_key(n->c)) return FG_OK;
  for (int i = 0; i < 4; ++i) FG_TRY(convl_pack(n->c, n->Dc[i], n->PD));
  FG_TRY(convl_pack(n->c, n->DL1, n->PD));
  n->D_packed = true;
  n->D_pack_impl = pack_key(n->c);
  return FG_OK;
}

// noise [B][1][32][32] and cond [B][C][32][32] are NCHW device pointers; the diff lands in G_z[4] (NHWC)
int G_forward(fg_c2f* n, const float* noise, const float* cond, int B) {
  fg_ctx* c = n->c;
  FG_REQUIRE(B >= 1 && B <= n->maxB, "c2f G forward: batch %d out of range [1,%d]", B, n->maxB);
  FG_TRY(pack_G(n));
  FG_TRY(k_join_to_nhwc(c, noise, cond, n->G_x, B, n->C, 1024));
  const float* cur = n->G_x;
  for (int i = 0; i < 5; ++i) {
    FG_TRY(convl_fwd(n, n->Gc[i], cur, n->PG, n->G_z[i], B));
    if (i < 4) {
      FG_TRY(k_prelu_fwd(c, n->G_z[i], n->PG + n->Gca[i], n->G_h[i], (int64_t)B * 1024 * n->Gc[i].Cout));
      cur = n->G_h[i];
    }
  }
  n->G_B = B;
  n->G_valid = true;
  return FG_OK;
}
// ddiff: NHWC [B][32][32][C]; accumulates into gG
int G_backward(fg_c2f* n, const float* ddiff) {
  fg_ctx* c = n->c;
  if (!n->G_valid) {
    fg_set_error("c2f G backward needs a preceding G forward");
    return FG_ERR_STATE;
  }
  const int B = n->G_B;
  const float* dcur = ddiff;
  for (int i = 4; i >= 0; --i) {
    const float* in = i == 0 ? n->G_x : n->G_h[i - 1];
    FG_TRY(convl_bwd(n, n->Gc[i], in, dcur, n->gG, i > 0 ? n->ga : nullptr, B));
    if (i > 0) {
      FG_TRY(k_prelu_bwd(c, n->ga, n->G_z[i - 1], n->PG + n->Gca[i - 1], n->gb, n->gG + n->Gca[i - 1], B, 32, 32,
                         n->Gc[i - 1].Cout, 0));
      dcur = n->gb;
    }
  }
  return FG_OK;
}

// diff, cond: NHWC device pointers; dropout keep flags already in D_masks when training
int D_forward(fg_c2f* n, const float* diff, const float* cond, int B, bool training, float p_drop) {
  fg_ctx* c = n->c;
  FG_REQUIRE(B >= 1 && B <= n->maxB, "c2f D forward: batch %d out of range [1,%d]", B, n->maxB);
  FG_TRY(pack_D(n));
  const float* P = n->PD;
  FG_TRY(k_add(c, diff, cond, n->D_x, (int64_t)B * 1024 * n->C));  // nn.CAddTable
  const float* cur = n->D_x;
  for (int i = 0; i < 4; ++i) {
    const ConvL& L = n->Dc[i];
    FG_TRY(convl_fwd(n, n->Dc[i], cur, P, n->D_z[i], B));
    FG_TRY(k_prelu_fwd(c, n->D_z[i], P + n->Dca[i], n->D_h[i], (int64_t)B * L.H * L.H * L.Cout));
    cur = n->D_h[i];
    if (i == 1) {
      FG_TRY(k_maxpool2_fwd(c, n->D_h[1], n->D_p2, B, 32, 32, 64));
      cur = n->D_p2;
    } else if (i == 3) {
      FG_TRY(k_maxpool2_fwd(c, n->D_h[3], n->D_p4, B, 16, 16, 256));
    }
  }
  n->D_scale = 1.0f / (1.0f - p_drop);
  const float* d4 = n->D_p4;
  if (training) {  // nn.Dropout (v2): mask/(1-p) in training, identity in evaluation
    FG_TRY(k_dropout_nhwc(c, n->D_p4, n->D_masks, kC2fMask, 0, 64, 256, n->D_scale, n->D_d4, B));
    d4 = n->D_d4;
  }
  FG_TRY(convl_fwd(n, n->DL1, d4, P, n->D_zl1, B));
  FG_TRY(k_prelu_fwd(c, n->D_zl1, P + n->Da5, n->D_al1, (int64_t)B * 512));
  const float* hl1 = n->D_al1;
  if (training) {
    FG_TRY(k_dropout_nhwc(c, n->D_al1, n->D_masks, kC2fMask, 16384, 1, 512, n->D_scale, n->D_hl1, B));
    hl1 = n->D_hl1;
  }
  {
    ScopedTimer tm(c, "c2f.D.L2.fwd");
    FG_TRY(k_gemv_fwd(c, hl1, P + n->DL2W, P + n->DL2b, n->D_logit, B, 512));
  }
  n->D_B = B;
  n->D_train = training;
  n->D_valid = true;
  return FG_OK;
}
// dlogit [B] = dLoss/dlogit; want_dx: gradient w.r.t. the diff input (MODEL_D.gradInput[1]) into D_dx (NHWC)
int D_backward(fg_c2f* n, const float* dlogit, bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  if (!n->D_valid) {
    fg_set_error("c2f D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const int B = n->D_B;
  const float* P = n->PD;
  float* G = want_wgrad ? n->gD : nullptr;
  const bool tr = n->D_train;
  const float* hl1 = tr ? n->D_hl1 : n->D_al1;
  const float* d4 = tr ? n->D_d4 : n->D_p4;
  if (G) FG_TRY(k_gemv_wgrad_add(c, hl1, dlogit, G + n->DL2W, G + n->DL2b, B, 512));
  float *cur = n->ga, *oth = n->gb;  // gradient ping-pong: every stage reads `cur`, writes `oth`, then they swap
  FG_TRY(k_gemv_dgrad(c, dlogit, P + n->DL2W, cur, B, 512));
  if (tr) {
    FG_TRY(k_dropout_nhwc(c, cur, n->D_masks, kC2fMask, 16384, 1, 512, n->D_scale, oth, B));
    std::swap(cur, oth);
  }
  FG_TRY(k_prelu_bwd(c, cur, n->D_zl1, P + n->Da5, oth, G ? G + n->Da5 : nullptr, B, 1, 1, 512, 0));
  std::swap(cur, oth);
  FG_TRY(convl_bwd(n, n->DL1, d4, cur, G, oth, B));  // -> gradient of the View(16384) input, [B][8][8][256]
  std::swap(cur, oth);
  if (tr) {
    FG_TRY(k_dropout_nhwc(c, cur, n->D_masks, kC2fMask, 0, 64, 256, n->D_scale, oth, B));
    std::swap(cur, oth);
  }
  for (int i = 3; i >= 0; --i) {
    ConvL& L = n->Dc[i];
    if (i == 3 || i == 1) {  // cur is the gradient of the pooled map
      FG_TRY(k_maxpool2_bwd(c, cur, n->D_h[i], oth, B, L.H, L.H, L.Cout));
      std::swap(cur, oth);
    }
    FG_TRY(k_prelu_bwd(c, cur, n->D_z[i], P + n->Dca[i], oth, G ? G + n->Dca[i] : nullptr, B, L.H, L.H, L.Cout, 0));
    std::swap(cur, oth);
    const float* in = i == 0 ? n->D_x : (i == 2 ? n->D_p2 : n->D_h[i - 1]);
    float* din = i > 0 ? oth : (want_dx ? n->D_dx : nullptr);
    FG_TRY(convl_bwd(n, L, in, cur, G, din, B));
    if (i > 0) std::swap(cur, oth);
  }
  return FG_OK;
}

int optim(fg_c2f* n, int net, const fg_hyper* h, float grad_scale) {
  fg_ctx* c = n->c;
  const bool isD = net == FG_NET_D;
  float *p = isD ? n->PD : n->PG, *g = isD ? n->gD : n->gG, *m = isD ? n->mD : n->mG, *v = isD ? n->vD : n->vG;
  const int64_t cnt = isD ? n->nD : n->nG;
  const float l1 = isD ? h->D_L1 : h->G_L1, l2 = isD ? h->D_L2 : h->G_L2;
  const bool pen = l1 != 0.f || l2 != 0.f;
  const float l1_grad = !pen ? 0.f : (isD ? l1 : l2);  // adversarial_c2f.lua:108 scales sign(p) by G_L2
  if (pen) FG_TRY(k_penalty_loss(c, p, cnt, l1, l2, isD ? &n->dstats->loss_D : &n->dstats->loss_G));
  // optim.adam / optim.adagrad / optim.sgd (adversarial_c2f.lua:153-161, :177-185): same rules as the interruptable ones
  FG_TRY(k_optim_update(c, isD ? c->opt_D : c->opt_G, p, g, m, v, cnt, h->beta1, h->beta2, h->eps,
                        isD ? c->sgd_mom_D : c->sgd_mom_G, l1_grad, pen ? l2 : 0.f, isD ? h->D_clamp : h->G_clamp, grad_scale,
                        isD ? &n->dstats->step_D : &n->dstats->step_G, isD ? &n->dstats->do_train_D : &n->dstats->do_train_G,
                        isD ? &n->dstats->t_D : &n->dstats->t_G));
  if (isD) n->D_packed = false; else n->G_packed = false;
  return FG_OK;
}
// t += 1 and the Adam step size on the device (shares the kernel of the 32x32 loop; no accuracy gate here)
int prep(fg_c2f* n, int net, const fg_hyper* h, const float* tail4, int B) {
  fg_ctx* c = n->c;
  fg_hyper hh = *h;
  hh.D_maxAcc = 1e30f;
  DeviceStats* sd = c->dstats;
  float* sa = c->acc_hist;
  c->dstats = n->dstats;
  c->acc_hist = n->acc_hist;
  const int r = k_gate_and_prep(c, net, &hh, tail4, B, (float)c->world);
  c->dstats = sd;
  c->acc_hist = sa;
  return r;
}

int train_step(fg_c2f* n, const fg_hyper* h, int B, const float* real_diff, const float* condD, const float* noiseD,
               const float* condG, const float* noiseG, const float* masksD, const float* masksG, uint64_t seed) {
  fg_ctx* c = n->c;
  const int Bh = B / 2, C = n->C;
  const size_t img = (size_t)C * 1024;
  const float inv_world = 1.0f / (float)c->world;
  // ---- D step (adversarial_c2f.lua:121-163) ----
  FG_TRY(G_forward(n, noiseD, condD + Bh * img, Bh));
  FG_TRY(k_nchw_to_nhwc(c, real_diff, n->io, Bh, C, 1024));
  FG_CUDA(cudaMemcpyAsync(n->io + Bh * img, n->G_z[4], sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
  FG_TRY(k_nchw_to_nhwc(c, condD, n->D_cond, B, C, 1024));
  if (masksD)
    FG_CUDA(cudaMemcpyAsync(n->D_masks, masksD, sizeof(float) * (size_t)B * kC2fMask, cudaMemcpyDeviceToDevice, c->stream));
  else
    FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * kC2fMask, 1, h->p_drop, c->seed_dev));
  FG_CUDA(cudaMemsetAsync(n->gD, 0, sizeof(float) * (n->nD + kGradTail), c->stream));
  FG_TRY(D_forward(n, n->io, n->D_cond, B, true, h->p_drop));
  FG_TRY(k_sigmoid_bce(c, n->D_logit, n->D_out, n->D_dlogit, &n->dstats->loss_D, n->gD + n->nD, B, Bh));
  FG_TRY(D_backward(n, n->D_dlogit, true, false));
  if (c->world > 1) FG_TRY(net_allreduce(c, n->gD, n->nD + kGradTail));
  FG_TRY(prep(n, FG_NET_D, h, n->gD + n->nD, B));
  FG_TRY(optim(n, FG_NET_D, h, inv_world));
  // ---- G step (adversarial_c2f.lua:167-187) ----
  FG_CUDA(cudaMemsetAsync(n->gG, 0, sizeof(float) * (n->nG + kGradTail), c->stream));
  FG_TRY(G_forward(n, noiseG, condG, B));
  FG_TRY(k_nchw_to_nhwc(c, condG, n->D_cond, B, C, 1024));
  if (masksG)
    FG_CUDA(cudaMemcpyAsync(n->D_masks, masksG, sizeof(float) * (size_t)B * kC2fMask, cudaMemcpyDeviceToDevice, c->stream));
  else
    FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * kC2fMask, 2, h->p_drop, c->seed_dev));
  FG_TRY(D_forward(n, n->G_z[4], n->D_cond, B, true, h->p_drop));
  FG_TRY(k_sigmoid_bce(c, n->D_logit, n->D_out, n->D_dlogit, &n->dstats->loss_G, n->gG + n->nG, B, B));
  FG_TRY(D_backward(n, n->D_dlogit, false, true));  // D's weight grads are zeroed before use (:45) -> skipped
  FG_TRY(G_backward(n, n->D_dx));
  if (c->world > 1) FG_TRY(net_allreduce(c, n->gG, n->nG + kGradTail));
  FG_TRY(prep(n, FG_NET_G, h, n->gG + n->nG, B));
  FG_TRY(optim(n, FG_NET_G, h, inv_world));
  FG_CUDA(cudaMemcpyAsync(n->hstats, n->dstats, sizeof(DeviceStats), cudaMemcpyDeviceToHost, c->stream));
  return FG_OK;
}
}  // namespace

#define ENTER(n)                                         \
  do {                                                   \
    if (!(n) || !(n)->c) {                               \
      fg_set_error("null fg_c2f");                       \
      return FG_ERR_INVALID;                             \
    }                                                    \
    FG_CUDA(cudaSetDevice((n)->c->device));              \
  } while (0)

extern "C" {

int fg_c2f_create(fg_ctx* ctx, fg_c2f** out) {
  if (!ctx || !out) {
    fg_set_error("fg_c2f_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_c2f* n = new fg_c2f();
  n->c = ctx;
  n->maxB = ctx->maxB;
  n->C = ctx->C;
  const int r = c2f_alloc(n);
  if (r != FG_OK) {
    fg_c2f_destroy(n);
    return r;
  }
  *out = n;
  return FG_OK;
}
int fg_c2f_destroy(fg_c2f* n) {
  if (!n) return FG_OK;
  if (n->c) {
    cudaSetDevice(n->c->device);
    cudaStreamSynchronize(n->c->stream);
  }
  for (auto& g : n->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  for (void* p : n->allocs) cudaFree(p);
  if (n->hstats) cudaFreeHost(n->hstats);
  delete n;
  return FG_OK;
}
int64_t fg_c2f_param_count(int net, int channels) {
  fg_c2f tmp;
  tmp.C = channels;
  make_layouts(&tmp);
  return net == FG_NET_D ? tmp.nD : tmp.nG;
}
int fg_c2f_mask_per_sample(void) { return kC2fMask; }

int fg_c2f_set_params(fg_c2f* n, int net, const float* src) {
  ENTER(n);
  FG_REQUIRE(src && (net == FG_NET_G || net == FG_NET_D), "fg_c2f_set_params: bad arguments");
  const bool isD = net == FG_NET_D;
  FG_CUDA(cudaMemcpyAsync(isD ? n->PD : n->PG, src, sizeof(float) * (isD ? n->nD : n->nG), cudaMemcpyDefault, n->c->stream));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  if (isD) n->D_packed = false; else n->G_packed = false;
  return FG_OK;
}
int fg_c2f_get_params(fg_c2f* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_c2f_get_params: bad arguments");
  const bool isD = net == FG_NET_D;
  return to_user(n->c, dst, isD ? n->PD : n->PG, isD ? n->nD : n->nG);
}
int fg_c2f_get_grads(fg_c2f* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_c2f_get_grads: bad arguments");
  const bool isD = net == FG_NET_D;
  return to_user(n->c, dst, isD ? n->gD : n->gG, isD ? n->nD : n->nG);
}
int fg_c2f_zero_grads(fg_c2f* n, int net) {
  ENTER(n);
  const bool isD = net == FG_NET_D;
  FG_CUDA(cudaMemsetAsync(isD ? n->gD : n->gG, 0, sizeof(float) * ((isD ? n->nD : n->nG) + kGradTail), n->c->stream));
  return FG_OK;
}
float* fg_c2f_params_ptr(fg_c2f* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->PD : n->PG); }
float* fg_c2f_grads_ptr(fg_c2f* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->gD : n->gG); }

int fg_c2f_set_adam_state(fg_c2f* n, int net, const float* m, const float* v, int t) {
  ENTER(n);
  const bool isD = net == FG_NET_D;
  const size_t cnt = isD ? n->nD : n->nG;
  if (m) FG_CUDA(cudaMemcpyAsync(isD ? n->mD : n->mG, m, sizeof(float) * cnt, cudaMemcpyDefault, n->c->stream));
  if (v) FG_CUDA(cudaMemcpyAsync(isD ? n->vD : n->vG, v, sizeof(float) * cnt, cudaMemcpyDefault, n->c->stream));
  FG_CUDA(cudaMemcpyAsync(isD ? &n->dstats->t_D : &n->dstats->t_G, &t, sizeof(int), cudaMemcpyHostToDevice, n->c->stream));
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}
int fg_c2f_get_adam_state(fg_c2f* n, int net, float* m, float* v, int* t) {
  ENTER(n);
  const bool isD = net == FG_NET_D;
  const size_t cnt = isD ? n->nD : n->nG;
  if (m) FG_TRY(to_user(n->c, m, isD ? n->mD : n->mG, cnt));
  if (v) FG_TRY(to_user(n->c, v, isD ? n->vD : n->vG, cnt));
  if (t) {
    FG_CUDA(cudaMemcpyAsync(t, isD ? &n->dstats->t_D : &n->dstats->t_G, sizeof(int), cudaMemcpyDeviceToHost, n->c->stream));
    FG_CUDA(cudaStreamSynchronize(n->c->stream));
  }
  return FG_OK;
}

int fg_c2f_G_forward(fg_c2f* n, const float* noise, const float* cond, int B, float* diff_out) {
  ENTER(n);
  FG_REQUIRE(noise && cond && B >= 1 && B <= n->maxB, "fg_c2f_G_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  const float *nd, *cd;
  FG_TRY(to_dev(n->c, noise, (size_t)B * 1024, n->in_c, &nd));
  FG_TRY(to_dev(n->c, cond, (size_t)B * n->C * 1024, n->in_b, &cd));
  FG_TRY(G_forward(n, nd, cd, B));
  if (diff_out) {
    FG_TRY(k_nhwc_to_nchw(n->c, n->G_z[4], n->io, B, n->C, 1024));
    FG_TRY(to_user(n->c, diff_out, n->io, (size_t)B * n->C * 1024));
  }
  return FG_OK;
}
int fg_c2f_G_backward(fg_c2f* n, const float* d_diff) {
  ENTER(n);
  FG_REQUIRE(d_diff, "fg_c2f_G_backward: null gradient");
  const float* dd;
  FG_TRY(to_dev(n->c, d_diff, (size_t)n->G_B * n->C * 1024, n->in_a, &dd));
  FG_TRY(k_nchw_to_nhwc(n->c, dd, n->io, n->G_B, n->C, 1024));
  return G_backward(n, n->io);
}
int fg_c2f_D_forward(fg_c2f* n, const float* diff, const float* cond, int B, int training, const float* masks,
                     uint64_t seed, float* out) {
  ENTER(n);
  FG_REQUIRE(diff && cond && B >= 1 && B <= n->maxB, "fg_c2f_D_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  fg_ctx* c = n->c;
  const float *dd, *cd;
  FG_TRY(to_dev(c, diff, (size_t)B * n->C * 1024, n->in_a, &dd));
  FG_TRY(to_dev(c, cond, (size_t)B * n->C * 1024, n->in_b, &cd));
  FG_TRY(k_nchw_to_nhwc(c, dd, n->io, B, n->C, 1024));
  FG_TRY(k_nchw_to_nhwc(c, cd, n->D_cond, B, n->C, 1024));
  if (training) {
    if (masks)
      FG_CUDA(cudaMemcpyAsync(n->D_masks, masks, sizeof(float) * (size_t)B * kC2fMask, cudaMemcpyDefault, c->stream));
    else
      FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * kC2fMask, seed, 0.5f));
  }
  FG_TRY(D_forward(n, n->io, n->D_cond, B, training != 0, 0.5f));
  FG_TRY(k_sigmoid_fwd(c, n->D_logit, n->D_out, B));
  if (out) FG_TRY(to_user(c, out, n->D_out, B));
  return FG_OK;
}
int fg_c2f_D_backward(fg_c2f* n, const float* d_out, int want_wgrad, float* d_diff) {
  ENTER(n);
  FG_REQUIRE(d_out, "fg_c2f_D_backward: null gradient");
  fg_ctx* c = n->c;
  const float* dd;
  FG_TRY(to_dev(c, d_out, (size_t)n->D_B, n->in_e, &dd));
  FG_TRY(k_sigmoid_bwd(c, dd, n->D_out, n->D_dlogit, n->D_B));
  FG_TRY(D_backward(n, n->D_dlogit, want_wgrad != 0, d_diff != nullptr));
  if (d_diff) {
    FG_TRY(k_nhwc_to_nchw(c, n->D_dx, n->io, n->D_B, n->C, 1024));
    FG_TRY(to_user(c, d_diff, n->io, (size_t)n->D_B * n->C * 1024));
  }
  return FG_OK;
}

// adversarial_c2f.lua:305-325 approxParzen, one sample: K generations G({noise_k, coarse}) + coarse for the SAME
// coarse image, the smallest torch.dist to the ground-truth fine image.  noise [K][1][32][32], coarse / fine
// [C][32][32] (host or device); *dist_out (host).
int fg_c2f_parzen_dist(fg_c2f* n, const float* noise, const float* coarse, const float* fine, int K, float* dist_out) {
  ENTER(n);
  FG_REQUIRE(noise && coarse && fine && dist_out && K >= 1 && K <= n->maxB, "fg_c2f_parzen_dist: bad arguments (K %d, max %d)", K,
             n->maxB);
  fg_ctx* c = n->c;
  const size_t img = (size_t)n->C * 1024;
  const float *nd, *fd;
  FG_TRY(to_dev(c, noise, (size_t)K * 1024, n->in_c, &nd));
  for (int k = 0; k < K; ++k)  // condInputs[i] = condInput:clone()  (:318-320)
    FG_CUDA(cudaMemcpyAsync(n->in_b + (size_t)k * img, coarse, img * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_TRY(G_forward(n, nd, n->in_b, K));
  FG_TRY(k_nchw_to_nhwc(c, n->in_b, n->D_cond, K, n->C, 1024));
  FG_TRY(k_add(c, n->G_z[4], n->D_cond, n->io, (int64_t)K * img));  // neighbors:add(condInputs)  (:322)
  FG_TRY(to_dev(c, fine, img, n->in_a, &fd));
  FG_TRY(k_nchw_to_nhwc(c, fd, n->in_d, 1, n->C, 1024));
  int32_t idx = 0;
  return fg_nearest(c, n->in_d, 1, n->io, K, (int)img, &idx, dist_out);
}

// data parallel: rank 0's c2f parameters, optimizer moments and step counters to every rank (the nets have no
// BatchNorm state); the communicator is the ctx's (fg_dp_init)
int fg_c2f_dp_broadcast_params(fg_c2f* n) {
  ENTER(n);
  fg_ctx* c = n->c;
  if (c->world <= 1) return FG_OK;
  FG_TRY(net_group(true));
  const size_t bG = n->nG * sizeof(float), bD = n->nD * sizeof(float);
  FG_TRY(net_broadcast(c, n->PG, bG));
  FG_TRY(net_broadcast(c, n->PD, bD));
  FG_TRY(net_broadcast(c, n->mG, bG));
  FG_TRY(net_broadcast(c, n->vG, bG));
  FG_TRY(net_broadcast(c, n->mD, bD));
  FG_TRY(net_broadcast(c, n->vD, bD));
  FG_TRY(net_broadcast(c, n->dstats, sizeof(DeviceStats)));
  FG_TRY(net_group(false));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  n->G_packed = n->D_packed = false;
  return FG_OK;
}

int fg_c2f_train_step(fg_c2f* n, const fg_hyper* h, int B, const float* real_diff, const float* cond_D,
                      const float* noise_D, const float* cond_G, const float* noise_G, const float* masks_D,
                      const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  FG_REQUIRE(h && real_diff && cond_D && noise_D && cond_G && noise_G, "fg_c2f_train_step: null input");
  FG_REQUIRE(B >= 4 && B % 2 == 0 && B <= n->maxB, "fg_c2f_train_step: batch %d must be even, >= 4 and <= max_batch %d", B,
             n->maxB);
  fg_ctx* c = n->c;
  const size_t img = (size_t)n->C * 1024;
  const float *rd, *cd, *nd, *cg, *ng, *md = nullptr, *mg = nullptr;
  FG_TRY(to_dev(c, real_diff, (size_t)(B / 2) * img, n->in_a, &rd));
  FG_TRY(to_dev(c, cond_D, (size_t)B * img, n->in_b, &cd));
  FG_TRY(to_dev(c, noise_D, (size_t)(B / 2) * 1024, n->in_c, &nd));
  FG_TRY(to_dev(c, cond_G, (size_t)B * img, n->in_d, &cg));
  FG_TRY(to_dev(c, noise_G, (size_t)B * 1024, n->in_e, &ng));
  if (masks_D) FG_TRY(to_dev(c, masks_D, (size_t)B * kC2fMask, n->in_m1, &md));
  if (masks_G) FG_TRY(to_dev(c, masks_G, (size_t)B * kC2fMask, n->in_m2, &mg));
  {  // eager the first time, then a captured CUDA graph of the step (nets.cu net_graph_run); the seed is read on the device
    std::vector<uint8_t> key;
    auto add = [&key](const void* p, size_t nb) { key.insert(key.end(), (const uint8_t*)p, (const uint8_t*)p + nb); };
    const void* ptrs[] = {rd, cd, nd, cg, ng, md, mg, (const void*)c->stream, c->nccl_comm};
    const int meta[3] = {c->graph_epoch, B, pack_key(c)};
    add(meta, sizeof(meta));
    add(h, sizeof(*h));
    add(ptrs, sizeof(ptrs));
    FG_TRY(net_graph_run(
        c, n->graphs, key, seed, [&]() { return train_step(n, h, B, rd, cd, nd, cg, ng, md, mg, 0); },
        [n]() { n->G_packed = n->D_packed = false; }, true));
  }
  if (stats) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    const DeviceStats& s = *n->hstats;
    stats->loss_D = s.loss_D;
    stats->loss_G = s.loss_G;
    for (int i = 0; i < 4; ++i) stats->conf[i] = s.conf[i];
    stats->trained_D = s.trained_D;
    stats->t_D = s.t_D;
    stats->t_G = s.t_G;
    stats->acc_D = s.acc_D;
  }
  return FG_OK;
}

}  // extern "C"
