// Orchestration of G (models.lua:57-81; gen.cu), D (models.lua:382-416) and their part of the adversarial.lua loop body
// (adversarial.lua:54-300; the loop itself is pair_train_step in netpair.cu) on one stream.  Kernels live in k_elem.cu / k_conv_simt.cu / k_conv_tc.cu.
#include <algorithm>

#include "convl.h"
#include "fg_internal.h"
#include "k_conv_tc.h"

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

namespace {
const int kDcin[4] = {0 /*C*/, 64, 128, 256}, kDcout[4] = {64, 128, 256, 512}, kDhw[4] = {32, 16, 8, 4};
const int kDmoff[4] = {0, 64, 192, 448};
inline int dcin(const fg_ctx* c, int i) { return i == 0 ? c->C : kDcin[i]; }

int dalloc(fg_ctx* c, float** p, size_t n) { return fg_dalloc(c, c->allocs, p, n); }
}  // namespace

int net_alloc(fg_ctx* c) {
  const size_t B = c->maxB, C = c->C;
  c->dl = make_d_layout(c->C);
  NetPair& p = c->net;
  FG_TRY(pair_alloc(c, c->allocs, p, make_g_layout(c->C, 32).total, c->dl.total, true));
  p.optim_timer[0] = "hbm.optim.G";
  p.optim_timer[1] = "hbm.optim.D";
  c->ownPG = p.PG; c->ownPD = p.PD; c->ownGG = p.gG; c->ownGD = p.gD;
  FG_TRY(dalloc(c, &c->tail_sep, 2 * kGradTail));
  float* tmp = nullptr;
  FG_TRY(dalloc(c, &c->lop_sx, 2));
  FG_TRY(dalloc(c, &c->lop_sy, 2));
  {
    float* sd = nullptr;
    FG_TRY(dalloc(c, &sd, 2 * kMaxIters));  // one stream root per iteration (k_seed_roots)
    c->seed_dev = reinterpret_cast<uint64_t*>(sd);
  }
  // the largest weight gradient: D.C4 / G's collapsed 5x5 layers; G.L1 on the tensor cores needs 8192 x (128 + 100)
  c->wgrad_ws_elems = std::max<size_t>(9 * 512 * 256, 8192 * (128 + kNoiseDim));
  FG_TRY(dalloc(c, &c->wgrad_ws, c->wgrad_ws_elems));
  c->splitk_ws_elems = (size_t)c->sm_count * 4 * 128 * 128;  // >= splits x output of every split-K weight gradient
  FG_TRY(dalloc(c, &c->splitk_ws, c->splitk_ws_elems));
  c->red_ws_elems = (size_t)4 << 20;  // >= blocks x partials of every ordered reduction (checked at each launch)
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->red_ws), 2 * c->red_ws_elems));
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->red_ws_opt), 2 * kOptRedRows));
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->red_ticket), 2));  // zeroed; every ordered reduction resets its ticket
  FG_TRY(dalloc(c, reinterpret_cast<float**>(&c->bwd_claim), 1));
  FG_TRY(dalloc(c, &c->small_ws, (size_t)kSmallMaxParts * 9 * 4 * 128));
  FG_TRY(dalloc(c, &tmp, 4 * 256 * 2));  // doubles
  c->bn_acc = (double*)tmp;
  FG_TRY(dalloc(c, &tmp, 32 * 4 * 256 * 2 + 64));  // doubles + tickets (zero-initialised)
  c->bn_slice_acc = (double*)tmp;
  FG_TRY(dalloc(c, &c->bn_parts, B * 3072));  // G.C2: 8 tiles/image x 3 x 128 ch; G.C1: 2 tiles/image x 3 x 256 ch
  // D activations
  FG_TRY(dalloc(c, &c->D_x, B * 1024 * C));
  for (int i = 0; i < 4; ++i) {
    const size_t n = B * (size_t)kDhw[i] * kDhw[i] * kDcout[i];
    FG_TRY(dalloc(c, &c->D_z[i], n));
    FG_TRY(dalloc(c, &c->D_p[i], n / 4));
  }
  FG_TRY(dalloc(c, &c->D_zl1, B * 512));
  FG_TRY(dalloc(c, &c->D_hl1, B * 512));
  FG_TRY(dalloc(c, &c->D_zl2, B * 512));
  FG_TRY(dalloc(c, &c->D_hl2, B * 512));
  FG_TRY(dalloc(c, &c->D_logit, B));
  FG_TRY(dalloc(c, &c->D_out, B));
  FG_TRY(dalloc(c, &c->D_masks, B * kMaskPerSample));
  FG_TRY(dalloc(c, &c->D_dlogit, B));
  FG_TRY(dalloc(c, &c->D_dh, B * 512));
  FG_TRY(dalloc(c, &c->D_dzl, B * 512));
  FG_TRY(dalloc(c, &c->D_dz, B * 65536));
  FG_TRY(dalloc(c, &c->D_dp, B * 16384));
  FG_TRY(dalloc(c, &c->D_dx, B * 1024 * C));
  FG_TRY(dalloc(c, &c->D_targets, B));
  c->io_dev_elems = std::max<size_t>(B * 1024 * C, B * kMaskPerSample);
  FG_TRY(dalloc(c, &c->io_dev, c->io_dev_elems));
  FG_TRY(dalloc(c, &c->io_dev2, c->io_dev_elems));
  {  // the layers (convl.h) and the scratch they share
    ConvLEnv& e = c->env;
    e.c = c;
    e.maxB = c->maxB;
    e.allocs = &c->allocs;
    e.ws = c->wgrad_ws;
    FG_TRY(dalloc(c, &e.dy.hi, B * 131072));
    FG_TRY(dalloc(c, &e.dy.lo, B * 131072));
    static const GenDesc g32{32, "", 128, true};  // G.L1 padded to K = 128 for the tensor cores; G.C1 / G.C2 may merge
    FG_TRY(gen_alloc(e, c->G, g32));
    ScalePairs& sp = c->D_pairs;  // every FP16-split operand of D gets its own scale pair
    FG_TRY(sp.alloc(c, c->allocs, 1 + 2 * 6));
    FG_TRY(sp.take(&e.dy.s));
    const DLayout& dl = c->dl;
    auto conv = [&](ConvL& L, int Cin, int Cout, int k, int H, int64_t w_off, int64_t b_off, const char* tf, const char* td,
                    const char* tw) {
      L.Cin = Cin; L.Cout = Cout; L.k = k; L.H = H;
      L.w_off = w_off; L.b_off = b_off;
      L.tf = tf; L.td = td; L.tw = tw;
    };
    static const char* tf[4] = {"D.C1.fwd", "D.C2.fwd", "D.C3.fwd", "D.C4.fwd"};
    static const char* td[4] = {"D.C1.dgrad", "D.C2.dgrad", "D.C3.dgrad", "D.C4.dgrad"};
    static const char* tw[4] = {"D.C1.wgrad", "D.C2.wgrad", "D.C3.wgrad", "D.C4.wgrad"};
    for (int i = 0; i < 4; ++i) conv(c->Dc[i], dcin(c, i), kDcout[i], 3, kDhw[i], dl.cW[i], dl.cb[i], tf[i], td[i], tw[i]);
    conv(c->DL1, 2048, 512, 1, 1, dl.L1W, dl.L1b, "D.L1.fwd", "D.L1.dgrad", "D.L1.wgrad");
    c->DL1.cA = 512; c->DL1.cS = 4;  // View(2048) flattens [512][2][2] in (c,h,w) order; ours is NHWC (h,w,c)
    conv(c->DL2, 512, 512, 1, 1, dl.L2W, dl.L2b, "D.L2.fwd", "D.L2.dgrad", "D.L2.wgrad");
    for (ConvL* L : {&c->Dc[0], &c->Dc[1], &c->Dc[2], &c->Dc[3], &c->DL1, &c->DL2}) {
      FG_TRY(sp.take(&L->x.s));
      FG_TRY(sp.take(&L->sdy));
      FG_TRY(convl_alloc(e, *L));
    }
  }
  FG_TRY(dalloc(c, &c->in_noiseD, B * kNoiseDim));
  FG_TRY(dalloc(c, &c->in_noiseG, B * kNoiseDim));
  p.keep = {{"Dstep.z1", c->D_z[0], 65536}, {"Dstep.z2", c->D_z[1], 32768}, {"Dstep.z3", c->D_z[2], 16384},
            {"Dstep.z4", c->D_z[3], 8192},  {"Dstep.zl1", c->D_zl1, 512},    {"Dstep.zl2", c->D_zl2, 512},
            {"Dstep.logit", c->D_logit, 1}, {"Dstep.out", c->D_out, 1}};
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

void net_free(fg_ctx* c) {
  pair_free(c->net);
  for (void* p : c->allocs) cudaFree(p);
  c->allocs.clear();
  if (c->stage_pinned) cudaFreeHost(c->stage_pinned);
  for (int i = 0; i < 8; ++i)
    if (c->scratch[i]) cudaFree(c->scratch[i]);
}

int net_pack_D(fg_ctx* c) {
  if (c->net.D_packed) return FG_OK;
  for (int i = 0; i < 4; ++i) FG_TRY(convl_pack(c, c->Dc[i], c->net.PD));
  FG_TRY(convl_pack(c, c->DL1, c->net.PD));
  FG_TRY(convl_pack(c, c->DL2, c->net.PD));
  c->net.D_packed = true;
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// D
// ---------------------------------------------------------------------------------------------------
int net_D_forward(fg_ctx* c, const float* x, int B, bool training, const fg_hyper* h) {
  FG_REQUIRE(B >= 1 && B <= c->maxB, "D forward: batch %d out of range [1,%d]", B, c->maxB);
  FG_TRY(net_pack_D(c));
  FG_TRY(c->D_pairs.reset(c));
  const DLayout& L = c->dl;
  float* P = c->net.PD;
  if (x != c->D_x)
    FG_CUDA(cudaMemcpyAsync(c->D_x, x, sizeof(float) * (size_t)B * 1024 * c->C, cudaMemcpyDeviceToDevice, c->stream));
  c->D_B = B;
  c->D_train = training;
  const float* masks = training ? c->D_masks : nullptr;
  const float* cur = c->D_x;
  for (int i = 0; i < 4; ++i) {
    const int H = kDhw[i];
    FG_TRY(convl_fwd(c->env, c->Dc[i], cur, P, c->D_z[i], B));
    // the pooled activation is the next layer's tensor-core operand: its TF32 split (or max|p|) comes out of the same kernel
    TcOp& nx = (i < 3 ? c->Dc[i + 1] : c->DL1).x;
    nx.split_ready = convl_tc_fwd(c, i < 3 ? c->Dc[i + 1] : c->DL1) && !tc_f16(c);
    {
      AmaxInto am(c, nx);
      FG_TRY(k_d_act_pool_fwd(c, c->D_z[i], P + L.ca[i], masks, kDmoff[i], 1.0f - h->p_spatial, c->D_p[i], B, H, H,
                              kDcout[i], nx.split_ready ? nx.hi : nullptr, nx.split_ready ? nx.lo : nullptr));
    }
    cur = c->D_p[i];
  }
  const float scale = 1.0f / (1.0f - h->p_drop);
  c->D_drop_scale = scale;
  c->D_spatial_eval = 1.0f - h->p_spatial;
  FG_TRY(convl_fwd(c->env, c->DL1, c->D_p[3], P, c->D_zl1, B));
  {
    AmaxInto am(c, c->DL2.x);
    FG_TRY(k_lin_act_drop_fwd(c, c->D_zl1, P + L.a5, masks, 960, scale, c->D_hl1, B, 512));
  }
  FG_TRY(convl_fwd(c->env, c->DL2, c->D_hl1, P, c->D_zl2, B));
  FG_TRY(k_lin_act_drop_fwd(c, c->D_zl2, P + L.a6, masks, 1472, scale, c->D_hl2, B, 512));
  {
    ScopedTimer tm(c, "D.L3.fwd");
    FG_TRY(k_gemv_fwd(c, c->D_hl2, P + L.L3W, P + L.L3b, c->D_logit, B, 512));
  }
  c->D_fwd_valid = true;
  return FG_OK;
}

int net_D_backward(fg_ctx* c, const float* dlogit, bool want_wgrad, bool want_dx) {
  if (!c->D_fwd_valid) {
    fg_set_error("D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const DLayout& L = c->dl;
  float *P = c->net.PD, *G = c->net.gD;
  const int B = c->D_B;
  const float* masks = c->D_train ? c->D_masks : nullptr;
  const float scale = c->D_drop_scale, eval_scale = c->D_spatial_eval;
  FG_TRY(c->D_pairs.reset(c));
  // L3
  if (want_wgrad) {
    ScopedTimer tm(c, "D.L3.wgrad");
    FG_TRY(k_gemv_wgrad_add(c, c->D_hl2, dlogit, G + L.L3W, G + L.L3b, B, 512));
  }
  {
    ScopedTimer tm(c, "D.L3.dgrad");
    FG_TRY(k_gemv_dgrad(c, dlogit, P + L.L3W, c->D_dh, B, 512));
  }
  TcOp& dy = c->env.dy;  // the producers below say in its flags what they already did for the layer that follows
  float* GD = want_wgrad ? G : nullptr;
  {
    AmaxInto am(c, c->DL2.sdy, &dy.amax_ready);
    FG_TRY(k_lin_act_drop_bwd(c, c->D_dh, c->D_zl2, P + L.a6, masks, 1472, scale, c->D_dzl, want_wgrad ? G + L.a6 : nullptr, B,
                              512));
  }
  FG_TRY(convl_bwd(c->env, c->DL2, c->D_hl1, c->D_dzl, GD, c->D_dh, B));
  {
    AmaxInto am(c, c->DL1.sdy, &dy.amax_ready);
    FG_TRY(k_lin_act_drop_bwd(c, c->D_dh, c->D_zl1, P + L.a5, masks, 960, scale, c->D_dzl, want_wgrad ? G + L.a5 : nullptr, B,
                              512));
  }
  FG_TRY(convl_bwd(c->env, c->DL1, c->D_p[3], c->D_dzl, GD, c->D_dp, B));
  for (int i = 3; i >= 0; --i) {
    const int H = kDhw[i];
    // dz and, for the tensor-core layers, its TF32 split in one pass, + the conv bias gradient (column sums of dz)
    dy.split_ready = convl_tc_bwd(c, c->Dc[i]) && !tc_f16(c);
    dy.bias_ready = want_wgrad;
    {
      AmaxInto am(c, c->Dc[i].sdy, &dy.amax_ready);
      FG_TRY(k_d_act_pool_bwd(c, c->D_dp, c->D_z[i], P + L.ca[i], masks, kDmoff[i], eval_scale, c->D_dz,
                              want_wgrad ? G + L.ca[i] : nullptr, B, H, H, kDcout[i], dy.split_ready ? dy.hi : nullptr,
                              dy.split_ready ? dy.lo : nullptr, want_wgrad ? G + L.cb[i] : nullptr));
    }
    float* din = i > 0 ? c->D_dp : want_dx ? c->D_dx : nullptr;
    FG_TRY(convl_bwd(c->env, c->Dc[i], i == 0 ? c->D_x : c->D_p[i - 1], c->D_dz, GD, din, B));
  }
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// the 32x32 nets in the adversarial.lua loop body (pair_train_step, netpair.cu)
// ---------------------------------------------------------------------------------------------------
NetStep::NetStep(fg_ctx* c, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG)
    : StepNets(c, c->net, h, B, c->D_logit, c->D_out, c->D_dlogit, c->D_masks, kMaskPerSample, true, true),
      real(real), noiseD(noiseD), noiseG(noiseG) {}
int NetStep::g_forward(int j, bool d_iter) {
  const int n = d_iter ? B / 2 : B;
  return gen_forward(c->env, c->G, c->net, (d_iter ? noiseD : noiseG) + (size_t)j * n * kNoiseDim, n, true);
}
int NetStep::d_input(int j) {
  const int Bh = B / 2;
  const size_t img = (size_t)c->C * 1024;
  FG_TRY(k_nchw_to_nhwc(c, real + (size_t)j * Bh * img, c->D_x, Bh, c->C, 1024));
  FG_CUDA(cudaMemcpyAsync(c->D_x + Bh * img, c->G.y, sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
  return FG_OK;
}
int NetStep::draw_masks(int kind, const uint64_t* root) { return k_masks_generate(c, c->D_masks, B, kind, h->p_spatial, h->p_drop, root); }
int NetStep::d_forward(bool on_g) { return net_D_forward(c, on_g ? c->G.y : c->D_x, B, true, h); }
int NetStep::d_backward(bool want_wgrad, bool want_dx) { return net_D_backward(c, c->D_dlogit, want_wgrad, want_dx); }
int NetStep::g_backward() { return gen_backward(c->env, c->G, c->net, c->D_dx, nullptr); }
