// The 32x32 nets of train.lua and their C entry points: G (models.lua:57-81; gen.cu), D (models.lua:382-416) and their
// trainer (UpsGan, ups_gan.cu) on one stream.  Kernels live in k_elem.cu / k_conv_simt.cu / k_conv_tc.cu.
#include <algorithm>

#include "fg_internal.h"
#include "k_conv_tc.h"
#include "ups_gan.h"

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

// D of the 32x32 nets (create_D32b): 4 x (conv 3x3, PReLU, SpatialDropout, average pool 2), View(2048), 2 x (Linear(512),
// PReLU, Dropout), Linear(1); D.L3 runs on the GEMV kernels.  Activations NHWC.
struct D32 final : GanD {
  DLayout dl;
  ConvL Dc[4], DL1, DL2;
  ScalePairs pairs;  // every FP16-split operand of D gets its own scale pair, env.dy's included
  bool train = true, fwd_valid = false;
  float *z[4] = {nullptr, nullptr, nullptr, nullptr}, *p[4] = {nullptr, nullptr, nullptr, nullptr};
  float *zl1 = nullptr, *hl1 = nullptr, *zl2 = nullptr, *hl2 = nullptr;
  float drop_scale = 2.0f, spatial_eval = 0.8f;  // 1/(1-p_drop), 1-p_spatial of the last forward
  float *dh = nullptr, *dz = nullptr, *dp = nullptr;
  float *dzl2 = nullptr, *dzl1 = nullptr;  // D.L2's and D.L1's dY: their bias gradients may still read them (bwd_streams)
  // option "debug_keep" (tests): the backward reuses dh / dp / dz across layers, so backward() copies each one as
  // a kernel wrote it ("Dbwd.*" debug tensors, the last D backward; Keep::src is unused here)
  std::vector<NetPair::Keep> bwd_keep;
  int bwd_keep_B = 0;

  ~D32() override {
    for (NetPair::Keep& k : bwd_keep)
      if (k.copy) cudaFree(k.copy);
  }
  int64_t layout(int C) override {
    dl = make_d_layout(C);
    return dl.total;
  }
  int dalloc(float** q, size_t elems) { return convl_dalloc(n->env, q, elems); }
  int alloc() override;
  int forward(const float* x, int B, bool training, const fg_hyper* h) override;
  int keep_bwd(int k, const float* src, int B);
  int backward(bool want_wgrad, bool want_dx) override;
  int draw_masks(int B, uint64_t seed, const fg_hyper* h, const uint64_t* root) override {
    return k_masks_generate(n->c, masks, B, seed, h->p_spatial, h->p_drop, root);
  }
  void debug_rows(std::vector<DebugTensor>& ents) const override;
};

int D32::alloc() {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  const size_t B = c->maxB, C = c->C;
  // the largest weight gradient: D.C4 / G's collapsed 5x5 layers; G.L1 on the tensor cores needs 8192 x (128 + 100)
  FG_TRY(dalloc(&e.ws, std::max<size_t>(9 * 512 * 256, 8192 * (128 + kNoiseDim))));
  FG_TRY(dalloc(&x, B * 1024 * C));
  for (int i = 0; i < 4; ++i) {
    const size_t n_z = B * (size_t)kDhw[i] * kDhw[i] * kDcout[i];
    FG_TRY(dalloc(&z[i], n_z));
    FG_TRY(dalloc(&p[i], n_z / 4));
  }
  FG_TRY(dalloc(&zl1, B * 512));
  FG_TRY(dalloc(&hl1, B * 512));
  FG_TRY(dalloc(&zl2, B * 512));
  FG_TRY(dalloc(&hl2, B * 512));
  FG_TRY(dalloc(&logit, B));
  FG_TRY(dalloc(&out, B));
  FG_TRY(dalloc(&masks, B * kMaskPerSample));
  FG_TRY(dalloc(&dlogit, B));
  FG_TRY(dalloc(&dh, B * 512));
  FG_TRY(dalloc(&dzl2, B * 512));
  FG_TRY(dalloc(&dzl1, B * 512));
  FG_TRY(dalloc(&dz, B * 65536));
  FG_TRY(dalloc(&dp, B * 16384));
  FG_TRY(dalloc(&dx, B * 1024 * C));
  // the split of every dY of G and D: the largest is G.C2's [B][32][32][128]
  FG_TRY(dalloc(&e.dy.hi, B * 131072));
  FG_TRY(dalloc(&e.dy.lo, B * 131072));
  FG_TRY(pairs.alloc(c, n->allocs, 1 + 2 * 6));
  FG_TRY(pairs.take(&e.dy.s));
  auto conv = [&](ConvL& L, int Cin, int Cout, int k, int H, int64_t w_off, int64_t b_off, const char* tf, const char* td,
                  const char* tw) {
    L.Cin = Cin; L.Cout = Cout; L.k = k; L.H = H;
    L.w_off = w_off; L.b_off = b_off;
    L.tf = tf; L.td = td; L.tw = tw;
  };
  static const char* tf[4] = {"D.C1.fwd", "D.C2.fwd", "D.C3.fwd", "D.C4.fwd"};
  static const char* td[4] = {"D.C1.dgrad", "D.C2.dgrad", "D.C3.dgrad", "D.C4.dgrad"};
  static const char* tw[4] = {"D.C1.wgrad", "D.C2.wgrad", "D.C3.wgrad", "D.C4.wgrad"};
  for (int i = 0; i < 4; ++i) conv(Dc[i], dcin(c, i), kDcout[i], 3, kDhw[i], dl.cW[i], dl.cb[i], tf[i], td[i], tw[i]);
  conv(DL1, 2048, 512, 1, 1, dl.L1W, dl.L1b, "D.L1.fwd", "D.L1.dgrad", "D.L1.wgrad");
  DL1.cA = 512; DL1.cS = 4;  // View(2048) flattens [512][2][2] in (c,h,w) order; ours is NHWC (h,w,c)
  conv(DL2, 512, 512, 1, 1, dl.L2W, dl.L2b, "D.L2.fwd", "D.L2.dgrad", "D.L2.wgrad");
  for (ConvL* L : {&Dc[0], &Dc[1], &Dc[2], &Dc[3], &DL1, &DL2}) {
    FG_TRY(pairs.take(&L->x.s));
    FG_TRY(pairs.take(&L->sdy));
    FG_TRY(convl_alloc(e, *L));
  }
  // the tensor-core layers split their dY into buffers of their own: with option bwd_streams a weight gradient on the
  // wgrad stream still reads a layer's split while the chain splits the next layer's dY
  for (ConvL* L : {&Dc[1], &Dc[2], &Dc[3], &DL1, &DL2}) {
    const size_t n_dy = B * (size_t)L->H * L->H * L->Cout;
    FG_TRY(dalloc(&L->dy_hi, n_dy));
    FG_TRY(dalloc(&L->dy_lo, n_dy));
  }
  n->net.keep = {{"Dstep.z1", z[0], 65536}, {"Dstep.z2", z[1], 32768}, {"Dstep.z3", z[2], 16384},
                 {"Dstep.z4", z[3], 8192},  {"Dstep.zl1", zl1, 512},    {"Dstep.zl2", zl2, 512},
                 {"Dstep.logit", logit, 1}, {"Dstep.out", out, 1}};
  bwd_keep = {{"Dbwd.dh3", nullptr, 512},    {"Dbwd.dzl2", nullptr, 512},  {"Dbwd.dh2", nullptr, 512},
              {"Dbwd.dzl1", nullptr, 512},   {"Dbwd.dp4", nullptr, 2048},  {"Dbwd.dz4", nullptr, 8192},
              {"Dbwd.dp3", nullptr, 4096},   {"Dbwd.dz3", nullptr, 16384}, {"Dbwd.dp2", nullptr, 8192},
              {"Dbwd.dz2", nullptr, 32768},  {"Dbwd.dp1", nullptr, 16384}, {"Dbwd.dz1", nullptr, 65536}};
  return FG_OK;
}

int D32::forward(const float* xin, int Bn, bool training, const fg_hyper* h) {
  fg_ctx* c = n->c;
  FG_REQUIRE(Bn >= 1 && Bn <= c->maxB, "D forward: batch %d out of range [1,%d]", Bn, c->maxB);
  FG_TRY(gan_pack_D(*n, {&Dc[0], &Dc[1], &Dc[2], &Dc[3], &DL1, &DL2}));
  FG_TRY(pairs.reset(c));
  const DLayout& L = dl;
  float* P = n->net.PD;
  ConvLEnv& e = n->env;
  if (xin != x) FG_CUDA(cudaMemcpyAsync(x, xin, sizeof(float) * (size_t)Bn * 1024 * c->C, cudaMemcpyDeviceToDevice, c->stream));
  B = Bn;
  train = training;
  const float* m = training ? masks : nullptr;
  const float* cur = x;
  for (int i = 0; i < 4; ++i) {
    const int H = kDhw[i];
    FG_TRY(convl_fwd(e, Dc[i], cur, P, z[i], B));
    // the pooled activation is the next layer's tensor-core operand: its TF32 split (or max|p|) comes out of the same kernel
    TcOp& nx = (i < 3 ? Dc[i + 1] : DL1).x;
    nx.split_ready = convl_tc_fwd(c, i < 3 ? Dc[i + 1] : DL1) && !tc_f16(c);
    {
      AmaxInto am(c, nx);
      FG_TRY(k_d_act_pool_fwd(c, z[i], P + L.ca[i], m, kDmoff[i], 1.0f - h->p_spatial, p[i], B, H, H, kDcout[i],
                              nx.split_ready ? nx.hi : nullptr, nx.split_ready ? nx.lo : nullptr));
    }
    cur = p[i];
  }
  const float scale = 1.0f / (1.0f - h->p_drop);
  drop_scale = scale;
  spatial_eval = 1.0f - h->p_spatial;
  FG_TRY(convl_fwd(e, DL1, p[3], P, zl1, B));
  {
    AmaxInto am(c, DL2.x);
    FG_TRY(k_lin_act_drop_fwd(c, zl1, P + L.a5, m, 960, scale, hl1, B, 512));
  }
  FG_TRY(convl_fwd(e, DL2, hl1, P, zl2, B));
  FG_TRY(k_lin_act_drop_fwd(c, zl2, P + L.a6, m, 1472, scale, hl2, B, 512));
  {
    ScopedTimer tm(c, "D.L3.fwd");
    FG_TRY(k_gemv_fwd(c, hl2, P + L.L3W, P + L.L3b, logit, B, 512));
  }
  fwd_valid = true;
  return FG_OK;
}

// option "debug_keep": bwd_keep[k].copy = the first B samples of src, bit for bit (allocated by the first use)
int D32::keep_bwd(int k, const float* src, int Bn) {
  fg_ctx* c = n->c;
  if (!c->debug_keep) return FG_OK;
  NetPair::Keep& e = bwd_keep[k];
  if (!e.copy) FG_CUDA(cudaMalloc((void**)&e.copy, sizeof(float) * c->maxB * e.per));
  FG_CUDA(cudaMemcpyAsync(e.copy, src, sizeof(float) * Bn * e.per, cudaMemcpyDeviceToDevice, c->stream));
  bwd_keep_B = Bn;
  return FG_OK;
}

int D32::backward(bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  if (!fwd_valid) {
    fg_set_error("D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const DLayout& L = dl;
  float *P = n->net.PD, *G = n->net.gD;
  const float* m = train ? masks : nullptr;
  const float scale = drop_scale, eval_scale = spatial_eval;
  ConvLEnv& e = n->env;
  FG_TRY(pairs.reset(c));
  // option bwd_streams: the weight gradients of D.L3 to D.C2 (and the bias gradients of the Linear layers) on the wgrad
  // stream, beside the data-gradient chain; each reads only its layer's input split and own dY (dY split, dzl2 /
  // dzl1), which the chain leaves alone until the join at the end.  D.C1's stays on the chain: nothing follows it there.
  const bool side = want_wgrad && wgrad_async(c, e);
  // L3
  if (want_wgrad) {
    OnWgradStream ws(e, side);
    FG_TRY(ws.r);
    ScopedTimer tm(c, "D.L3.wgrad");
    FG_TRY(k_gemv_wgrad_add(c, hl2, dlogit, G + L.L3W, G + L.L3b, B, 512));
  }
  {
    ScopedTimer tm(c, "D.L3.dgrad");
    FG_TRY(k_gemv_dgrad(c, dlogit, P + L.L3W, dh, B, 512));
  }
  FG_TRY(keep_bwd(0, dh, B));
  TcOp& dy = e.dy;  // the producers below say in its flags what they already did for the layer that follows
  float* GD = want_wgrad ? G : nullptr;
  {
    AmaxInto am(c, DL2.sdy, &dy.amax_ready);
    FG_TRY(k_lin_act_drop_bwd(c, dh, zl2, P + L.a6, m, 1472, scale, dzl2, want_wgrad ? G + L.a6 : nullptr, B, 512));
  }
  FG_TRY(keep_bwd(1, dzl2, B));
  FG_TRY(convl_bwd(e, DL2, hl1, dzl2, GD, dh, B, side));
  FG_TRY(keep_bwd(2, dh, B));
  {
    AmaxInto am(c, DL1.sdy, &dy.amax_ready);
    FG_TRY(k_lin_act_drop_bwd(c, dh, zl1, P + L.a5, m, 960, scale, dzl1, want_wgrad ? G + L.a5 : nullptr, B, 512));
  }
  FG_TRY(keep_bwd(3, dzl1, B));
  FG_TRY(convl_bwd(e, DL1, p[3], dzl1, GD, dp, B, side));
  for (int i = 3; i >= 0; --i) {
    const int H = kDhw[i];
    FG_TRY(keep_bwd(4 + 2 * (3 - i), dp, B));  // "Dbwd.dp<i+1>": the input of layer i's act/pool backward
    // dz and, for the tensor-core layers, its TF32 split in one pass, + the conv bias gradient (column sums of dz)
    ConvL& Li = Dc[i];
    dy.split_ready = convl_tc_bwd(c, Li) && !tc_f16(c);
    dy.bias_ready = want_wgrad;
    float *dy_hi = Li.dy_hi ? Li.dy_hi : dy.hi, *dy_lo = Li.dy_lo ? Li.dy_lo : dy.lo;
    {
      AmaxInto am(c, Li.sdy, &dy.amax_ready);
      FG_TRY(k_d_act_pool_bwd(c, dp, z[i], P + L.ca[i], m, kDmoff[i], eval_scale, dz, want_wgrad ? G + L.ca[i] : nullptr, B,
                              H, H, kDcout[i], dy.split_ready ? dy_hi : nullptr, dy.split_ready ? dy_lo : nullptr,
                              want_wgrad ? G + L.cb[i] : nullptr));
    }
    FG_TRY(keep_bwd(5 + 2 * (3 - i), dz, B));
    float* din = i > 0 ? dp : want_dx ? dx : nullptr;
    // off the tensor cores the weight gradient reads dz, which the next layer overwrites: on the chain then
    FG_TRY(convl_bwd(e, Li, i == 0 ? x : p[i - 1], dz, GD, din, B, side && i > 0 && convl_tc_wgrad(c, Li)));
  }
  return wgrad_join(e);
}

void D32::debug_rows(std::vector<DebugTensor>& ents) const {
  const int db = B;
  ents.insert(ents.end(), {{"D.z1", z[0], 65536, db}, {"D.z2", z[1], 32768, db}, {"D.z3", z[2], 16384, db},
                           {"D.z4", z[3], 8192, db}, {"D.p1", p[0], 16384, db}, {"D.p2", p[1], 8192, db},
                           {"D.p3", p[2], 4096, db}, {"D.p4", p[3], 2048, db}, {"D.logit", logit, 1, db},
                           {"D.out", out, 1, db}, {"D.dx", dx, 1024 * n->c->C, db}, {"D.masks", masks, kMaskPerSample, db},
                           {"D.zl1", zl1, 512, db}, {"D.hl1", hl1, 512, db}, {"D.zl2", zl2, 512, db},
                           {"D.hl2", hl2, 512, db}, {"D.dlogit", dlogit, 1, db}});
  for (const NetPair::Keep& k : bwd_keep) ents.push_back({k.name, k.copy, k.per, bwd_keep_B});
}
}  // namespace

// the 32x32 trainer and what fg_bind_params swaps: the library's own allocations (net.PG.. point here unless
// fg_bind_params borrowed caller-owned buffers) and the 8 DP-reduced scalars behind a bound gradient (behind the own
// gradient buffer they are contiguous with it)
struct Net32 : UpsGan {
  float *ownPG = nullptr, *ownPD = nullptr, *ownGG = nullptr, *ownGD = nullptr;
  float* tail_sep = nullptr;
};

int net32_alloc(fg_ctx* c, int disc) {
  Net32* n = c->n32 = new Net32();
  n->disc = disc;
  // G.L1 padded to K = 128 for the tensor cores; G.C1 / G.C2 may merge
  const bool b = disc == FG_DISC_D32B;
  const GanDesc k32{{32, "", 128, true}, b ? kMaskPerSample : dbr_mask_per_sample(disc), true};
  FG_TRY(gan_alloc(*n, c, k32, b ? std::make_unique<D32>() : dbr_make(disc), c->io_dev));
  NetPair& p = n->net;
  p.optim_timer[0] = "hbm.optim.G";
  p.optim_timer[1] = "hbm.optim.D";
  n->ownPG = p.PG; n->ownPD = p.PD; n->ownGG = p.gG; n->ownGD = p.gD;
  FG_TRY(fg_dalloc(c, n->allocs, &n->tail_sep, 2 * kGradTail));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
void net32_free(fg_ctx* c) {
  if (!c->n32) return;
  gan_free(*c->n32);
  delete c->n32;
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
// gan_train_step_iters on the 32x32 nets, for the entry `what`
int train_step_iters(fg_ctx* c, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                     const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                     fg_step_stats* stats) {
  ENTER(c);
  return gan_train_step_iters(*c->n32, what, h, B, d_iters, g_iters, real, noise_D, noise_G, masks_D, masks_G, seed, stats);
}

// gan_train_step_dataset_iters on the 32x32 nets, for the entry `what`
int train_step_dataset_iters(fg_ctx* c, fg_dataset* d, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters,
                             uint64_t seed, fg_step_stats* stats) {
  if (!d || !d->c) {
    fg_set_error("null fg_dataset");
    return FG_ERR_INVALID;
  }
  FG_CUDA(cudaSetDevice(d->c->device));
  if (!c) return step_check(c, what, B, d_iters, g_iters, h, d, true);  // fails: the dataset belongs to another context
  return gan_train_step_dataset_iters(*c->n32, d, what, h, B, d_iters, g_iters, seed, stats);
}
}  // namespace

extern "C" {

int fg_get_disc(fg_ctx* c) {
  if (!c) {
    fg_set_error("null fg_ctx");
    return FG_ERR_INVALID;
  }
  return c->n32->disc;
}
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
  c->n32->net.G_pack = -1;  // parameters may have been edited through fg_params_ptr()
  return gan_G_forward(*c->n32, noise, B, training != 0, images_out);
}
int fg_G_backward(fg_ctx* c, const float* d_images, float* d_noise) {
  ENTER(c);
  FG_REQUIRE(d_images, "fg_G_backward: d_images is null");
  return gan_G_backward(*c->n32, d_images, d_noise);
}
int fg_D_forward(fg_ctx* c, const float* images, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(c);
  FG_REQUIRE(images && B >= 1 && B <= c->maxB, "fg_D_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  c->n32->net.D_pack = -1;
  return gan_D_forward(*c->n32, images, B, training != 0, masks, seed, out);
}
int fg_D_backward(fg_ctx* c, const float* d_out, int want_wgrad, float* d_images) {
  ENTER(c);
  FG_REQUIRE(d_out, "fg_D_backward: d_out is null");
  return gan_D_backward(*c->n32, d_out, want_wgrad != 0, d_images);
}
int fg_bce_forward(fg_ctx* c, const float* x, const float* t, int n, float* loss_out) {
  ENTER(c);
  FG_REQUIRE(x && t && loss_out && n > 0 && n <= c->maxB, "fg_bce_forward: bad arguments");
  const float *xd, *td;
  FG_TRY(fg_to_dev(c, x, n, c->n32->img[0], &xd));
  FG_TRY(fg_to_dev(c, t, n, c->n32->img[1], &td));
  FG_TRY(k_bce_fwd(c, xd, td, n, c->n32->z[0]));
  return fg_to_user(c, loss_out, c->n32->z[0], 1);
}
int fg_bce_backward(fg_ctx* c, const float* x, const float* t, int n, float* dx) {
  ENTER(c);
  FG_REQUIRE(x && t && dx && n > 0 && n <= c->maxB, "fg_bce_backward: bad arguments");
  const float *xd, *td;
  FG_TRY(fg_to_dev(c, x, n, c->n32->img[0], &xd));
  FG_TRY(fg_to_dev(c, t, n, c->n32->img[1], &td));
  FG_TRY(k_bce_bwd(c, xd, td, n, c->n32->z[0]));
  return fg_to_user(c, dx, c->n32->z[0], n);
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
    FG_TRY(fg_to_dev(c, noise + (size_t)s * kNoiseDim, (size_t)b * kNoiseDim, n->z[0], &nd));
    // sample.lua never calls :evaluate() => BatchNorm uses the statistics of each chunk (SURVEY 3.4)
    FG_TRY(gen_forward(n->env, n->G, n->net, nd, b, true));
    float* dst = images_out + (size_t)s * img;
    if (out_dev) {
      FG_TRY(k_nhwc_to_nchw(c, n->G.y, dst, b, c->C, 1024));
    } else {
      FG_TRY(k_nhwc_to_nchw(c, n->G.y, n->img[0], b, c->C, 1024));
      FG_CUDA(cudaMemcpyAsync(dst, n->img[0], b * img * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
      if (s + chunk < N) FG_CUDA(cudaStreamSynchronize(c->stream));  // img[0] is reused by the next chunk
    }
  }
  if (!out_dev) FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int64_t fg_debug_tensor(fg_ctx* c, const char* name, float* dst, int64_t max_elems) {
  if (!c || !name) return -1;
  return gan_debug_tensor(*c->n32, "fg_debug_tensor", name, dst, max_elems);
}

}  // extern "C"
