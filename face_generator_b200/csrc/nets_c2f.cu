// Coarse-to-fine GAN (BASELINE configs[3], train_c2f.lua) on the same kernels as the 32x32 nets, at fine size
// S = train_c2f.lua --fineSize in {16, 32, 64} (the pyramid levels a 64x64 training set feeds), with any of
// models_c2f.lua's generators and discriminators (the default pair: create_G_d / create_D_c):
//   G = JoinTable{noise[1xSxS], coarse[CxSxS]} -> SCU(C+1->c1,k1) PReLU ... SCU(->C,kn)          (all at SxS)
//       create_G_d (:113-145) (64,3) (64,3) (128,5) (256,5) (C,7); create_G_a (:16-45) (64,3) (128,7) (C,5);
//       create_G_b (:47-78) (64,3) (64,3) (256,5) (C,7); create_G_c (:80-111) (64,3) (128,3) (256,5) (C,7)
//   D = CAddTable{diff, coarse} -> conv(C->c1,3) PReLU [MaxPool2] ... Dropout View Linear(512) PReLU Dropout Linear(1)
//       Sigmoid; create_D_c (:237-278) (64,-) (64,pool) (128,-) (256,pool); create_D_a (:156-192) (64,-) (64,pool);
//       create_D_b (:194-235) (64,-) (64,pool) (128,-) (128,pool)
//   loop = adversarial_c2f.lua:121-187 (fevalD :40-81, fevalG_on_D :85-116, optim.adam)
// cudnn.SpatialConvolutionUpsample with factor 1 (layers/cudnnSpatialConvolutionUpsample.lua:4-28) is a "same"
// convolution whose output view is the identity, so every layer maps onto the tap-GEMM convolution kernels through
// ConvL: wgmma (chunk-promoted 3xFP16 / 3xTF32) where the channel counts make a dense contraction (64->64, 64->128,
// 128->128, 64/128->256 and the Linear), the bandwidth-shaped small-channel kernels for (C+1)->64 / C->64 and, for the
// ->C output layers, a wgmma forward and weight gradient with the output channels zero-padded to a 64-row tile
// (ConvL::pad_out) and an FFMA data gradient.
#include <algorithm>
#include <deque>
#include <string>

#include "convl.h"
#include "fg_internal.h"
#include "k_conv_tc.h"
#include "k_misc.h"
#include "k_rng.cuh"
#include "k_scale.cuh"

namespace {
constexpr int kMaxGL = 5, kMaxDL = 4;
// a generator: its "same" convolutions after the C+1 joined input planes; Cout 0 is the C image channels of the last
// layer (no activation after it), every other layer is followed by a one-slope PReLU
struct C2fGDesc {
  const char* name;
  const char* tag;  // of the timer names of a pair other than the default one
  int n;
  struct { int Cout, k; } L[kMaxGL];
};
// a discriminator: 3x3 convolutions, each followed by a one-slope PReLU and optionally a 2x2 max pool; the last pooled
// map ([view_c][S/view_div][S/view_div]) goes through Dropout and View into Linear(512)
struct C2fDDesc {
  const char* name;
  const char* tag;
  int n;
  struct { int Cout; bool pool; } L[kMaxDL];
  int view_c, view_div;
};
// indexed by FG_C2F_G_* / FG_C2F_D_* (DEFAULT is the models_c2f.lua create_G / create_D default)
const C2fGDesc kGens[] = {
    {"create_G_d", "Gd", 5, {{64, 3}, {64, 3}, {128, 5}, {256, 5}, {0, 7}}},
    {"create_G_d", "Gd", 5, {{64, 3}, {64, 3}, {128, 5}, {256, 5}, {0, 7}}},
    {"create_G_a", "Ga", 3, {{64, 3}, {128, 7}, {0, 5}}},
    {"create_G_b", "Gb", 4, {{64, 3}, {64, 3}, {256, 5}, {0, 7}}},
    {"create_G_c", "Gc", 4, {{64, 3}, {128, 3}, {256, 5}, {0, 7}}},
};
const C2fDDesc kDiscs[] = {
    {"create_D_c", "Dc", 4, {{64, false}, {64, true}, {128, false}, {256, true}}, 256, 4},
    {"create_D_c", "Dc", 4, {{64, false}, {64, true}, {128, false}, {256, true}}, 256, 4},
    {"create_D_a", "Da", 2, {{64, false}, {64, true}}, 64, 2},
    {"create_D_b", "Db", 4, {{64, false}, {64, true}, {128, false}, {128, true}}, 128, 4},
};
constexpr int kNGens = sizeof(kGens) / sizeof(kGens[0]), kNDiscs = sizeof(kDiscs) / sizeof(kDiscs[0]);
bool c2f_size_ok(int S) { return S == 16 || S == 32 || S == 64; }
bool c2f_gen_ok(int g) { return g >= 0 && g < kNGens; }
bool c2f_disc_ok(int d) { return d >= 0 && d < kNDiscs; }
// View(view_c*(S/view_div)^2) of D's last pooled map: D.L1's input width
int c2f_flat(const C2fDDesc& d, int S) { return d.view_c * (S / d.view_div) * (S / d.view_div); }
// nn.Dropout keep flags per sample: the pooled map (NCHW order) then [512]
int c2f_mask(const C2fDDesc& d, int S) { return c2f_flat(d, S) + 512; }
}  // namespace

struct fg_c2f {
  fg_ctx* c = nullptr;
  int maxB = 0, C = 3;
  int S = 32;           // fine size: every image, noise and activation of G and D's first stage is S x S
  int HW = 1024;        // S * S
  int gen = FG_C2F_G_D, disc = FG_C2F_D_C;      // never DEFAULT
  const C2fGDesc* gd = &kGens[FG_C2F_G_D];
  const C2fDDesc* dd = &kDiscs[FG_C2F_D_C];
  int flat = 16384;     // c2f_flat(*dd, S)
  int mask = 16896;     // c2f_mask(*dd, S)
  int nGc = 5, nDc = 4;  // layer counts of the descriptors
  std::deque<std::string> names;  // timer names (stable storage: the layers point into it)
  NetPair net;  // no BatchNorm
  int64_t Gca[kMaxGL] = {}, Dca[kMaxDL] = {}, Da5 = 0, DL2W = 0, DL2b = 0;
  ConvL Gc[kMaxGL], Dc[kMaxDL], DL1;
  const char* D_L2_timer = "";
  const char *t_refine_prep = "", *t_refine_pick = "";  // fg_c2f_refine's own kernels
  float *G_x = nullptr, *G_z[kMaxGL] = {}, *G_h[kMaxGL] = {};
  // D_p[i]: the 2x2 max pool of D_h[i] (layers with a pool only); D_pv = the last of them, the map View flattens
  float *D_x = nullptr, *D_cond = nullptr, *D_z[kMaxDL] = {}, *D_h[kMaxDL] = {}, *D_p[kMaxDL] = {}, *D_pv = nullptr,
        *D_d4 = nullptr;
  float *D_zl1 = nullptr, *D_al1 = nullptr, *D_hl1 = nullptr, *D_logit = nullptr, *D_out = nullptr, *D_masks = nullptr,
        *D_dlogit = nullptr, *D_dx = nullptr;
  float *ga = nullptr, *gb = nullptr, *ws = nullptr;
  float *in_a = nullptr, *in_b = nullptr, *in_c = nullptr, *in_d = nullptr, *in_e = nullptr, *io = nullptr;
  IterStage iter_stage;  // the inputs of the host-fed and device-fed train steps, stacked per iteration
  int G_B = 0, D_B = 0;
  bool G_valid = false, D_valid = false, D_train = true;
  float D_scale = 2.f;
  std::vector<void*> allocs;
  ConvLEnv env;  // shared scratch of the ConvL layers (filled by c2f_alloc)
  float* G_y() const { return G_z[nGc - 1]; }  // G's output (the diff), NHWC
};

namespace {
int dalloc(fg_c2f* n, float** p, size_t elems) { return convl_dalloc(n->env, p, elems); }
inline int convl_alloc(fg_c2f* n, ConvL& L) { return ::convl_alloc(n->env, L); }
inline int convl_fwd(fg_c2f* n, ConvL& L, const float* in, const float* P, float* out, int B) { return ::convl_fwd(n->env, L, in, P, out, B); }
inline int convl_bwd(fg_c2f* n, ConvL& L, const float* in, const float* dy, float* G, float* din, int B) {
  return ::convl_bwd(n->env, L, in, dy, G, din, B);
}

// "c2f.<layer>" at S = 32 (the names profiles/bench_configs.py reads), "c2f16.<layer>" / "c2f64.<layer>" otherwise, so
// that nets of two sizes on one ctx keep their timings apart; a pair other than create_G_d / create_D_c adds its nets'
// tags ("c2f32.Ga.Dc.<layer>"), so that two pairs of one size keep theirs apart too
const char* timer_name(fg_c2f* n, const char* layer) {
  std::string p = n->S == 32 ? std::string("c2f.") : "c2f" + std::to_string(n->S) + ".";
  if (n->gen != FG_C2F_G_D || n->disc != FG_C2F_D_C)
    p = "c2f" + std::to_string(n->S) + "." + n->gd->tag + "." + n->dd->tag + ".";
  n->names.push_back(p + layer);
  return n->names.back().c_str();
}

// the pad rules of the ConvL dispatch (DESIGN.md §7.2): a ->C output layer runs its forward and weight gradient with the
// output channels padded to a 64-row tile, a 64 -> 64 layer its weight gradient with dY padded to 128 rows
void set_pads(ConvL& L) {
  if (L.Cout <= 4 && L.Cin % 128 == 0) L.pad_out = 64;
  if (L.Cout == 64 && L.Cin % 64 == 0) L.pad_dy = 128;
}

void make_layouts(fg_c2f* n) {
  const int C = n->C, S = n->S;
  const C2fGDesc& gd = *n->gd;
  const C2fDDesc& dd = *n->dd;
  n->HW = S * S;
  n->flat = c2f_flat(dd, S);
  n->mask = c2f_mask(dd, S);
  n->nGc = gd.n;
  n->nDc = dd.n;
  n->names.clear();
  {
    int64_t o = 0;
    int ci = C + 1;
    for (int i = 0; i < gd.n; ++i) {
      const bool last = i == gd.n - 1;
      const int co = last ? C : gd.L[i].Cout, k = gd.L[i].k;
      ConvL& L = n->Gc[i];
      L = ConvL{};
      L.Cin = ci; L.Cout = co; L.k = k; L.H = S;
      L.w_off = o; o += (int64_t)co * ci * k * k;
      L.b_off = o; o += co;
      if (!last) { n->Gca[i] = o; o += 1; }
      L.need_dgrad = i > 0;
      const std::string l = "G.c" + std::to_string(i + 1);
      L.tf = timer_name(n, (l + ".fwd").c_str()); L.td = timer_name(n, (l + ".dgrad").c_str()); L.tw = timer_name(n, (l + ".wgrad").c_str());
      set_pads(L);
      ci = co;
    }
    n->net.nG = o;
  }
  {
    int64_t o = 0;
    int ci = C, H = S;
    for (int i = 0; i < dd.n; ++i) {
      const int co = dd.L[i].Cout;
      ConvL& L = n->Dc[i];
      L = ConvL{};
      L.Cin = ci; L.Cout = co; L.k = 3; L.H = H;
      L.w_off = o; o += (int64_t)co * ci * 9;
      L.b_off = o; o += co;
      n->Dca[i] = o; o += 1;
      const std::string l = "D.c" + std::to_string(i + 1);
      L.tf = timer_name(n, (l + ".fwd").c_str()); L.td = timer_name(n, (l + ".dgrad").c_str()); L.tw = timer_name(n, (l + ".wgrad").c_str());
      set_pads(L);
      ci = co;
      if (dd.L[i].pool) H /= 2;
    }
    ConvL& L = n->DL1;
    L = ConvL{};
    L.Cin = n->flat; L.Cout = 512; L.k = 1; L.H = 1;
    // View(view_c*(S/view_div)^2) flattens [view_c][S/view_div][S/view_div]; ours is [S/view_div][S/view_div][view_c]
    L.cA = dd.view_c; L.cS = (S / dd.view_div) * (S / dd.view_div);
    L.w_off = o; o += (int64_t)512 * n->flat;
    L.b_off = o; o += 512;
    L.tf = timer_name(n, "D.L1.fwd"); L.td = timer_name(n, "D.L1.dgrad"); L.tw = timer_name(n, "D.L1.wgrad");
    n->D_L2_timer = timer_name(n, "D.L2.fwd");
    n->t_refine_prep = timer_name(n, "refine_prep");
    n->t_refine_pick = timer_name(n, "refine_pick");
    n->Da5 = o; o += 1;
    n->DL2W = o; o += 512;
    n->DL2b = o; o += 1;
    n->net.nD = o;
  }
}

int c2f_alloc(fg_c2f* n) {
  make_layouts(n);
  const size_t B = n->maxB, C = n->C, HW = n->HW, flat = n->flat, mask = n->mask;
  n->env.c = n->c;
  n->env.maxB = n->maxB;
  n->env.allocs = &n->allocs;
  FG_TRY(pair_alloc(n->c, n->allocs, n->net, n->net.nG, n->net.nD, false));
  // per-sample scratch sizes, the maximum over the layers of both nets:
  //   act  the largest activation / gradient map (the gradient ping-pong, the dY split, a pad_out forward's padded
  //        output); G's first layer (64 channels at S x S) keeps it above fg_c2f_refine's C x 64 x 64 image staging
  //   pad  the largest channel-padded dY (pad_out / pad_dy layers)
  //   wsz  the largest packed weight gradient (whole, not per sample)
  size_t act = 0, pad = 0, wsz = (size_t)512 * flat;
  auto visit = [&](const ConvL& L) {
    const size_t hw = (size_t)L.H * L.H, KK = (size_t)L.k * L.k;
    act = std::max(act, hw * std::max({L.Cin, L.Cout, L.pad_out}));
    pad = std::max(pad, hw * std::max(L.pad_out, L.pad_dy));
    wsz = std::max(wsz, KK * L.Cin * (L.pad_out ? L.pad_out : L.pad_dy ? L.pad_dy : L.Cout));
  };
  for (int i = 0; i < n->nGc; ++i) visit(n->Gc[i]);
  for (int i = 0; i < n->nDc; ++i) visit(n->Dc[i]);
  act = std::max(act, (size_t)flat);
  for (int i = 0; i < n->nGc; ++i) FG_TRY(convl_alloc(n, n->Gc[i]));
  for (int i = 0; i < n->nDc; ++i) FG_TRY(convl_alloc(n, n->Dc[i]));
  FG_TRY(convl_alloc(n, n->DL1));
  FG_TRY(dalloc(n, &n->G_x, B * HW * (C + 1)));
  for (int i = 0; i < n->nGc; ++i) {
    FG_TRY(dalloc(n, &n->G_z[i], B * HW * n->Gc[i].Cout));
    if (i < n->nGc - 1) FG_TRY(dalloc(n, &n->G_h[i], B * HW * n->Gc[i].Cout));
  }
  FG_TRY(dalloc(n, &n->D_x, B * HW * C));
  FG_TRY(dalloc(n, &n->D_cond, B * HW * C));
  for (int i = 0; i < n->nDc; ++i) {
    const ConvL& L = n->Dc[i];
    const size_t e = B * (size_t)L.H * L.H * L.Cout;
    FG_TRY(dalloc(n, &n->D_z[i], e));
    FG_TRY(dalloc(n, &n->D_h[i], e));
    if (n->dd->L[i].pool) {
      FG_TRY(dalloc(n, &n->D_p[i], e / 4));
      n->D_pv = n->D_p[i];
    }
  }
  FG_TRY(dalloc(n, &n->D_d4, B * flat));
  FG_TRY(dalloc(n, &n->D_zl1, B * 512));
  FG_TRY(dalloc(n, &n->D_al1, B * 512));
  FG_TRY(dalloc(n, &n->D_hl1, B * 512));
  FG_TRY(dalloc(n, &n->D_logit, B));
  FG_TRY(dalloc(n, &n->D_out, B));
  FG_TRY(dalloc(n, &n->D_dlogit, B));
  FG_TRY(dalloc(n, &n->D_masks, B * mask));
  FG_TRY(dalloc(n, &n->D_dx, B * HW * C));
  const size_t big = B * act;
  FG_TRY(dalloc(n, &n->ga, big));
  FG_TRY(dalloc(n, &n->gb, big));
  FG_TRY(dalloc(n, &n->env.dy.hi, big));
  FG_TRY(dalloc(n, &n->env.dy.lo, big));
  FG_TRY(dalloc(n, &n->env.pad.hi, B * pad));
  FG_TRY(dalloc(n, &n->env.pad.lo, B * pad));
  FG_TRY(dalloc(n, &n->ws, wsz));
  n->env.ga = n->ga; n->env.ws = n->ws;
  FG_TRY(dalloc(n, &n->in_a, B * HW * C));
  FG_TRY(dalloc(n, &n->in_b, B * HW * C));
  FG_TRY(dalloc(n, &n->in_c, B * HW));
  FG_TRY(dalloc(n, &n->in_d, B * HW * C));
  FG_TRY(dalloc(n, &n->in_e, B * HW));
  FG_TRY(dalloc(n, &n->io, B * HW * C));
  n->net.keep.clear();
  for (int i = 0; i < n->nDc; ++i) {
    n->names.push_back("Dstep.z" + std::to_string(i + 1));
    n->net.keep.push_back({n->names.back().c_str(), n->D_z[i], (int64_t)n->Dc[i].H * n->Dc[i].H * n->Dc[i].Cout});
  }
  n->net.keep.push_back({"Dstep.zl1", n->D_zl1, 512});
  n->net.keep.push_back({"Dstep.logit", n->D_logit, 1});
  n->net.keep.push_back({"Dstep.out", n->D_out, 1});
  FG_CUDA(cudaStreamSynchronize(n->c->stream));
  return FG_OK;
}

// packs are rebuilt after every optimizer step / set_params, and when the ctx's "conv_impl" changed since the last
// pack (the TF32 splits are only produced for the tensor-core implementations)
int pack_G(fg_c2f* n) {
  if (n->net.G_pack == pack_key(n->c)) return FG_OK;
  for (int i = 0; i < n->nGc; ++i) FG_TRY(convl_pack(n->c, n->Gc[i], n->net.PG));
  n->net.G_pack = pack_key(n->c);
  return FG_OK;
}
int pack_D(fg_c2f* n) {
  if (n->net.D_pack == pack_key(n->c)) return FG_OK;
  for (int i = 0; i < n->nDc; ++i) FG_TRY(convl_pack(n->c, n->Dc[i], n->net.PD));
  FG_TRY(convl_pack(n->c, n->DL1, n->net.PD));
  n->net.D_pack = pack_key(n->c);
  return FG_OK;
}

// G on the joined NHWC input already in G_x (nn.JoinTable order: the noise channel, then the C condition channels);
// the diff lands in G_y() (NHWC)
int G_forward_joined(fg_c2f* n, int B) {
  fg_ctx* c = n->c;
  FG_TRY(pack_G(n));
  const float* cur = n->G_x;
  for (int i = 0; i < n->nGc; ++i) {
    FG_TRY(convl_fwd(n, n->Gc[i], cur, n->net.PG, n->G_z[i], B));
    if (i < n->nGc - 1) {
      FG_TRY(k_prelu_fwd(c, n->G_z[i], n->net.PG + n->Gca[i], n->G_h[i], (int64_t)B * n->HW * n->Gc[i].Cout));
      cur = n->G_h[i];
    }
  }
  n->G_B = B;
  n->G_valid = true;
  return FG_OK;
}
// noise [B][1][S][S] and cond [B][C][S][S] are NCHW device pointers; the diff lands in G_y() (NHWC)
int G_forward(fg_c2f* n, const float* noise, const float* cond, int B) {
  FG_REQUIRE(B >= 1 && B <= n->maxB, "c2f G forward: batch %d out of range [1,%d]", B, n->maxB);
  FG_TRY(pack_G(n));
  FG_TRY(k_join_to_nhwc(n->c, noise, cond, n->G_x, B, n->C, n->HW));
  return G_forward_joined(n, B);
}
// ddiff: NHWC [B][S][S][C]; accumulates into gG
int G_backward(fg_c2f* n, const float* ddiff) {
  fg_ctx* c = n->c;
  if (!n->G_valid) {
    fg_set_error("c2f G backward needs a preceding G forward");
    return FG_ERR_STATE;
  }
  const int B = n->G_B;
  const float* dcur = ddiff;
  for (int i = n->nGc - 1; i >= 0; --i) {
    const float* in = i == 0 ? n->G_x : n->G_h[i - 1];
    FG_TRY(convl_bwd(n, n->Gc[i], in, dcur, n->net.gG, i > 0 ? n->ga : nullptr, B));
    if (i > 0) {
      FG_TRY(k_prelu_bwd(c, n->ga, n->G_z[i - 1], n->net.PG + n->Gca[i - 1], n->gb, n->net.gG + n->Gca[i - 1], B, n->S, n->S,
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
  const float* P = n->net.PD;
  FG_TRY(k_add(c, diff, cond, n->D_x, (int64_t)B * n->HW * n->C));  // nn.CAddTable
  const float* cur = n->D_x;
  for (int i = 0; i < n->nDc; ++i) {
    const ConvL& L = n->Dc[i];
    FG_TRY(convl_fwd(n, n->Dc[i], cur, P, n->D_z[i], B));
    FG_TRY(k_prelu_fwd(c, n->D_z[i], P + n->Dca[i], n->D_h[i], (int64_t)B * L.H * L.H * L.Cout));
    cur = n->D_h[i];
    if (n->D_p[i]) {
      FG_TRY(k_maxpool2_fwd(c, n->D_h[i], n->D_p[i], B, L.H, L.H, L.Cout));
      cur = n->D_p[i];
    }
  }
  n->D_scale = 1.0f / (1.0f - p_drop);
  const float* d4 = n->D_pv;
  if (training) {  // nn.Dropout (v2): mask/(1-p) in training, identity in evaluation
    FG_TRY(k_dropout_nhwc(c, n->D_pv, n->D_masks, n->mask, 0, n->DL1.cS, n->DL1.cA, n->D_scale, n->D_d4, B));
    d4 = n->D_d4;
  }
  FG_TRY(convl_fwd(n, n->DL1, d4, P, n->D_zl1, B));
  FG_TRY(k_prelu_fwd(c, n->D_zl1, P + n->Da5, n->D_al1, (int64_t)B * 512));
  const float* hl1 = n->D_al1;
  if (training) {
    FG_TRY(k_dropout_nhwc(c, n->D_al1, n->D_masks, n->mask, n->flat, 1, 512, n->D_scale, n->D_hl1, B));
    hl1 = n->D_hl1;
  }
  {
    ScopedTimer tm(c, n->D_L2_timer);
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
  const float* P = n->net.PD;
  float* G = want_wgrad ? n->net.gD : nullptr;
  const bool tr = n->D_train;
  const float* hl1 = tr ? n->D_hl1 : n->D_al1;
  const float* d4 = tr ? n->D_d4 : n->D_pv;
  if (G) FG_TRY(k_gemv_wgrad_add(c, hl1, dlogit, G + n->DL2W, G + n->DL2b, B, 512));
  float *cur = n->ga, *oth = n->gb;  // gradient ping-pong: every stage reads `cur`, writes `oth`, then they swap
  FG_TRY(k_gemv_dgrad(c, dlogit, P + n->DL2W, cur, B, 512));
  if (tr) {
    FG_TRY(k_dropout_nhwc(c, cur, n->D_masks, n->mask, n->flat, 1, 512, n->D_scale, oth, B));
    std::swap(cur, oth);
  }
  FG_TRY(k_prelu_bwd(c, cur, n->D_zl1, P + n->Da5, oth, G ? G + n->Da5 : nullptr, B, 1, 1, 512, 0));
  std::swap(cur, oth);
  FG_TRY(convl_bwd(n, n->DL1, d4, cur, G, oth, B));  // -> gradient of the View input, NHWC
  std::swap(cur, oth);
  if (tr) {
    FG_TRY(k_dropout_nhwc(c, cur, n->D_masks, n->mask, 0, n->DL1.cS, n->DL1.cA, n->D_scale, oth, B));
    std::swap(cur, oth);
  }
  for (int i = n->nDc - 1; i >= 0; --i) {
    ConvL& L = n->Dc[i];
    if (n->D_p[i]) {  // cur is the gradient of the pooled map
      FG_TRY(k_maxpool2_bwd(c, cur, n->D_h[i], oth, B, L.H, L.H, L.Cout));
      std::swap(cur, oth);
    }
    FG_TRY(k_prelu_bwd(c, cur, n->D_z[i], P + n->Dca[i], oth, G ? G + n->Dca[i] : nullptr, B, L.H, L.H, L.Cout, 0));
    std::swap(cur, oth);
    const float* in = i == 0 ? n->D_x : (n->D_p[i - 1] ? n->D_p[i - 1] : n->D_h[i - 1]);
    float* din = i > 0 ? oth : (want_dx ? n->D_dx : nullptr);
    FG_TRY(convl_bwd(n, L, in, cur, G, din, B));
    if (i > 0) std::swap(cur, oth);
  }
  return FG_OK;
}

// the c2f nets in the loop body of adversarial_c2f.lua:121-187 (pair_train_step, netpair.cu): D iteration j reads
// real_diff [B/2][C][S][S], condD [B][C][S][S] (the real pairs' condition, then the fakes') and noiseD [B/2][1][S][S],
// G iteration j condG [B][C][S][S] and noiseG [B][1][S][S].  optim.adam / adagrad / sgd (:153-161, :177-185) follow
// the same rules as the interruptable optimizers, without the accuracy gate.
struct C2fStep final : StepNets {
  fg_c2f* n;
  const float *real_diff, *condD, *noiseD, *condG, *noiseG;
  C2fStep(fg_c2f* n, const fg_hyper* h, int B, const float* real_diff, const float* condD, const float* noiseD,
          const float* condG, const float* noiseG)
      : StepNets(n->c, n->net, h, B, n->D_logit, n->D_out, n->D_dlogit, n->D_masks, n->mask, false, false), n(n),
        real_diff(real_diff), condD(condD), noiseD(noiseD), condG(condG), noiseG(noiseG) {}
  size_t img() const { return (size_t)n->C * n->HW; }
  int g_forward(int j, bool d_iter) override {
    if (d_iter) {  // the fakes take the second half of D's condition rows
      const float* cd = condD + (size_t)j * B * img();
      return G_forward(n, noiseD + (size_t)j * (B / 2) * n->HW, cd + (B / 2) * img(), B / 2);
    }
    const float* cg = condG + (size_t)j * B * img();
    FG_TRY(G_forward(n, noiseG + (size_t)j * B * n->HW, cg, B));
    return k_nchw_to_nhwc(c, cg, n->D_cond, B, n->C, n->HW);
  }
  int d_input(int j) override {
    const int Bh = B / 2;
    FG_TRY(k_nchw_to_nhwc(c, real_diff + (size_t)j * Bh * img(), n->io, Bh, n->C, n->HW));
    FG_CUDA(cudaMemcpyAsync(n->io + Bh * img(), n->G_y(), sizeof(float) * Bh * img(), cudaMemcpyDeviceToDevice, c->stream));
    return k_nchw_to_nhwc(c, condD + (size_t)j * B * img(), n->D_cond, B, n->C, n->HW);
  }
  int draw_masks(int kind, const uint64_t* root) override {
    return k_bernoulli_keep(c, n->D_masks, (int64_t)B * n->mask, kind, h->p_drop, root);
  }
  int d_forward(bool on_g) override { return D_forward(n, on_g ? n->G_y() : n->io, n->D_cond, B, true, h->p_drop); }
  // D's weight grads of the G iteration are zeroed before use (:45): skipped
  int d_backward(bool want_wgrad, bool want_dx) override { return D_backward(n, n->D_dlogit, want_wgrad, want_dx); }
  int g_backward() override { return G_backward(n, n->D_dx); }
};

// ---- fg_c2f_refine: sample.lua:176-214 c2f() around the G and D forwards ----------------------------------------
constexpr int kRefineThreads = 256;
// The input side of one chunk, one CTA per base image i (global image i0 + i):
//   up        = image.scale(image i, S, S), from the image staged in shared memory (C*in*in floats, <= 48 KB)
//   G_x       [r][p] = {noise, up[0..C)} for the chunk rows r = i*tries + t (NHWC, nn.JoinTable(2,2) order), noise =
//             noise[r*S*S + p] (the caller's, offset to the chunk) or element ((i0+i)*tries + t)*S*S + p of the uniform
//             stream noise_seed (fg_noise_uniform's formula, so the draw does not depend on the chunking)
//   D_cond    [r][p][ch] = up[ch][p]  (D's condition, NHWC)
//   up_out    [i][ch][p] = up[ch][p]  (NCHW, for the final add)
__global__ void __launch_bounds__(kRefineThreads) refine_prep_kernel(const float* __restrict__ images, int C, int in, int S,
                                                                     int tries, int64_t i0, const float* __restrict__ noise,
                                                                     uint64_t noise_seed, float* __restrict__ G_x,
                                                                     float* __restrict__ D_cond, float* __restrict__ up_out) {
  extern __shared__ float img_s[];
  const int i = blockIdx.x, HW = S * S, plane = in * in, n_in = C * plane;
  const float* src = images + (int64_t)i * n_in;
  for (int k = threadIdx.x; k < n_in; k += blockDim.x) img_s[k] = src[k];
  __syncthreads();
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const int y = p / S, x = p - y * S;
    float up[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      if (ch < C) {
        up[ch] = scale_pixel(PlaneSrc{img_s + ch * plane, in}, y, x, in, in, S, S);
        up_out[((int64_t)i * C + ch) * HW + p] = up[ch];
      }
    }
    for (int t = 0; t < tries; ++t) {
      const int64_t r = (int64_t)i * tries + t, e = r * HW + p;
      const float z = noise ? noise[e] : uniform_pm1_at(noise_seed, (uint64_t)(((i0 + i) * tries + t) * HW + p));
      float* gx = G_x + e * (C + 1);
      float* dc = D_cond + e * C;
      gx[0] = z;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        if (ch < C) {
          gx[1 + ch] = up[ch];
          dc[ch] = up[ch];
        }
      }
    }
  }
}
// The output side, one CTA per base image i: pick = the first try with the largest prediction (the strict > of
// sample.lua:201-207, so a NaN wins only at t = 0), out[i] = up[i] + diff[i*tries + pick] (NCHW; diff is G's NHWC
// output, transposed in the same pass).
__global__ void __launch_bounds__(kRefineThreads) refine_pick_kernel(const float* __restrict__ pred, const float* __restrict__ diff,
                                                                     const float* __restrict__ up, int C, int HW, int tries,
                                                                     float* __restrict__ out, int32_t* __restrict__ pick_out) {
  __shared__ int pick_s;
  const int i = blockIdx.x;
  if (threadIdx.x == 0) {
    const float* pr = pred + (int64_t)i * tries;
    int best = 0;
    float m = pr[0];
    for (int t = 1; t < tries; ++t) {
      if (pr[t] > m) {
        m = pr[t];
        best = t;
      }
    }
    pick_s = best;
    if (pick_out) pick_out[i] = best;
  }
  __syncthreads();
  const int n = C * HW;
  const float* d = diff + ((int64_t)i * tries + pick_s) * n;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int ch = k / HW, p = k - ch * HW;
    out[(int64_t)i * n + k] = up[(int64_t)i * n + k] + d[(int64_t)p * C + ch];
  }
}
}  // namespace

namespace {
// getParameters() length of G (net FG_NET_G) or D of the pair (gen, disc) with C channels at fine size S
int64_t c2f_count(int gen, int disc, int C, int S, int net) {
  fg_c2f tmp;
  tmp.C = C;
  tmp.S = S;
  tmp.gd = &kGens[gen];
  tmp.dd = &kDiscs[disc];
  make_layouts(&tmp);
  return net == FG_NET_D ? tmp.net.nD : tmp.net.nG;
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

namespace {
// d_iters D iterations + g_iters G iterations of the c2f loop body on the fg_c2f_train_step inputs stacked per
// iteration, for the entry `what`
int train_step_iters(fg_c2f* n, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real_diff,
                     const float* cond_D, const float* noise_D, const float* cond_G, const float* noise_G, const float* masks_D,
                     const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  fg_ctx* c = n->c;
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h && real_diff && cond_D && noise_D && cond_G && noise_G));
  const size_t nd = d_iters, ng = g_iters, Bh = B / 2, M = n->maxB, img = (size_t)n->C * n->HW, hw = n->HW, mk = n->mask;
  IterStage& s = n->iter_stage;
  const float *rd, *cd, *zd, *cg, *zg, *md, *mg;
  FG_TRY(s.in(c, n->allocs, 0, real_diff, nd * Bh * img, nd * M / 2 * img, &rd));
  FG_TRY(s.in(c, n->allocs, 1, cond_D, nd * B * img, nd * M * img, &cd));
  FG_TRY(s.in(c, n->allocs, 2, noise_D, nd * Bh * hw, nd * M / 2 * hw, &zd));
  FG_TRY(s.in(c, n->allocs, 3, cond_G, ng * B * img, ng * M * img, &cg));
  FG_TRY(s.in(c, n->allocs, 4, noise_G, ng * B * hw, ng * M * hw, &zg));
  FG_TRY(s.in(c, n->allocs, 5, masks_D, nd * B * mk, nd * M * mk, &md));
  FG_TRY(s.in(c, n->allocs, 6, masks_G, ng * B * mk, ng * M * mk, &mg));
  C2fStep st(n, h, B, rd, cd, zd, cg, zg);
  return pair_train_step(st, d_iters, g_iters, md, mg, seed, {rd, cd, zd, cg, zg, md, mg, nullptr, nullptr}, nullptr, stats);
}

// the same fed on the device: D iteration j draws the streams 8*r_j .. 8*r_j+1 and 8*r_j+3, G iteration j the streams
// 8*r_j+2 and 8*r_j+4 (r_j: fg_b200.h; r_0 = seed); the draws run inside the step
int train_step_dataset_iters(fg_c2f* n, fg_dataset* d, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters,
                             int coarse_size, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  fg_ctx* c = n->c;
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h, d, true));
  FG_REQUIRE(coarse_size >= 1 && coarse_size <= n->S, "%s: coarse size %d outside [1, %d]", what, coarse_size, n->S);
  const int Bh = B / 2, S = n->S;
  const size_t M = n->maxB, img = (size_t)n->C * n->HW, hw = n->HW;
  IterStage& s = n->iter_stage;
  FG_TRY(s.reserve(c, n->allocs, 0, d_iters * M / 2 * img));
  FG_TRY(s.reserve(c, n->allocs, 1, d_iters * M * img));
  FG_TRY(s.reserve(c, n->allocs, 2, d_iters * M / 2 * hw));
  FG_TRY(s.reserve(c, n->allocs, 3, g_iters * M * img));
  FG_TRY(s.reserve(c, n->allocs, 4, g_iters * M * hw));
  float *rd = s.p[0], *cd = s.p[1], *zd = s.p[2], *cg = s.p[3], *zg = s.p[4];
  const std::function<int()> feed = [&]() -> int {
    for (int j = 0; j < d_iters; ++j) {
      const uint64_t* r = c->seed_dev + j;
      float* cdj = cd + (size_t)j * B * img;
      FG_TRY(dataset_draw_gather_c2f(d, 0, Bh, S, coarse_size, nullptr, cdj, rd + (size_t)j * Bh * img, r, 8));
      FG_TRY(dataset_draw_gather_c2f(d, 1, Bh, S, coarse_size, nullptr, cdj + Bh * img, nullptr, r, 8));
      FG_TRY(noise_uniform_dev(c, 3, (int64_t)Bh * hw, zd + (size_t)j * Bh * hw, r, 8));
    }
    for (int j = 0; j < g_iters; ++j) {
      const uint64_t* r = c->seed_dev + j;
      FG_TRY(dataset_draw_gather_c2f(d, 2, B, S, coarse_size, nullptr, cg + (size_t)j * B * img, nullptr, r, 8));
      FG_TRY(noise_uniform_dev(c, 4, (int64_t)B * hw, zg + (size_t)j * B * hw, r, 8));
    }
    return FG_OK;
  };
  C2fStep st(n, h, B, rd, cd, zd, cg, zg);
  return pair_train_step(st, d_iters, g_iters, nullptr, nullptr, seed,
                         {rd, cd, zd, cg, zg, nullptr, nullptr, d, (const void*)(intptr_t)coarse_size}, &feed, stats);
}
}  // namespace

extern "C" {

int fg_c2f_create(fg_ctx* ctx, fg_c2f** out) { return fg_c2f_create_sized(ctx, 32, out); }
int fg_c2f_create_sized(fg_ctx* ctx, int fine_size, fg_c2f** out) {
  return fg_c2f_create_nets(ctx, fine_size, FG_C2F_G_DEFAULT, FG_C2F_D_DEFAULT, out);
}
int fg_c2f_create_nets(fg_ctx* ctx, int fine_size, int gen, int disc, fg_c2f** out) {
  if (!ctx || !out) {
    fg_set_error("fg_c2f_create_nets: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  if (!c2f_size_ok(fine_size)) {
    fg_set_error("fg_c2f_create_nets: fine size %d is not supported (16, 32 or 64)", fine_size);
    return FG_ERR_UNSUPPORTED;
  }
  if (!c2f_gen_ok(gen) || !c2f_disc_ok(disc)) {
    fg_set_error("fg_c2f_create_nets: unknown generator %d or discriminator %d (FG_C2F_G_* 0..%d, FG_C2F_D_* 0..%d)", gen,
                 disc, kNGens - 1, kNDiscs - 1);
    return FG_ERR_UNSUPPORTED;
  }
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_c2f* n = new fg_c2f();
  n->c = ctx;
  n->S = fine_size;
  n->gen = gen == FG_C2F_G_DEFAULT ? FG_C2F_G_D : gen;
  n->disc = disc == FG_C2F_D_DEFAULT ? FG_C2F_D_C : disc;
  n->gd = &kGens[n->gen];
  n->dd = &kDiscs[n->disc];
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
int fg_c2f_get_gen(fg_c2f* n) { return n ? n->gen : -1; }
int fg_c2f_get_disc(fg_c2f* n) { return n ? n->disc : -1; }
int fg_c2f_destroy(fg_c2f* n) {
  if (!n) return FG_OK;
  if (n->c) {
    cudaSetDevice(n->c->device);
    cudaStreamSynchronize(n->c->stream);
  }
  pair_free(n->net);
  for (void* p : n->allocs) cudaFree(p);
  delete n;
  return FG_OK;
}
int64_t fg_c2f_param_count(int net, int channels) { return fg_c2f_param_count_sized(net, channels, 32); }
int64_t fg_c2f_param_count_sized(int net, int channels, int fine_size) {
  if (!c2f_size_ok(fine_size)) return -1;
  return c2f_count(FG_C2F_G_DEFAULT, FG_C2F_D_DEFAULT, channels, fine_size, net);
}
int64_t fg_c2f_gen_param_count(int gen, int channels) {
  return c2f_gen_ok(gen) && channels >= 1 ? c2f_count(gen, FG_C2F_D_DEFAULT, channels, 32, FG_NET_G) : -1;
}
int64_t fg_c2f_disc_param_count(int disc, int channels, int fine_size) {
  return c2f_disc_ok(disc) && channels >= 1 && c2f_size_ok(fine_size)
             ? c2f_count(FG_C2F_G_DEFAULT, disc, channels, fine_size, FG_NET_D) : -1;
}
int fg_c2f_mask_per_sample(void) { return c2f_mask(kDiscs[FG_C2F_D_DEFAULT], 32); }
int fg_c2f_mask_per_sample_sized(int fine_size) { return fg_c2f_disc_mask_per_sample(FG_C2F_D_DEFAULT, fine_size); }
int fg_c2f_disc_mask_per_sample(int disc, int fine_size) {
  return c2f_disc_ok(disc) && c2f_size_ok(fine_size) ? c2f_mask(kDiscs[disc], fine_size) : -1;
}
int fg_c2f_fine_size(fg_c2f* n) { return n ? n->S : 0; }

int fg_c2f_set_params(fg_c2f* n, int net, const float* src) {
  ENTER(n);
  FG_REQUIRE(src && (net == FG_NET_G || net == FG_NET_D), "fg_c2f_set_params: bad arguments");
  return pair_set_params(n->c, n->net, net, src);
}
int fg_c2f_get_params(fg_c2f* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_c2f_get_params: bad arguments");
  return pair_get_params(n->c, n->net, net, dst);
}
int fg_c2f_get_grads(fg_c2f* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_c2f_get_grads: bad arguments");
  return pair_get_grads(n->c, n->net, net, dst);
}
int fg_c2f_zero_grads(fg_c2f* n, int net) {
  ENTER(n);
  return pair_zero_grads(n->c, n->net, net);
}
float* fg_c2f_params_ptr(fg_c2f* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->net.PD : n->net.PG); }
float* fg_c2f_grads_ptr(fg_c2f* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->net.gD : n->net.gG); }

int fg_c2f_set_adam_state(fg_c2f* n, int net, const float* m, const float* v, int t) {
  ENTER(n);
  return pair_set_adam_state(n->c, n->net, net, m, v, t);
}
int fg_c2f_get_adam_state(fg_c2f* n, int net, float* m, float* v, int* t) {
  ENTER(n);
  return pair_get_adam_state(n->c, n->net, net, m, v, t);
}

int fg_c2f_G_forward(fg_c2f* n, const float* noise, const float* cond, int B, float* diff_out) {
  ENTER(n);
  FG_REQUIRE(noise && cond && B >= 1 && B <= n->maxB, "fg_c2f_G_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  const float *nd, *cd;
  FG_TRY(fg_to_dev(n->c, noise, (size_t)B * n->HW, n->in_c, &nd));
  FG_TRY(fg_to_dev(n->c, cond, (size_t)B * n->C * n->HW, n->in_b, &cd));
  FG_TRY(G_forward(n, nd, cd, B));
  if (diff_out) {
    FG_TRY(k_nhwc_to_nchw(n->c, n->G_y(), n->io, B, n->C, n->HW));
    FG_TRY(fg_to_user(n->c, diff_out, n->io, (size_t)B * n->C * n->HW));
  }
  return FG_OK;
}
int fg_c2f_G_backward(fg_c2f* n, const float* d_diff) {
  ENTER(n);
  FG_REQUIRE(d_diff, "fg_c2f_G_backward: null gradient");
  const float* dd;
  FG_TRY(fg_to_dev(n->c, d_diff, (size_t)n->G_B * n->C * n->HW, n->in_a, &dd));
  FG_TRY(k_nchw_to_nhwc(n->c, dd, n->io, n->G_B, n->C, n->HW));
  return G_backward(n, n->io);
}
int fg_c2f_D_forward(fg_c2f* n, const float* diff, const float* cond, int B, int training, const float* masks,
                     uint64_t seed, float* out) {
  ENTER(n);
  FG_REQUIRE(diff && cond && B >= 1 && B <= n->maxB, "fg_c2f_D_forward: bad arguments (batch %d, max %d)", B, n->maxB);
  fg_ctx* c = n->c;
  const float *dd, *cd;
  FG_TRY(fg_to_dev(c, diff, (size_t)B * n->C * n->HW, n->in_a, &dd));
  FG_TRY(fg_to_dev(c, cond, (size_t)B * n->C * n->HW, n->in_b, &cd));
  FG_TRY(k_nchw_to_nhwc(c, dd, n->io, B, n->C, n->HW));
  FG_TRY(k_nchw_to_nhwc(c, cd, n->D_cond, B, n->C, n->HW));
  if (training) {
    if (masks)
      FG_CUDA(cudaMemcpyAsync(n->D_masks, masks, sizeof(float) * (size_t)B * n->mask, cudaMemcpyDefault, c->stream));
    else
      FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)B * n->mask, seed, 0.5f));
  }
  FG_TRY(D_forward(n, n->io, n->D_cond, B, training != 0, 0.5f));
  FG_TRY(k_sigmoid_fwd(c, n->D_logit, n->D_out, B));
  if (out) FG_TRY(fg_to_user(c, out, n->D_out, B));
  return FG_OK;
}
int fg_c2f_D_backward(fg_c2f* n, const float* d_out, int want_wgrad, float* d_diff) {
  ENTER(n);
  FG_REQUIRE(d_out, "fg_c2f_D_backward: null gradient");
  fg_ctx* c = n->c;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_out, (size_t)n->D_B, n->in_e, &dd));
  FG_TRY(k_sigmoid_bwd(c, dd, n->D_out, n->D_dlogit, n->D_B));
  FG_TRY(D_backward(n, n->D_dlogit, want_wgrad != 0, d_diff != nullptr));
  if (d_diff) {
    FG_TRY(k_nhwc_to_nchw(c, n->D_dx, n->io, n->D_B, n->C, n->HW));
    FG_TRY(fg_to_user(c, d_diff, n->io, (size_t)n->D_B * n->C * n->HW));
  }
  return FG_OK;
}

// adversarial_c2f.lua:305-325 approxParzen, one sample: K generations G({noise_k, coarse}) + coarse for the SAME
// coarse image, the smallest torch.dist to the ground-truth fine image.  noise [K][1][S][S], coarse / fine
// [C][S][S] (host or device); *dist_out (host).
int fg_c2f_parzen_dist(fg_c2f* n, const float* noise, const float* coarse, const float* fine, int K, float* dist_out) {
  ENTER(n);
  FG_REQUIRE(noise && coarse && fine && dist_out && K >= 1 && K <= n->maxB, "fg_c2f_parzen_dist: bad arguments (K %d, max %d)", K,
             n->maxB);
  fg_ctx* c = n->c;
  const size_t img = (size_t)n->C * n->HW;
  const float *nd, *fd;
  FG_TRY(fg_to_dev(c, noise, (size_t)K * n->HW, n->in_c, &nd));
  for (int k = 0; k < K; ++k)  // condInputs[i] = condInput:clone()  (:318-320)
    FG_CUDA(cudaMemcpyAsync(n->in_b + (size_t)k * img, coarse, img * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_TRY(G_forward(n, nd, n->in_b, K));
  FG_TRY(k_nchw_to_nhwc(c, n->in_b, n->D_cond, K, n->C, n->HW));
  FG_TRY(k_add(c, n->G_y(), n->D_cond, n->io, (int64_t)K * img));  // neighbors:add(condInputs)  (:322)
  FG_TRY(fg_to_dev(c, fine, img, n->in_a, &fd));
  FG_TRY(k_nchw_to_nhwc(c, fd, n->in_d, 1, n->C, n->HW));
  int32_t idx = 0;
  return fg_nearest(c, n->in_d, 1, n->io, K, (int)img, &idx, dist_out);
}

// sample.lua:176-214 c2f(images, G, D, fineSize), `chunk` base images (chunk * tries rows of G and D) per pass; see
// fg_b200.h.  Host inputs and outputs are staged through the net's buffers:
//   gb    the chunk's images (C*in*in <= 3*64*64 floats per image; gb holds at least 64*S*S >= 3*64*64 per
//         row at S >= 16, G's first layer having 64 channels)          in_c  the caller's noise rows
//   in_a  up (NCHW)      io  out on its way to the host      in_e  pick on its way to the host (int32 storage)
// Nothing synchronises per chunk: host copies are ordered on the stream behind the kernels that fill their source.
int fg_c2f_refine(fg_c2f* n, const float* images, int64_t N, int in_size, int tries, int chunk, int training, const float* noise,
                  const float* masks, uint64_t seed, float* out, int32_t* pick_out, float* pred_out) {
  ENTER(n);
  FG_REQUIRE(images && out && N >= 1, "fg_c2f_refine: need images, out and N >= 1");
  FG_REQUIRE(tries >= 1 && chunk >= 1 && (int64_t)chunk * tries <= n->maxB,
             "fg_c2f_refine: chunk %d x tries %d rows must be in [1, max_batch %d]", chunk, tries, n->maxB);
  FG_REQUIRE(in_size >= 1 && in_size <= 64, "fg_c2f_refine: input size %d outside [1, 64]", in_size);
  fg_ctx* c = n->c;
  const int C = n->C, HW = n->HW;
  const size_t img_in = (size_t)C * in_size * in_size, img = (size_t)C * HW, mask = n->mask;
  const size_t smem = sizeof(float) * img_in;  // <= 3 x 64 x 64 floats: the default 48 KB
  const bool out_dev = fg_is_dev(out), pick_dev = pick_out && fg_is_dev(pick_out);
  const bool pred_dev = pred_out && fg_is_dev(pred_out);
  for (int64_t s0 = 0; s0 < N; s0 += chunk) {
    const int b = (int)std::min<int64_t>(chunk, N - s0), R = b * tries;
    const int64_t r0 = s0 * tries;
    const float *imd, *nz = nullptr;
    FG_TRY(fg_to_dev(c, images + s0 * img_in, b * img_in, n->gb, &imd));
    if (noise) FG_TRY(fg_to_dev(c, noise + r0 * HW, (size_t)R * HW, n->in_c, &nz));
    {
      ScopedTimer tm(c, n->t_refine_prep);
      refine_prep_kernel<<<b, kRefineThreads, smem, c->stream>>>(imd, C, in_size, n->S, tries, s0, nz, 2 * seed, n->G_x, n->D_cond,
                                                                 n->in_a);
      LAUNCH_CHECK(c);
    }
    FG_TRY(G_forward_joined(n, R));
    if (training) {
      if (masks)
        FG_CUDA(cudaMemcpyAsync(n->D_masks, masks + r0 * mask, sizeof(float) * R * mask, cudaMemcpyDefault, c->stream));
      else
        FG_TRY(k_bernoulli_keep(c, n->D_masks, (int64_t)R * mask, 2 * seed + 1, 0.5f, nullptr, r0 * (int64_t)mask));
    }
    FG_TRY(D_forward(n, n->G_y(), n->D_cond, R, training != 0, 0.5f));
    FG_TRY(k_sigmoid_fwd(c, n->D_logit, n->D_out, R));
    float* od = out_dev ? out + s0 * img : n->io;
    int32_t* pk = pick_dev ? pick_out + s0 : (pick_out ? reinterpret_cast<int32_t*>(n->in_e) : nullptr);
    {
      ScopedTimer tm(c, n->t_refine_pick);
      refine_pick_kernel<<<b, kRefineThreads, 0, c->stream>>>(n->D_out, n->G_y(), n->in_a, C, HW, tries, od, pk);
      LAUNCH_CHECK(c);
    }
    if (!out_dev) FG_CUDA(cudaMemcpyAsync(out + s0 * img, od, sizeof(float) * b * img, cudaMemcpyDeviceToHost, c->stream));
    if (pick_out && !pick_dev)
      FG_CUDA(cudaMemcpyAsync(pick_out + s0, pk, sizeof(int32_t) * b, cudaMemcpyDeviceToHost, c->stream));
    if (pred_out) FG_CUDA(cudaMemcpyAsync(pred_out + r0, n->D_out, sizeof(float) * R, cudaMemcpyDefault, c->stream));
  }
  if (!out_dev || (pick_out && !pick_dev) || (pred_out && !pred_dev)) FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

// data parallel: rank 0's c2f parameters, optimizer moments, step counters and accuracy history (the nets have no
// BatchNorm state) to every rank; the communicator is the ctx's (fg_dp_init)
int fg_c2f_dp_broadcast_params(fg_c2f* n) {
  ENTER(n);
  return pair_broadcast(n->c, n->net);
}

int fg_c2f_train_step(fg_c2f* n, const fg_hyper* h, int B, const float* real_diff, const float* cond_D,
                      const float* noise_D, const float* cond_G, const float* noise_G, const float* masks_D,
                      const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  return train_step_iters(n, "fg_c2f_train_step", h, B, 1, 1, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D, masks_G,
                          seed, stats);
}

// one adversarial_c2f.lua:121-187 loop body fed on the device (the draws of :124-141 and :168-174):
//   real pairs  = gather_c2f(draw(8*seed,   B/2)) -> real_diff, cond_D rows [0, B/2)
//   fake cond   = gather_c2f(draw(8*seed+1, B/2)) -> cond_D rows [B/2, B)
//   G-step cond = gather_c2f(draw(8*seed+2, B))   -> cond_G
//   noise_D = uniform(8*seed+3), noise_G = uniform(8*seed+4), dropout masks from `seed`.
int fg_c2f_train_step_dataset(fg_c2f* n, fg_dataset* d, const fg_hyper* h, int B, int coarse_size, uint64_t seed,
                              fg_step_stats* stats) {
  return train_step_dataset_iters(n, d, "fg_c2f_train_step_dataset", h, B, 1, 1, coarse_size, seed, stats);
}

// d_iters D iterations + g_iters G iterations of the c2f loop body on the fg_c2f_train_step inputs stacked per iteration
int fg_c2f_train_step_iters(fg_c2f* n, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real_diff,
                            const float* cond_D, const float* noise_D, const float* cond_G, const float* noise_G,
                            const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  return train_step_iters(n, "fg_c2f_train_step_iters", h, B, d_iters, g_iters, real_diff, cond_D, noise_D, cond_G, noise_G,
                          masks_D, masks_G, seed, stats);
}

// fg_c2f_train_step_iters fed on the device: D iteration j draws the streams 8*r_j .. 8*r_j+1 and 8*r_j+3, G iteration
// j the streams 8*r_j+2 and 8*r_j+4, as fg_c2f_train_step_dataset does for r_0 = seed (r_j: fg_b200.h)
int fg_c2f_train_step_dataset_iters(fg_c2f* n, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters,
                                    int coarse_size, uint64_t seed, fg_step_stats* stats) {
  return train_step_dataset_iters(n, d, "fg_c2f_train_step_dataset_iters", h, B, d_iters, g_iters, coarse_size, seed, stats);
}

int64_t fg_c2f_debug_tensor(fg_c2f* n, const char* name, float* dst, int64_t max_elems) {
  if (!n || !n->c || !name) {
    fg_set_error("fg_c2f_debug_tensor: null argument");
    return -1;
  }
  cudaSetDevice(n->c->device);
  const int gb = n->G_B, db = n->D_B, C = n->C, HW = n->HW;
  auto g = [&](const float* p) { return n->G_valid ? p : nullptr; };
  auto d = [&](const float* p) { return n->D_valid ? p : nullptr; };
  std::vector<DebugTensor> ents = {{"G.x", g(n->G_x), HW * (C + 1), gb}, {"D.x", d(n->D_x), HW * C, db}};
  std::deque<std::string> rows;  // the names of the per-layer rows (stable storage)
  for (int i = 0; i < n->nGc; ++i) {
    rows.push_back("G.z" + std::to_string(i + 1));
    ents.push_back({rows.back().c_str(), g(n->G_z[i]), HW * n->Gc[i].Cout, gb});
  }
  for (int i = 0; i < n->nDc; ++i) {
    const ConvL& L = n->Dc[i];
    const int64_t e = (int64_t)L.H * L.H * L.Cout;
    rows.push_back("D.z" + std::to_string(i + 1));
    ents.push_back({rows.back().c_str(), d(n->D_z[i]), e, db});
    if (n->D_p[i]) {
      rows.push_back("D.p" + std::to_string(i + 1));
      ents.push_back({rows.back().c_str(), d(n->D_p[i]), e / 4, db});
    }
  }
  ents.push_back({"D.zl1", d(n->D_zl1), 512, db});
  ents.push_back({"D.logit", d(n->D_logit), 1, db});
  ents.push_back({"D.out", d(n->D_out), 1, db});
  pair_keep_rows(n->net, ents);
  return debug_tensor_copy(n->c, "fg_c2f_debug_tensor", ents.data(), ents.size(), name, dst, max_elems);
}

}  // extern "C"
