// UpsGen: the generator of models.lua at side S, create_G_decoder_upsampling32 (models.lua:57-81, S = 32) or
// create_G_decoder_upsampling16 (models.lua:27-51, S = 16: the same layers with every spatial size halved).  The trainer
// of the 32x32 and --scale 16 nets (UpsGan, ups_gan.cu) owns one; what differs between the sizes is data (GenDesc).
#include "convl.h"

GLayout make_g_layout(int C, int side) {
  const int64_t n0 = 128 * (side / 4) * (side / 4);  // G.L1's outputs, View(128, S/4, S/4)
  GLayout L;
  int64_t o = 0;
  L.L1W = o; o += n0 * kNoiseDim;
  L.L1b = o; o += n0;
  L.a1 = o; o += 1;
  L.C1W = o; o += 256 * 128 * 25;
  L.C1b = o; o += 256;
  L.g1 = o; o += 256;
  L.be1 = o; o += 256;
  L.a2 = o; o += 1;
  L.C2W = o; o += 128 * 256 * 25;
  L.C2b = o; o += 128;
  L.g2 = o; o += 128;
  L.be2 = o; o += 128;
  L.a3 = o; o += 1;
  L.C3W = o; o += (int64_t)C * 128 * 9;
  L.C3b = o; o += C;
  L.total = o;
  return L;
}

namespace {
// what a forward writes besides the layers' input operands: noise, activations and batch statistics
int alloc_fwd(ConvLEnv& e, UpsGen& G) {
  const int S = G.S;
  const size_t B = e.maxB, n0 = G.GL1.Cout, n1 = (size_t)256 * (S / 2) * (S / 2), n2 = (size_t)128 * S * S,
               n3 = (size_t)G.C * S * S;
  for (auto [p, n] : {std::pair<float**, size_t>{&G.noise, kNoiseDim}, {&G.z0, n0}, {&G.h0, n0}, {&G.z1, n1}, {&G.h1, n1},
                      {&G.z2, n2}, {&G.h2, n2}, {&G.z3, n3}, {&G.y, n3}})
    FG_TRY(convl_dalloc(e, p, B * n));
  for (int i = 0; i < 2; ++i) {
    FG_TRY(convl_dalloc(e, &G.bn_mean[i], G.GU[i].Cout));
    FG_TRY(convl_dalloc(e, &G.bn_istd[i], G.GU[i].Cout));
  }
  return FG_OK;
}
}  // namespace

int gen_alloc(ConvLEnv& e, UpsGen& G, const GenDesc& d) {
  fg_ctx* c = e.c;
  const int S = d.side, C = c->C;
  G.S = S;
  G.C = C;
  G.gl = make_g_layout(C, S);
  const GLayout& gl = G.gl;
  auto timer = [&](const char* name) {
    G.names.push_back(std::string(d.prefix) + name);
    return G.names.back().c_str();
  };
  FG_TRY(G.pairs.alloc(c, *e.allocs, 8));  // x and dY of G.L1, G.C1, G.C2 and G.C3
  ConvL& L1 = G.GL1;
  L1.Cin = kNoiseDim; L1.Cout = 128 * (S / 4) * (S / 4); L1.k = 1; L1.H = 1;
  L1.w_off = gl.L1W; L1.b_off = gl.L1b;
  L1.nA = 128; L1.nS = (S / 4) * (S / 4);  // View(128,S/4,S/4): reference row c*nS+s <-> our NHWC row s*128+c
  L1.kpad = d.l1_kpad;                     // K = 100 is no multiple of 32: zero-padded for the tensor cores
  L1.tf = timer("G.L1.fwd"); L1.td = timer("G.L1.dgrad"); L1.tw = timer("G.L1.wgrad");
  ConvL& C3 = G.GC3;
  C3.Cin = 128; C3.Cout = C; C3.k = 3; C3.H = S;
  C3.w_off = gl.C3W; C3.b_off = gl.C3b;
  C3.tf = timer("G.C3.fwd"); C3.td = timer("G.C3.dgrad"); C3.tw = timer("G.C3.wgrad");
  for (ConvL* L : {&L1, &C3}) {
    FG_TRY(G.pairs.take(&L->x.s));
    FG_TRY(G.pairs.take(&L->sdy));
    FG_TRY(convl_alloc(e, *L));
  }
  // G.L1 splits its dY into buffers of its own: with option bwd_streams G.C1's weight gradient on the wgrad stream still
  // reads G.C1's split in the shared ConvLEnv::dy while G.L1 splits
  FG_TRY(convl_dalloc(e, &L1.dy_hi, (size_t)e.maxB * L1.Cout));
  FG_TRY(convl_dalloc(e, &L1.dy_lo, (size_t)e.maxB * L1.Cout));
  static const char* uf[2] = {"G.C1.fwd", "G.C2.fwd"};
  static const char* ud[2] = {"G.C1.dgrad", "G.C2.dgrad"};
  static const char* uw[2] = {"G.C1.wgrad", "G.C2.wgrad"};
  static const char* ub[2] = {"G.C1.wgrad+dgrad", "G.C2.wgrad+dgrad"};
  const int ci[2] = {128, 256}, co[2] = {256, 128}, hs[2] = {S / 2, S};
  const int64_t wo[2] = {gl.C1W, gl.C2W}, bo[2] = {gl.C1b, gl.C2b};
  for (int i = 0; i < 2; ++i) {
    UpsL& U = G.GU[i];
    U.Cin = ci[i]; U.Cout = co[i]; U.H = hs[i];
    U.w_off = wo[i]; U.b_off = bo[i];
    U.tf = timer(uf[i]); U.td = timer(ud[i]); U.tw = timer(uw[i]);
    U.tb = d.bwd_merge ? timer(ub[i]) : nullptr;
    FG_TRY(G.pairs.take(&U.x.s));
    FG_TRY(G.pairs.take(&G.sdz[i]));
    FG_TRY(upsl_alloc(e, U));
  }
  // "hbm.*" timers: the bandwidth-bound kernels bench.py reports against the measured HBM peak
  G.t_bn2_finalize = timer("G.bn2.finalize");
  G.t_bn2_stats = timer("hbm.G.bn2.stats");
  G.t_bn2_apply = timer("hbm.G.bn2.apply");
  G.t_bn2_bwd_reduce = timer("hbm.G.bn2.bwd_reduce");
  G.t_bn2_bwd_apply = timer("hbm.G.bn2.bwd_apply");
  FG_TRY(alloc_fwd(e, G));
  const size_t B = e.maxB, n0 = L1.Cout, n1 = (size_t)256 * (S / 2) * (S / 2), n2 = (size_t)128 * S * S, n3 = (size_t)C * S * S;
  for (auto [p, n] : {std::pair<float**, size_t>{&G.dz3, n3},
                      {&G.dfull, (size_t)256 * S * S},  // full-resolution dgrad of G.C2 on the FFMA path: [B][S][S][256]
                      {&G.dz2, n2}, {&G.dz1, n1}, {&G.dz0, n0}})
    FG_TRY(convl_dalloc(e, p, B * n));
  return convl_dalloc(e, &G.bn_mg, 512);
}

int gen_alloc_fwd(ConvLEnv& e, UpsGen& F, UpsGen& G) {
  F.S = G.S;
  F.C = G.C;
  F.gl = G.gl;
  F.owner = &G;
  // the layers as G's: its weight packs and timer names; the input operands are replaced below
  F.GL1 = G.GL1;
  F.GC3 = G.GC3;
  F.GU[0] = G.GU[0];
  F.GU[1] = G.GU[1];
  F.t_bn2_finalize = G.t_bn2_finalize;
  F.t_bn2_stats = G.t_bn2_stats;
  F.t_bn2_apply = G.t_bn2_apply;
  F.t_bn2_bwd_reduce = G.t_bn2_bwd_reduce;
  F.t_bn2_bwd_apply = G.t_bn2_bwd_apply;
  FG_TRY(F.pairs.alloc(e.c, *e.allocs, 4));  // x of G.L1, G.C1, G.C2 and G.C3
  for (ConvL* L : {&F.GL1, &F.GC3}) {
    L->x = TcOp{};
    L->xpad = nullptr;
    L->sdy = L->dy_hi = L->dy_lo = nullptr;
    FG_TRY(F.pairs.take(&L->x.s));
    FG_TRY(convl_alloc_x(e, *L));
  }
  for (UpsL& U : F.GU) {
    U.x = TcOp{};
    FG_TRY(F.pairs.take(&U.x.s));
    FG_TRY(upsl_alloc_x(e, U));
  }
  return alloc_fwd(e, F);
}

int gen_pack(fg_ctx* c, UpsGen& G, NetPair& p) {
  if (p.G_pack == pack_key(c)) return FG_OK;
  FG_TRY(convl_pack(c, G.GL1, p.PG));
  for (int i = 0; i < 2; ++i) FG_TRY(upsl_pack(c, G.GU[i], p.PG));
  FG_TRY(convl_pack(c, G.GC3, p.PG));
  p.G_pack = pack_key(c);
  return FG_OK;
}

namespace {
// BatchNorm statistics of G.C(i+1)'s output z -> bn_mean[i] / bn_istd[i].  Training: from the convolution epilogue's
// per-tile partials when it ran on the tensor cores (parts > 0), otherwise from a separate pass over z.
int bn_stats(fg_ctx* c, UpsGen& G, NetPair& p, int i, const float* z, int B, bool training, int parts, const char* t_finalize,
             const char* t_stats) {
  const int Cc = G.GU[i].Cout;
  const int64_t P = (int64_t)B * G.GU[i].H * G.GU[i].H;
  float *rm = p.bnG + (i == 0 ? 0 : 512), *rv = rm + Cc;
  if (!training) return k_bn_eval_prep(c, rm, rv, G.bn_mean[i], G.bn_istd[i], Cc);
  if (parts) {
    ScopedTimer tm(c, t_finalize);
    return k_bn_finalize_parts(c, c->bn_parts, parts, 4, G.bn_mean[i], G.bn_istd[i], rm, rv, P, Cc);  // 4 upsampling phases
  }
  {
    ScopedTimer tm(c, t_stats);
    FG_TRY(k_bn_stats(c, z, c->bn_acc, P, Cc));
  }
  return k_bn_finalize(c, c->bn_acc, G.bn_mean[i], G.bn_istd[i], rm, rv, P, Cc);
}
}  // namespace

int gen_forward(ConvLEnv& e, UpsGen& G, NetPair& p, const float* noise, int B, bool training) {
  fg_ctx* c = e.c;
  FG_REQUIRE(B >= 1 && B <= e.maxB, "G forward: batch %d out of range [1,%d]", B, e.maxB);
  if (G.owner) {  // forward-only: the owner's packs, read in the format they were made in
    FG_TRY(gen_pack(c, *G.owner, p));
    G.GL1.packed_f16 = G.owner->GL1.packed_f16;
    G.GC3.packed_f16 = G.owner->GC3.packed_f16;
  } else {
    FG_TRY(gen_pack(c, G, p));
  }
  const GLayout& L = G.gl;
  const float* P = p.PG;
  const int S = G.S;
  if (noise != G.noise)
    FG_CUDA(cudaMemcpyAsync(G.noise, noise, sizeof(float) * B * kNoiseDim, cudaMemcpyDeviceToDevice, c->stream));
  G.B = B;
  G.train = training;
  FG_TRY(G.pairs.reset(c));
  FG_TRY(convl_fwd(e, G.GL1, G.noise, P, G.z0, B));
  {
    AmaxInto am(c, G.GU[0].x);
    FG_TRY(k_prelu_fwd(c, G.z0, P + L.a1, G.h0, (int64_t)B * G.GL1.Cout));
  }
  int parts = training ? 1 : 0;
  FG_TRY(upsl_fwd(e, G.GU[0], G.h0, P, G.z1, B, &parts));
  FG_TRY(bn_stats(c, G, p, 0, G.z1, B, training, parts, nullptr, nullptr));
  UpsL& C2 = G.GU[1];
  C2.x.split_ready = training && upsl_tc(c, C2) && !tc_f16(c);  // the TF32 tensor-core path reads h1 only as its split
  {
    AmaxInto am(c, C2.x);
    FG_TRY(k_bn_prelu_apply(c, G.z1, G.bn_mean[0], G.bn_istd[0], P + L.g1, P + L.be1, P + L.a2, G.h1,
                            (int64_t)B * (S / 2) * (S / 2), 256, C2.x.split_ready ? C2.x.hi : nullptr,
                            C2.x.split_ready ? C2.x.lo : nullptr));
  }
  parts = training ? 1 : 0;
  FG_TRY(upsl_fwd(e, C2, G.h1, P, G.z2, B, &parts));
  FG_TRY(bn_stats(c, G, p, 1, G.z2, B, training, parts, G.t_bn2_finalize, G.t_bn2_stats));
  {
    ScopedTimer tm(c, G.t_bn2_apply);
    FG_TRY(k_bn_prelu_apply(c, G.z2, G.bn_mean[1], G.bn_istd[1], P + L.g2, P + L.be2, P + L.a3, G.h2, (int64_t)B * S * S, 128));
  }
  FG_TRY(convl_fwd(e, G.GC3, G.h2, P, G.z3, B));
  FG_TRY(k_sigmoid_fwd(c, G.z3, G.y, (int64_t)B * S * S * G.C));
  G.valid = true;
  return FG_OK;
}

int gen_backward(ConvLEnv& e, UpsGen& G, NetPair& p, const float* dy, float* dnoise) {
  fg_ctx* c = e.c;
  if (!G.valid || !G.train) {
    fg_set_error("G backward needs a preceding training-mode G forward");
    return FG_ERR_STATE;
  }
  const GLayout& L = G.gl;
  const float* P = p.PG;
  float* g = p.gG;
  const int B = G.B, S = G.S, h = S / 2;
  FG_TRY(G.pairs.reset(c));
  FG_TRY(k_sigmoid_bwd(c, dy, G.y, G.dz3, (int64_t)B * S * S * G.C));
  // option bwd_streams: G.C3's weight gradient (a read of all of h2) beside its data gradient and the BN2 backward; it
  // reads h2 and dz3, which nothing below writes.  G.L1's stays here: with no noise gradient it is the last launch of
  // the pass, so on another stream it would overlap nothing (it runs beside G.C1's instead).
  FG_TRY(convl_bwd(e, G.GC3, G.h2, G.dz3, g, G.dfull, B, wgrad_async(c, e)));
  // BN2 + PReLU
  {
    ScopedTimer tm(c, G.t_bn2_bwd_reduce);
    FG_TRY(k_bn_prelu_bwd_reduce(c, G.dfull, G.z2, G.bn_mean[1], G.bn_istd[1], P + L.g2, P + L.be2, P + L.a3, c->bn_acc,
                                 g + L.a3, B, S, S, 128, 0));
  }
  FG_TRY(k_bn_bwd_finalize(c, c->bn_acc, G.bn_mg, g + L.g2, g + L.be2, (int64_t)B * S * S, 128));
  // in tensor-core mode the BN-backward kernels also emit the TF32 hi/lo split of dz (no separate split pass); with the
  // FP16 split they reduce max|dz| into dz's own scale pair
  const bool tf32 = !tc_f16(c);
  TcOp dz2{e.dy.hi, e.dy.lo, G.sdz[1]};
  dz2.split_ready = upsl_tc(c, G.GU[1]) && tf32;
  {
    ScopedTimer tm(c, G.t_bn2_bwd_apply);
    AmaxInto am(c, dz2);
    FG_TRY(k_bn_prelu_bwd_apply(c, G.dfull, G.z2, G.bn_mean[1], G.bn_istd[1], P + L.g2, P + L.be2, P + L.a3, G.bn_mg, G.dz2,
                                B, S, S, 128, 0, dz2.split_ready ? dz2.hi : nullptr, dz2.split_ready ? dz2.lo : nullptr,
                                g + L.C2b));  // + the bias gradient of C2 (column sums of dz2) in the same pass
  }
  // C2
  bool pooled = false;
  FG_TRY(upsl_bwd(e, G.GU[1], dz2, G.h1, G.dz2, g, G.dfull, B, &pooled));
  // BN1 + PReLU (the 2x2 sum = backward of the nearest upsample is folded into the loads)
  FG_TRY(k_bn_prelu_bwd_reduce(c, G.dfull, G.z1, G.bn_mean[0], G.bn_istd[0], P + L.g1, P + L.be1, P + L.a2, c->bn_acc,
                               g + L.a2, B, h, h, 256, pooled ? 0 : 1));
  FG_TRY(k_bn_bwd_finalize(c, c->bn_acc, G.bn_mg, g + L.g1, g + L.be1, (int64_t)B * h * h, 256));
  TcOp dz1{e.dy.hi, e.dy.lo, G.sdz[0]};
  dz1.split_ready = upsl_tc(c, G.GU[0]) && tf32 && pooled;
  {
    AmaxInto am(c, dz1);
    FG_TRY(k_bn_prelu_bwd_apply(c, G.dfull, G.z1, G.bn_mean[0], G.bn_istd[0], P + L.g1, P + L.be1, P + L.a2, G.bn_mg, G.dz1,
                                B, h, h, 256, pooled ? 0 : 1, dz1.split_ready ? dz1.hi : nullptr,
                                dz1.split_ready ? dz1.lo : nullptr, g + L.C1b));
  }
  // C1
  // option bwd_streams: G.C1's weight gradient beside its data gradient and the G.L1 tail; it reads h0's split and dz1's
  // in ConvLEnv::dy, which G.L1 (splitting into its own buffers) leaves alone.  Where the merged launch runs (bwd_merge)
  // there is no separate weight gradient to move.
  FG_TRY(upsl_bwd(e, G.GU[0], dz1, G.h0, G.dz1, g, G.dfull, B, &pooled, wgrad_async(c, e)));
  {
    AmaxInto am(c, G.GL1.sdy, &e.dy.amax_ready);
    FG_TRY(k_prelu_bwd(c, G.dfull, G.z0, P + L.a1, G.dz0, g + L.a1, B, S / 4, S / 4, 128, pooled ? 0 : 1));
  }
  FG_TRY(convl_bwd(e, G.GL1, G.noise, G.dz0, g, dnoise, B));
  return wgrad_join(e);
}

void gen_debug_rows(const UpsGen& G, std::vector<DebugTensor>& rows) {
  const int64_t n0 = G.GL1.Cout, n1 = 256 * (G.S / 2) * (G.S / 2), n2 = 128 * G.S * G.S, n3 = (int64_t)G.C * G.S * G.S;
  const int B = G.B;
  for (const DebugTensor& r : {DebugTensor{"G.z0", G.z0, n0, B}, {"G.h0", G.h0, n0, B}, {"G.z1", G.z1, n1, B},
                               {"G.h1", G.h1, n1, B}, {"G.z2", G.z2, n2, B}, {"G.h2", G.h2, n2, B}, {"G.z3", G.z3, n3, B},
                               {"G.y", G.y, n3, B}, {"G.dz2", G.dz2, n2, B}, {"G.dz1", G.dz1, n1, B}, {"G.dz0", G.dz0, n0, B},
                               {"G.bn_mean1", G.bn_mean[0], 256, 1}, {"G.bn_istd1", G.bn_istd[0], 256, 1},
                               {"G.bn_mean2", G.bn_mean[1], 128, 1}, {"G.bn_istd2", G.bn_istd[1], 128, 1}})
    rows.push_back({r.name, G.valid ? r.p : nullptr, r.per, r.B});  // nothing before the first forward
}
