// The branched discriminators of models.lua: create_D32 (:322-376) at 32x32 and create_D16_d (:279-316, the --scale 16
// default), create_D16 (:110-159), create_D16_b (:161-216), create_D16_c (:218-277) at 16x16.  Each is
//   ConcatTable{branch, ...} -> JoinTable(2) [-> Linear -> PReLU -> Dropout] -> Linear(1) -> Sigmoid
// and differs from the others only in data: one descriptor (DbrDesc) per net, one GanD type (DBr) built from it.
//   conv branch : conv (PReLU) [MaxPool(2,2) | AvgPool(2,2)] ... SpatialDropout View Linear PReLU [Dropout] [Linear PReLU]
//   dense branch: View(C*S*S) Linear PReLU Dropout Linear PReLU
// create_D32 and create_D16 / _b / _c have a fine (3x3) and a coarse (5x5) conv branch, a dense branch and a hidden
// head; create_D16_d has one conv branch, a dense branch and no hidden head.
// Every convolution and Linear is a ConvL (convl.h) through the shared dispatch.  A stride-2 "same" convolution is the
// stride-1 one sampled at the even pixels: forward = stride-1 kernel + subsample, backward = the stride-1 dgrad / wgrad
// of dY with zeros inserted at the odd pixels.  That is exact (the inserted zeros contribute nothing) and keeps the
// layer on the tensor cores.  The elementwise stages are one kernel pair: PReLU -> optional 2x2 max pooling -> optional
// (spatial) dropout forward, writing the window's arg-max, and its backward, which reduces the PReLU slope gradient in
// a fixed order (k_ordered.cuh), so a step stays bit-reproducible.  A 2x2 average pooling runs after its stage's PReLU
// as a kernel of its own.
#include <deque>
#include <string>

#include "fg_internal.h"
#include "k_misc.h"
#include "k_ordered.cuh"
#include "ups_gan.h"

namespace {
constexpr float kP = 0.5f;  // nn.SpatialDropout() / nn.Dropout() default probability

// ---- descriptor --------------------------------------------------------------------------------------------------
// the names a layer's timers and debug rows take instead of the generated "D.<branch>.*" ones (each may be null):
// timer stem t (t.fwd / .dgrad / .wgrad), pre-activation z ("D.z", "Dstep.z"), stage output h ("D.h")
struct DbrNames {
  const char *t, *z, *h;
};
enum DbrPool { kNoPool, kMaxPool, kAvgPool };  // nn.SpatialMaxPooling(2, 2) / nn.SpatialAveragePooling(2, 2) after the PReLU
struct DbrConvDesc {
  int cout, k, stride;
  DbrPool pool;
  DbrNames nm;
};
struct DbrLinDesc {
  int out;
  bool drop;  // nn.Dropout() after the PReLU
  DbrNames nm;
};
// a conv branch ends in nn.SpatialDropout() + View; a branch without convolutions is the dense branch (View of the image)
struct DbrBranchDesc {
  const char* name;
  int nconv;
  DbrConvDesc conv[5];
  int nlin;
  DbrLinDesc lin[2];
};
struct DbrDesc {
  int disc, side, nbr;
  DbrBranchDesc br[3];  // ConcatTable order
  // Linear(joint, head.out) PReLU Dropout, then Linear(head.out, 1); head.out 0: Linear(joint, 1) on the joint row
  DbrLinDesc head;
};

constexpr DbrBranchDesc kDense = {"dense", 0, {}, 2, {{1024, true}, {1024, false}}};
const DbrDesc kDescs[] = {
    {FG_DISC_D32, 32, 3,
     {{"fine", 2, {{64, 3, 1, kNoPool}, {64, 3, 1, kMaxPool}}, 1, {{1024, false}}},
      {"coarse", 4, {{32, 5, 1, kNoPool}, {32, 5, 1, kMaxPool}, {54, 5, 1, kNoPool}, {54, 5, 1, kMaxPool}}, 2,
       {{1024, true}, {1024, false}}},
      kDense},
     {1024, true}},
    {FG_DISC_D16_D, 16, 2,
     {{"conv", 4,
       {{128, 3, 1, kNoPool, {"s16.D.c1", "z1"}},
        {128, 3, 1, kAvgPool, {"s16.D.c2", "z2", "p1"}},
        {512, 3, 2, kNoPool, {"s16.D.c3", "z3"}},
        {1024, 3, 2, kNoPool, {"s16.D.c4", "z4"}}},
       1, {{1024, false, {"s16.D.F1", "zf"}}}},
      {"dense", 0, {}, 2, {{128, true, {"s16.D.E1", "ze1"}}, {128, false, {"s16.D.E2", "ze2"}}}}},
     {0, false}},
    {FG_DISC_D16, 16, 3,
     {{"fine", 2, {{64, 3, 1, kNoPool}, {64, 3, 1, kMaxPool}}, 1, {{1024, true}}},
      {"coarse", 2, {{32, 5, 1, kNoPool}, {64, 5, 1, kMaxPool}}, 1, {{1024, true}}},
      kDense},
     {1024, true}},
    {FG_DISC_D16_B, 16, 3,
     {{"fine", 4, {{64, 3, 1, kNoPool}, {64, 3, 1, kNoPool}, {128, 3, 1, kNoPool}, {128, 3, 2, kNoPool}}, 1, {{512, true}}},
      {"coarse", 4, {{64, 5, 1, kNoPool}, {64, 5, 1, kNoPool}, {128, 5, 1, kNoPool}, {128, 5, 2, kNoPool}}, 1, {{512, true}}},
      kDense},
     {1024, true}},
    {FG_DISC_D16_C, 16, 3,
     {{"fine", 5,
       {{64, 3, 1, kNoPool}, {64, 3, 1, kNoPool}, {128, 3, 1, kNoPool}, {128, 3, 2, kNoPool}, {512, 3, 2, kNoPool}}, 1,
       {{1024, false}}},
      {"coarse", 5,
       {{64, 5, 1, kNoPool}, {64, 5, 1, kNoPool}, {128, 5, 1, kNoPool}, {128, 5, 2, kNoPool}, {512, 5, 2, kNoPool}}, 1,
       {{1024, false}}},
      kDense},
     {1024, true}},
};

const DbrDesc* find_desc(int disc) {
  for (const DbrDesc& d : kDescs)
    if (d.disc == disc) return &d;
  return nullptr;
}

// ---- kernels -----------------------------------------------------------------------------------------------------
// The multiplier of a (spatial) dropout on output (b, ch): keep flag * train_scale in training (keep != null), else
// eval_scale.  nn.SpatialDropout: train 1, eval 1-p; nn.Dropout: train 1/(1-p), eval 1; none: keep null, eval 1.
__device__ __forceinline__ float drop_mul(const float* __restrict__ keep, int64_t mstride, int moff, int64_t b, int ch,
                                          float train_scale, float eval_scale) {
  return keep ? keep[b * mstride + moff + ch] * train_scale : eval_scale;
}

// z [B][H][W][C] -> y [B][H/POOL][W/POOL][C] = drop(maxpool_POOL(prelu(z))); code (POOL 2): the window's arg-max
// (0..3, row-major, first strict maximum)
template <int POOL>
__global__ void __launch_bounds__(256) dbr_act_fwd_kernel(const float* __restrict__ z, const float* __restrict__ slope,
                                                          const float* __restrict__ keep, int64_t mstride, int moff,
                                                          float train_scale, float eval_scale, float* __restrict__ y,
                                                          uint8_t* __restrict__ code, int B, int H, int W, int C) {
  const float a = *slope;
  const int Ho = H / POOL, Wo = W / POOL;
  const int64_t n = (int64_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    float m;
    int64_t b;
    if (POOL == 2) {
      int64_t r = i / C;
      const int xo = (int)(r % Wo);
      r /= Wo;
      const int yo = (int)(r % Ho);
      b = r / Ho;
      const int64_t base = ((b * H + 2 * yo) * W + 2 * xo) * C + ch, rs = (int64_t)W * C;
      const float v0 = z[base], v1 = z[base + C], v2 = z[base + rs], v3 = z[base + rs + C];
      code[i] = (uint8_t)argmax4(v0 > 0.f ? v0 : a * v0, v1 > 0.f ? v1 : a * v1, v2 > 0.f ? v2 : a * v2,
                                 v3 > 0.f ? v3 : a * v3, &m);
    } else {
      b = i / ((int64_t)H * W * C);
      const float v = z[i];
      m = v > 0.f ? v : a * v;
    }
    y[i] = m * drop_mul(keep, mstride, moff, b, ch, train_scale, eval_scale);
  }
}

// the adjoint: dz [B][H][W][C] from dy [B][H/POOL][W/POOL][C]: the dropout multiplier, dY routed to the window's
// arg-max (zeros elsewhere), PReLU's derivative at z; *dslope += sum over routed z <= 0 of dY * z, summed per block in
// a fixed order and the blocks in block order
template <int POOL>
__global__ void __launch_bounds__(256) dbr_act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ z,
                                                          const uint8_t* __restrict__ code, const float* __restrict__ slope,
                                                          const float* __restrict__ keep, int64_t mstride, int moff,
                                                          float train_scale, float eval_scale, float* __restrict__ dz,
                                                          float* __restrict__ dslope, int B, int H, int W, int C,
                                                          double* __restrict__ ws, unsigned* __restrict__ ticket) {
  const float a = *slope;
  const int Ho = H / POOL, Wo = W / POOL;
  const int64_t n = (int64_t)B * Ho * Wo * C;
  double s = 0;
  GRID_STRIDE(i, n) {
    const int ch = (int)(i % C);
    if (POOL == 2) {
      int64_t r = i / C;
      const int xo = (int)(r % Wo);
      r /= Wo;
      const int yo = (int)(r % Ho);
      const int64_t b = r / Ho;
      const float g = dy[i] * drop_mul(keep, mstride, moff, b, ch, train_scale, eval_scale);
      const int64_t base = ((b * H + 2 * yo) * W + 2 * xo) * C + ch, rs = (int64_t)W * C;
      const int j = code[i];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t o = base + (q & 1) * (int64_t)C + (q >> 1) * rs;
        float d = 0.f;
        if (q == j) {
          const float v = z[o];
          if (v > 0.f) {
            d = g;
          } else {
            d = a * g;
            s += (double)g * (double)v;
          }
        }
        dz[o] = d;
      }
    } else {
      const int64_t b = i / ((int64_t)H * W * C);
      const float g = dy[i] * drop_mul(keep, mstride, moff, b, ch, train_scale, eval_scale);
      const float v = z[i];
      if (v > 0.f) {
        dz[i] = g;
      } else {
        dz[i] = a * g;
        s += (double)g * (double)v;
      }
    }
  }
  if (!dslope) return;
  s = block_sum(s);
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *dslope += (float)ordered_sum(ws, gridDim.x, 1, 0);
    ordered_release(ticket);
  }
}

// nn.SpatialAveragePooling(2,2,2,2): x [B][H][W][C] -> y [B][H/2][W/2][C], and its adjoint
__global__ void __launch_bounds__(256) avgpool2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H,
                                                           int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  GRID_STRIDE(i, (int64_t)B * Ho * Wo * C) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    const float* p = x + (((b * H + 2 * yo) * W + 2 * xo) * (int64_t)C + ch);
    y[i] = 0.25f * ((p[0] + p[C]) + (p[(int64_t)W * C] + p[(int64_t)W * C + C]));
  }
}
__global__ void __launch_bounds__(256) avgpool2_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int H,
                                                           int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  GRID_STRIDE(i, (int64_t)B * H * W * C) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H);
    const int64_t b = r / H;
    dx[i] = 0.25f * dy[((b * Ho + yy / 2) * Wo + xx / 2) * (int64_t)C + ch];
  }
}
// the stride-2 sampling of a stride-1 "same" convolution output: y[b][yo][xo][c] = x[b][2yo][2xo][c] (H, W: the
// stride-1 size), and its adjoint: dx[b][y][x][c] = (y, x both even) ? dy[b][y/2][x/2][c] : 0
__global__ void __launch_bounds__(256) subsample2_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H,
                                                         int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  GRID_STRIDE(i, (int64_t)B * Ho * Wo * C) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t b = r / Ho;
    y[i] = x[((b * H + 2 * yo) * W + 2 * xo) * (int64_t)C + ch];
  }
}
__global__ void __launch_bounds__(256) zero_insert2_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int H,
                                                           int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  GRID_STRIDE(i, (int64_t)B * H * W * C) {
    const int ch = (int)(i % C);
    int64_t r = i / C;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H);
    const int64_t b = r / H;
    dx[i] = ((xx | yy) & 1) ? 0.f : dy[((b * Ho + yy / 2) * Wo + xx / 2) * (int64_t)C + ch];
  }
}

// nn.JoinTable(2) of two or three inputs [B][w_k] -> [B][sum w_k] (w[2] = 0 for two), and the split of its gradient
constexpr int kMaxJoin = 3;
struct JoinArgs {
  float* p[kMaxJoin];
  int w[kMaxJoin];
};
__device__ __forceinline__ float* join_slot(const JoinArgs& a, int64_t i, int N) {  // static indices: no local memory
  int j = (int)(i % N);
  const int64_t r = i / N;
  if (j < a.w[0]) return a.p[0] + r * a.w[0] + j;
  j -= a.w[0];
  if (j < a.w[1]) return a.p[1] + r * a.w[1] + j;
  return a.p[2] + r * a.w[2] + (j - a.w[1]);
}
__global__ void __launch_bounds__(256) joinN_kernel(JoinArgs a, float* __restrict__ out, int B, int N) {
  GRID_STRIDE(i, (int64_t)B * N) out[i] = *join_slot(a, i, N);
}
__global__ void __launch_bounds__(256) splitN_kernel(JoinArgs a, const float* __restrict__ in, int B, int N) {
  GRID_STRIDE(i, (int64_t)B * N) *join_slot(a, i, N) = in[i];
}

// ---- the net -----------------------------------------------------------------------------------------------------
// one PReLU [-> MaxPool(2,2) | AvgPool(2,2)] [-> (spatial) dropout] stage on a [B][H][W][C] pre-activation z
struct Act {
  int64_t a_off = 0;  // slope
  int H = 1, W = 1, C = 0, pool = 1;
  bool avg = false;  // pool 2 is an average: the PReLU (and dropout) into DBr::full, then the average into h
  int moff = -1;     // keep-flag offset in the sample's row; -1: no dropout
  float train_scale = 1.f, eval_scale = 1.f;
  float *z = nullptr, *h = nullptr;
  uint8_t* code = nullptr;
  int64_t out_per() const { return (int64_t)(H / pool) * (W / pool) * C; }
};
struct Layer {
  ConvL L;
  int stride = 1;
  Act act;
  const float* in = nullptr;  // its forward input
};
struct Branch {
  std::vector<Layer> conv, lin;
  int out = 0;                                   // width of its output row
  float *dsplit = nullptr, *dxb = nullptr;       // its share of the joint gradient, its input gradient
};

struct DBr final : GanD {
  const DbrDesc& dd;
  int mask = 0;
  Branch br[3];
  Layer head;             // when dd.head.out
  int64_t JW = 0, Jb = 0;  // the last Linear(top_w, 1)
  int joint_w = 0, top_w = 0;  // widths of the joint row and of the last Linear's input
  // full: the stride-1 output of a stride-2 convolution, or the PReLU of an average-pooled stage before its pooling
  float *full = nullptr, *joint = nullptr, *djoint = nullptr, *ga = nullptr, *gb = nullptr;
  bool train = true, valid = false;
  std::deque<std::string> names;  // timer and debug names (stable storage)
  std::vector<DebugTensor> rows;   // "D.*" of fg_*debug_tensor

  explicit DBr(const DbrDesc& d) : dd(d) {}
  const char* name(const std::string& s) {
    names.push_back(s);
    return names.back().c_str();
  }
  std::vector<Layer*> layers() {
    std::vector<Layer*> v;
    for (int k = 0; k < dd.nbr; ++k) {
      for (Layer& l : br[k].conv) v.push_back(&l);
      for (Layer& l : br[k].lin) v.push_back(&l);
    }
    if (dd.head.out) v.push_back(&head);
    return v;
  }
  int64_t layout(int C) override;
  int dalloc(float** q, size_t elems) { return convl_dalloc(n->env, q, elems); }
  int alloc() override;
  int act_fwd(const Act& A, int Bn, bool training);
  int act_bwd(const Act& A, const float* dy, float* dz, float* G, int Bn);
  int forward(const float* x, int B, bool training, const fg_hyper* h) override;
  int backward(bool want_wgrad, bool want_dx) override;
  int draw_masks(int Bn, uint64_t seed, const fg_hyper*, const uint64_t* root) override {
    return k_bernoulli_keep(n->c, masks, (int64_t)Bn * mask, seed, kP, root);
  }
  void debug_rows(std::vector<DebugTensor>& ents) const override {
    for (const DebugTensor& r : rows) ents.push_back({r.name, valid ? r.p : nullptr, r.per, B});
  }
};

// getParameters() order: module order through the ConcatTable, then the head; keep flags in the same order
int64_t DBr::layout(int C) {
  names.clear();
  int64_t o = 0;
  int m = 0;
  auto timers = [&](ConvL& L, const char* t, const std::string& gen) {
    const std::string s = t ? t : gen;
    L.tf = name(s + ".fwd");
    L.td = name(s + ".dgrad");
    L.tw = name(s + ".wgrad");
  };
  auto linear = [&](Layer& l, const std::string& pre, int j, int cin, const DbrLinDesc& ld, int cA, int cS) {
    ConvL& L = l.L;
    L.Cin = cin; L.Cout = ld.out; L.k = 1; L.H = 1;
    L.cA = cA; L.cS = cS;  // View flattens [C][H][W]; ours is [H][W][C]
    L.w_off = o; o += (int64_t)ld.out * cin;
    L.b_off = o; o += ld.out;
    l.act.a_off = o; o += 1;
    l.act.C = ld.out;
    timers(L, ld.nm.t, pre + ".L" + std::to_string(j + 1));
    if (ld.drop) {  // nn.Dropout(): 1/(1-p) in training, identity in evaluation
      l.act.moff = m;
      m += ld.out;
      l.act.train_scale = 1.f / (1.f - kP);
    }
  };
  joint_w = 0;
  for (int k = 0; k < dd.nbr; ++k) {
    const DbrBranchDesc& bd = dd.br[k];
    Branch& b = br[k];
    const std::string pre = std::string("D.") + bd.name;
    b.conv.assign(bd.nconv, Layer{});
    b.lin.assign(bd.nlin, Layer{});
    int s = dd.side, cin = C;
    for (int i = 0; i < bd.nconv; ++i) {
      const DbrConvDesc& cd = bd.conv[i];
      Layer& l = b.conv[i];
      ConvL& L = l.L;
      L.Cin = cin; L.Cout = cd.cout; L.k = cd.k; L.H = s;
      L.w_off = o; o += (int64_t)cd.cout * cin * cd.k * cd.k;
      L.b_off = o; o += cd.cout;
      l.act.a_off = o; o += 1;
      timers(L, cd.nm.t, pre + ".c" + std::to_string(i + 1));
      l.stride = cd.stride;
      s /= cd.stride;
      l.act.H = l.act.W = s;
      l.act.C = cd.cout;
      l.act.pool = cd.pool == kNoPool ? 1 : 2;
      l.act.avg = cd.pool == kAvgPool;
      s /= l.act.pool;
      cin = cd.cout;
    }
    if (bd.nconv) {  // nn.SpatialDropout(): one flag per plane, no rescale in training, 1-p in evaluation
      Act& a = b.conv.back().act;
      a.moff = m;
      m += cin;
      a.eval_scale = 1.f - kP;
    }
    for (int j = 0; j < bd.nlin; ++j)
      linear(b.lin[j], pre, j, j ? bd.lin[j - 1].out : cin * s * s, bd.lin[j], j ? 0 : cin, j ? 0 : s * s);
    b.out = bd.lin[bd.nlin - 1].out;
    joint_w += b.out;
  }
  head = Layer{};
  if (dd.head.out) linear(head, "D.head", 0, joint_w, dd.head, 0, 0);
  top_w = dd.head.out ? dd.head.out : joint_w;
  JW = o; o += top_w;
  Jb = o; o += 1;
  mask = m;
  return o;
}

int DBr::alloc() {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  const size_t B = e.maxB, C = c->C, S = dd.side;
  // the scratch both nets share: the largest dY split and weight gradient of either net (G's needs from the trainer)
  size_t dy = n->g_dy, ws = n->g_ws, g = B * S * S * C, nfull = 0;
  for (Layer* l : layers()) {
    ConvL& L = l->L;
    const size_t P = B * L.H * L.H;
    dy = std::max(dy, P * L.Cout);
    ws = std::max(ws, (size_t)L.k * L.k * L.Cout * L.Cin);
    g = std::max(g, std::max(P * L.Cout, P * L.Cin));
    if (l->stride == 2) nfull = std::max(nfull, P * L.Cout);
    if (l->act.avg) nfull = std::max(nfull, B * l->act.H * l->act.W * l->act.C);
    FG_TRY(convl_alloc(e, L));
  }
  FG_TRY(dalloc(&e.ws, ws));
  FG_TRY(dalloc(&e.dy.hi, dy));
  FG_TRY(dalloc(&e.dy.lo, dy));
  FG_TRY(dalloc(&ga, g));
  FG_TRY(dalloc(&gb, g));
  if (nfull) FG_TRY(dalloc(&full, nfull));
  FG_TRY(dalloc(&x, B * S * S * C));
  FG_TRY(dalloc(&dx, B * S * S * C));
  rows.clear();
  n->net.keep.clear();
  // a pre-activation's "D.*" row and "Dstep.*" keep entry: nm.z, else the generated name
  auto zrow = [&](const DbrNames& nm, const std::string& gen, float* p, int64_t per) {
    const std::string zn = nm.z ? nm.z : gen;
    rows.push_back({name("D." + zn), p, per, 0});
    n->net.keep.push_back({name("Dstep." + zn), p, per});
  };
  for (int k = 0; k < dd.nbr; ++k) {
    const DbrBranchDesc& bd = dd.br[k];
    Branch& b = br[k];
    const std::string pre = std::string(bd.name) + ".";
    const float* in = x;
    for (int i = 0; i < bd.nconv; ++i) {
      Layer& l = b.conv[i];
      Act& a = l.act;
      const int64_t zper = (int64_t)a.H * a.W * a.C;
      const DbrNames& nm = bd.conv[i].nm;
      l.in = in;
      FG_TRY(dalloc(&a.z, B * zper));
      FG_TRY(dalloc(&a.h, B * a.out_per()));
      if (a.pool == 2 && !a.avg) {
        float* q;
        FG_TRY(dalloc(&q, (B * a.out_per() + 3) / 4));
        a.code = reinterpret_cast<uint8_t*>(q);
      }
      zrow(nm, pre + "z" + std::to_string(i + 1), a.z, zper);
      rows.push_back({name("D." + (nm.h ? std::string(nm.h) : pre + "h" + std::to_string(i + 1))), a.h, a.out_per(), 0});
      in = a.h;
    }
    for (int j = 0; j < bd.nlin; ++j) {
      Layer& l = b.lin[j];
      l.in = in;
      FG_TRY(dalloc(&l.act.z, B * l.act.C));
      FG_TRY(dalloc(&l.act.h, B * l.act.C));
      zrow(bd.lin[j].nm, pre + "zl" + std::to_string(j + 1), l.act.z, l.act.C);
      in = l.act.h;
    }
    FG_TRY(dalloc(&b.dsplit, B * b.out));
    if (k) FG_TRY(dalloc(&b.dxb, B * S * S * C));
  }
  br[0].dxb = dx;
  FG_TRY(dalloc(&joint, B * joint_w));
  FG_TRY(dalloc(&djoint, B * joint_w));
  rows.push_back({"D.joint", joint, joint_w, 0});
  if (dd.head.out) {
    head.in = joint;
    FG_TRY(dalloc(&head.act.z, B * head.act.C));
    FG_TRY(dalloc(&head.act.h, B * head.act.C));
    zrow({}, "head.z", head.act.z, head.act.C);
  }
  FG_TRY(dalloc(&logit, B));
  FG_TRY(dalloc(&out, B));
  FG_TRY(dalloc(&dlogit, B));
  FG_TRY(dalloc(&masks, B * mask));
  rows.insert(rows.end(), {{"D.logit", logit, 1, 0}, {"D.out", out, 1, 0}, {"D.masks", masks, mask, 0},
                           {"D.dx", dx, (int64_t)(S * S * C), 0}});
  n->net.keep.insert(n->net.keep.end(), {{"Dstep.logit", logit, 1}, {"Dstep.out", out, 1}});
  return FG_OK;
}

int DBr::act_fwd(const Act& A, int Bn, bool training) {
  fg_ctx* c = n->c;
  const float* keep = training && A.moff >= 0 ? masks : nullptr;
  const float es = training ? 1.f : A.eval_scale;
  const float* P = n->net.PD;
  if (A.pool == 2 && !A.avg) {
    const int64_t nout = (int64_t)Bn * A.out_per();
    dbr_act_fwd_kernel<2><<<grid_for(nout, 256), 256, 0, c->stream>>>(A.z, P + A.a_off, keep, mask, A.moff, A.train_scale,
                                                                       es, A.h, A.code, Bn, A.H, A.W, A.C);
    LAUNCH_CHECK(c);
    return FG_OK;
  }
  const int64_t nz = (int64_t)Bn * A.H * A.W * A.C;
  dbr_act_fwd_kernel<1><<<grid_for(nz, 256), 256, 0, c->stream>>>(A.z, P + A.a_off, keep, mask, A.moff, A.train_scale, es,
                                                                   A.avg ? full : A.h, nullptr, Bn, A.H, A.W, A.C);
  LAUNCH_CHECK(c);
  if (A.avg) {
    avgpool2_fwd_kernel<<<grid_for((int64_t)Bn * A.out_per(), 256), 256, 0, c->stream>>>(full, A.h, Bn, A.H, A.W, A.C);
    LAUNCH_CHECK(c);
  }
  return FG_OK;
}

// dy: the gradient of A.h, or of the PReLU's full-size output on an average-pooled stage
int DBr::act_bwd(const Act& A, const float* dy, float* dz, float* G, int Bn) {
  fg_ctx* c = n->c;
  const float* keep = train && A.moff >= 0 ? masks : nullptr;
  const float es = train ? 1.f : A.eval_scale;
  const float* P = n->net.PD;
  float* ds = G ? G + A.a_off : nullptr;
  const bool max2 = A.pool == 2 && !A.avg;
  const int64_t nout = (int64_t)Bn * (max2 ? A.out_per() : (int64_t)A.H * A.W * A.C);
  const int grid = grid_for(nout, 256, 132 * 8);
  FG_TRY(red_check(c, grid, 1));
  if (max2)
    dbr_act_bwd_kernel<2><<<grid, 256, 0, c->stream>>>(dy, A.z, A.code, P + A.a_off, keep, mask, A.moff, A.train_scale, es,
                                                       dz, ds, Bn, A.H, A.W, A.C, c->red_ws, c->red_ticket);
  else
    dbr_act_bwd_kernel<1><<<grid, 256, 0, c->stream>>>(dy, A.z, nullptr, P + A.a_off, keep, mask, A.moff, A.train_scale, es,
                                                       dz, ds, Bn, A.H, A.W, A.C, c->red_ws, c->red_ticket);
  LAUNCH_CHECK(c);
  return FG_OK;
}

int DBr::forward(const float* xin, int Bn, bool training, const fg_hyper*) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  FG_REQUIRE(Bn >= 1 && Bn <= e.maxB, "D forward: batch %d out of range [1,%d]", Bn, e.maxB);
  std::vector<ConvL*> Ls;
  for (Layer* l : layers()) Ls.push_back(&l->L);
  FG_TRY(gan_pack_D(*n, Ls));
  const float* P = n->net.PD;
  const int S = dd.side;
  if (xin != x) FG_CUDA(cudaMemcpyAsync(x, xin, sizeof(float) * (size_t)Bn * S * S * c->C, cudaMemcpyDeviceToDevice, c->stream));
  JoinArgs ja{};
  for (int k = 0; k < dd.nbr; ++k) {
    Branch& b = br[k];
    for (Layer& l : b.conv) {
      if (l.stride == 2) {  // stride 1, then every other pixel
        const int H = l.L.H, Co = l.L.Cout;
        FG_TRY(convl_fwd(e, l.L, l.in, P, full, Bn));
        subsample2_kernel<<<grid_for((int64_t)Bn * (H / 2) * (H / 2) * Co, 256), 256, 0, c->stream>>>(full, l.act.z, Bn, H,
                                                                                                      H, Co);
        LAUNCH_CHECK(c);
      } else {
        FG_TRY(convl_fwd(e, l.L, l.in, P, l.act.z, Bn));
      }
      FG_TRY(act_fwd(l.act, Bn, training));
    }
    for (Layer& l : b.lin) {
      FG_TRY(convl_fwd(e, l.L, l.in, P, l.act.z, Bn));
      FG_TRY(act_fwd(l.act, Bn, training));
    }
    ja.p[k] = b.lin.back().act.h;
    ja.w[k] = b.out;
  }
  joinN_kernel<<<grid_for((int64_t)Bn * joint_w, 256), 256, 0, c->stream>>>(ja, joint, Bn, joint_w);
  LAUNCH_CHECK(c);
  const float* top = joint;
  if (dd.head.out) {
    FG_TRY(convl_fwd(e, head.L, joint, P, head.act.z, Bn));
    FG_TRY(act_fwd(head.act, Bn, training));
    top = head.act.h;
  }
  FG_TRY(k_gemv_fwd(c, top, P + JW, P + Jb, logit, Bn, top_w));
  B = Bn;
  train = training;
  valid = true;
  return FG_OK;
}

// want_dx: the image gradient is the sum of the branches' (nn.ConcatTable backward), in branch order
int DBr::backward(bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  if (!valid) {
    fg_set_error("D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const float* P = n->net.PD;
  float* G = want_wgrad ? n->net.gD : nullptr;
  if (dd.head.out) {
    if (G) FG_TRY(k_gemv_wgrad_add(c, head.act.h, dlogit, G + JW, G + Jb, B, top_w));
    FG_TRY(k_gemv_dgrad(c, dlogit, P + JW, ga, B, top_w));
    FG_TRY(act_bwd(head.act, ga, gb, G, B));
    FG_TRY(convl_bwd(e, head.L, joint, gb, G, djoint, B));
  } else {
    if (G) FG_TRY(k_gemv_wgrad_add(c, joint, dlogit, G + JW, G + Jb, B, top_w));
    FG_TRY(k_gemv_dgrad(c, dlogit, P + JW, djoint, B, top_w));
  }
  JoinArgs ja{};
  for (int k = 0; k < dd.nbr; ++k) {
    ja.p[k] = br[k].dsplit;
    ja.w[k] = br[k].out;
  }
  splitN_kernel<<<grid_for((int64_t)B * joint_w, 256), 256, 0, c->stream>>>(ja, djoint, B, joint_w);
  LAUNCH_CHECK(c);
  for (int k = 0; k < dd.nbr; ++k) {
    Branch& b = br[k];
    const float* cur = b.dsplit;  // the gradient of the current stage's output
    float *t0 = ga, *t1 = gb;     // ping-pong: a stage reads cur and writes the other buffer
    auto next = [&]() { return cur == t0 ? t1 : t0; };
    for (int j = (int)b.lin.size() - 1; j >= 0; --j) {
      Layer& l = b.lin[j];
      float* dz = next();
      FG_TRY(act_bwd(l.act, cur, dz, G, B));
      const bool first = j == 0 && b.conv.empty();
      float* din = first ? (want_dx ? b.dxb : nullptr) : (dz == t0 ? t1 : t0);
      FG_TRY(convl_bwd(e, l.L, l.in, dz, G, din, B));
      cur = din;
    }
    for (int i = (int)b.conv.size() - 1; i >= 0; --i) {
      Layer& l = b.conv[i];
      const Act& a = l.act;
      if (a.avg) {  // the average's adjoint: the gradient of the PReLU's full-size output
        float* dfull = next();
        avgpool2_bwd_kernel<<<grid_for((int64_t)B * a.H * a.W * a.C, 256), 256, 0, c->stream>>>(cur, dfull, B, a.H, a.W, a.C);
        LAUNCH_CHECK(c);
        cur = dfull;
      }
      float* dz = next();
      FG_TRY(act_bwd(a, cur, dz, G, B));
      if (l.stride == 2) {  // the adjoint of the subsample: zeros at the odd pixels
        const int H = l.L.H, Co = l.L.Cout;
        float* dzfull = dz == t0 ? t1 : t0;
        zero_insert2_kernel<<<grid_for((int64_t)B * H * H * Co, 256), 256, 0, c->stream>>>(dz, dzfull, B, H, H, Co);
        LAUNCH_CHECK(c);
        dz = dzfull;
      }
      float* din = i == 0 ? (want_dx ? b.dxb : nullptr) : (dz == t0 ? t1 : t0);
      FG_TRY(convl_bwd(e, l.L, l.in, dz, G, din, B));
      cur = din;
    }
  }
  if (want_dx)
    for (int k = 1; k < dd.nbr; ++k) FG_TRY(k_add(c, dx, br[k].dxb, dx, (int64_t)B * dd.side * dd.side * c->C));
  return FG_OK;
}
}  // namespace

int dbr_side(int disc) {
  const DbrDesc* d = find_desc(disc);
  return d ? d->side : 0;
}
int64_t dbr_param_count(int disc, int C) {
  const DbrDesc* d = find_desc(disc);
  return d ? DBr(*d).layout(C) : -1;
}
int dbr_mask_per_sample(int disc) {
  const DbrDesc* d = find_desc(disc);
  if (!d) return -1;
  DBr D(*d);
  D.layout(1);
  return D.mask;
}
std::unique_ptr<GanD> dbr_make(int disc) {
  const DbrDesc* d = find_desc(disc);
  if (!d) return nullptr;
  return std::make_unique<DBr>(*d);
}
