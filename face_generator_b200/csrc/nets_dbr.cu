// The branched discriminators of models.lua that create_D does not pick: create_D32 (:322-376) at 32x32 and
// create_D16 (:110-159), create_D16_b (:161-216), create_D16_c (:218-277) at 16x16.  Each is
//   ConcatTable{fine conv branch (3x3), coarse conv branch (5x5), dense branch} -> JoinTable(2) -> Linear -> PReLU
//   -> Dropout -> Linear(1) -> Sigmoid
// and differs from the others only in data: one descriptor (DbrDesc) per net, one GanD type (DBr) built from it.
//   conv branch : conv (PReLU) [MaxPool(2,2)] ... SpatialDropout View Linear PReLU [Dropout] [Linear PReLU]
//   dense branch: View(C*S*S) Linear(.., 1024) PReLU Dropout Linear(1024, 1024) PReLU
// Every convolution and Linear is a ConvL (convl.h) through the shared dispatch; a stride-2 convolution runs at stride 1
// and is subsampled, as D16_d does (nets_s16.cu).  The elementwise stages are one kernel pair: PReLU -> optional 2x2
// max pooling -> optional (spatial) dropout forward, writing the window's arg-max, and its backward, which reduces
// the PReLU slope gradient in a fixed order (k_ordered.cuh), so a step stays bit-reproducible.
#include <deque>
#include <string>

#include "fg_internal.h"
#include "k_misc.h"
#include "k_ordered.cuh"
#include "ups_gan.h"

namespace {
constexpr float kP = 0.5f;  // nn.SpatialDropout() / nn.Dropout() default probability

// ---- descriptor --------------------------------------------------------------------------------------------------
struct DbrConvDesc {
  int cout, k, stride;
  bool pool;  // nn.SpatialMaxPooling(2, 2) after the PReLU
};
struct DbrLinDesc {
  int out;
  bool drop;  // nn.Dropout() after the PReLU
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
  int disc, side;
  DbrBranchDesc br[3];  // ConcatTable order
  DbrLinDesc head;      // Linear(joint, head.out) PReLU Dropout; then Linear(head.out, 1)
};

constexpr DbrBranchDesc kDense = {"dense", 0, {}, 2, {{1024, true}, {1024, false}}};
const DbrDesc kDescs[] = {
    {FG_DISC_D32, 32,
     {{"fine", 2, {{64, 3, 1, false}, {64, 3, 1, true}}, 1, {{1024, false}}},
      {"coarse", 4, {{32, 5, 1, false}, {32, 5, 1, true}, {54, 5, 1, false}, {54, 5, 1, true}}, 2, {{1024, true}, {1024, false}}},
      kDense},
     {1024, true}},
    {FG_DISC_D16, 16,
     {{"fine", 2, {{64, 3, 1, false}, {64, 3, 1, true}}, 1, {{1024, true}}},
      {"coarse", 2, {{32, 5, 1, false}, {64, 5, 1, true}}, 1, {{1024, true}}},
      kDense},
     {1024, true}},
    {FG_DISC_D16_B, 16,
     {{"fine", 4, {{64, 3, 1, false}, {64, 3, 1, false}, {128, 3, 1, false}, {128, 3, 2, false}}, 1, {{512, true}}},
      {"coarse", 4, {{64, 5, 1, false}, {64, 5, 1, false}, {128, 5, 1, false}, {128, 5, 2, false}}, 1, {{512, true}}},
      kDense},
     {1024, true}},
    {FG_DISC_D16_C, 16,
     {{"fine", 5, {{64, 3, 1, false}, {64, 3, 1, false}, {128, 3, 1, false}, {128, 3, 2, false}, {512, 3, 2, false}}, 1,
       {{1024, false}}},
      {"coarse", 5, {{64, 5, 1, false}, {64, 5, 1, false}, {128, 5, 1, false}, {128, 5, 2, false}, {512, 5, 2, false}}, 1,
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
  s = block_sum256(s);
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *dslope += (float)ordered_sum(ws, gridDim.x, 1, 0);
    ordered_release(ticket);
  }
}

// nn.JoinTable(2) of up to kMaxJoin inputs [B][w_k] -> [B][sum w_k], and the split of its gradient
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
// one PReLU [-> MaxPool(2,2)] [-> (spatial) dropout] stage on a [B][H][W][C] pre-activation z
struct Act {
  int64_t a_off = 0;  // slope
  int H = 1, W = 1, C = 0, pool = 1;
  int moff = -1;  // keep-flag offset in the sample's row; -1: no dropout
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
  Layer head;
  int64_t JW = 0, Jb = 0;  // the last Linear(head.out, 1)
  int joint_w = 0;
  float *zfull = nullptr, *joint = nullptr, *djoint = nullptr, *ga = nullptr, *gb = nullptr;
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
    for (Branch& b : br) {
      for (Layer& l : b.conv) v.push_back(&l);
      for (Layer& l : b.lin) v.push_back(&l);
    }
    v.push_back(&head);
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
  auto linear = [&](Layer& l, const char* pre, int j, int cin, int cout, int cA, int cS) {
    ConvL& L = l.L;
    L.Cin = cin; L.Cout = cout; L.k = 1; L.H = 1;
    L.cA = cA; L.cS = cS;  // View flattens [C][H][W]; ours is [H][W][C]
    L.w_off = o; o += (int64_t)cout * cin;
    L.b_off = o; o += cout;
    l.act.a_off = o; o += 1;
    l.act.C = cout;
    L.tf = name(std::string(pre) + ".L" + std::to_string(j + 1) + ".fwd");
    L.td = name(std::string(pre) + ".L" + std::to_string(j + 1) + ".dgrad");
    L.tw = name(std::string(pre) + ".L" + std::to_string(j + 1) + ".wgrad");
  };
  auto dropout = [&](Act& a, int width) {
    a.moff = m;
    m += width;
  };
  joint_w = 0;
  for (int k = 0; k < 3; ++k) {
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
      L.tf = name(pre + ".c" + std::to_string(i + 1) + ".fwd");
      L.td = name(pre + ".c" + std::to_string(i + 1) + ".dgrad");
      L.tw = name(pre + ".c" + std::to_string(i + 1) + ".wgrad");
      l.stride = cd.stride;
      s /= cd.stride;
      l.act.H = l.act.W = s;
      l.act.C = cd.cout;
      l.act.pool = cd.pool ? 2 : 1;
      s /= l.act.pool;
      cin = cd.cout;
    }
    if (bd.nconv) {  // nn.SpatialDropout(): one flag per plane, no rescale in training, 1-p in evaluation
      Act& a = b.conv.back().act;
      dropout(a, cin);
      a.eval_scale = 1.f - kP;
    }
    for (int j = 0; j < bd.nlin; ++j) {
      const int in = j ? bd.lin[j - 1].out : cin * s * s;
      linear(b.lin[j], pre.c_str(), j, in, bd.lin[j].out, j ? 0 : cin, j ? 0 : s * s);
      if (bd.lin[j].drop) {  // nn.Dropout(): 1/(1-p) in training, identity in evaluation
        dropout(b.lin[j].act, bd.lin[j].out);
        b.lin[j].act.train_scale = 1.f / (1.f - kP);
      }
    }
    b.out = bd.lin[bd.nlin - 1].out;
    joint_w += b.out;
  }
  head = Layer{};
  linear(head, "D.head", 0, joint_w, dd.head.out, 0, 0);
  if (dd.head.drop) {
    dropout(head.act, dd.head.out);
    head.act.train_scale = 1.f / (1.f - kP);
  }
  JW = o; o += dd.head.out;
  Jb = o; o += 1;
  mask = m;
  return o;
}

int DBr::alloc() {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  const size_t B = e.maxB, C = c->C, S = dd.side;
  // the scratch both nets share: the largest dY split and weight gradient of either net (G's needs from the trainer)
  size_t dy = n->g_dy, ws = n->g_ws, g = B * S * S * C, full = 0;
  for (Layer* l : layers()) {
    ConvL& L = l->L;
    const size_t P = B * L.H * L.H;
    dy = std::max(dy, P * L.Cout);
    ws = std::max(ws, (size_t)L.k * L.k * L.Cout * L.Cin);
    g = std::max(g, std::max(P * L.Cout, P * L.Cin));
    if (l->stride == 2) full = std::max(full, P * L.Cout);
    FG_TRY(convl_alloc(e, L));
  }
  FG_TRY(dalloc(&e.ws, ws));
  FG_TRY(dalloc(&e.dy.hi, dy));
  FG_TRY(dalloc(&e.dy.lo, dy));
  FG_TRY(dalloc(&ga, g));
  FG_TRY(dalloc(&gb, g));
  if (full) FG_TRY(dalloc(&zfull, full));
  FG_TRY(dalloc(&x, B * S * S * C));
  FG_TRY(dalloc(&dx, B * S * S * C));
  rows.clear();
  n->net.keep.clear();
  for (int k = 0; k < 3; ++k) {
    Branch& b = br[k];
    const std::string pre = std::string("D.") + dd.br[k].name;
    const float* in = x;
    for (size_t i = 0; i < b.conv.size(); ++i) {
      Layer& l = b.conv[i];
      Act& a = l.act;
      const int64_t zper = (int64_t)a.H * a.W * a.C;
      l.in = in;
      FG_TRY(dalloc(&a.z, B * zper));
      FG_TRY(dalloc(&a.h, B * a.out_per()));
      if (a.pool == 2) {
        float* q;
        FG_TRY(dalloc(&q, (B * a.out_per() + 3) / 4));
        a.code = reinterpret_cast<uint8_t*>(q);
      }
      const std::string zn = pre + ".z" + std::to_string(i + 1);
      rows.push_back({name(zn), a.z, zper, 0});
      rows.push_back({name(pre + ".h" + std::to_string(i + 1)), a.h, a.out_per(), 0});
      n->net.keep.push_back({name("Dstep." + zn.substr(2)), a.z, zper});
      in = a.h;
    }
    for (size_t j = 0; j < b.lin.size(); ++j) {
      Layer& l = b.lin[j];
      l.in = in;
      FG_TRY(dalloc(&l.act.z, B * l.act.C));
      FG_TRY(dalloc(&l.act.h, B * l.act.C));
      const std::string zn = pre + ".zl" + std::to_string(j + 1);
      rows.push_back({name(zn), l.act.z, l.act.C, 0});
      n->net.keep.push_back({name("Dstep." + zn.substr(2)), l.act.z, l.act.C});
      in = l.act.h;
    }
    FG_TRY(dalloc(&b.dsplit, B * b.out));
    if (k) FG_TRY(dalloc(&b.dxb, B * S * S * C));
  }
  br[0].dxb = dx;
  FG_TRY(dalloc(&joint, B * joint_w));
  FG_TRY(dalloc(&djoint, B * joint_w));
  head.in = joint;
  FG_TRY(dalloc(&head.act.z, B * head.act.C));
  FG_TRY(dalloc(&head.act.h, B * head.act.C));
  FG_TRY(dalloc(&logit, B));
  FG_TRY(dalloc(&out, B));
  FG_TRY(dalloc(&dlogit, B));
  FG_TRY(dalloc(&masks, B * mask));
  rows.insert(rows.end(), {{"D.joint", joint, joint_w, 0}, {"D.head.z", head.act.z, head.act.C, 0},
                           {"D.logit", logit, 1, 0}, {"D.out", out, 1, 0}, {"D.masks", masks, mask, 0},
                           {"D.dx", dx, (int64_t)(S * S * C), 0}});
  n->net.keep.insert(n->net.keep.end(), {{"Dstep.head.z", head.act.z, head.act.C}, {"Dstep.logit", logit, 1},
                                         {"Dstep.out", out, 1}});
  return FG_OK;
}

int DBr::act_fwd(const Act& A, int Bn, bool training) {
  fg_ctx* c = n->c;
  const float* keep = training && A.moff >= 0 ? masks : nullptr;
  const float es = training ? 1.f : A.eval_scale;
  const float* P = n->net.PD;
  const int64_t nout = (int64_t)Bn * A.out_per();
  if (A.pool == 2)
    dbr_act_fwd_kernel<2><<<grid_for(nout, 256), 256, 0, c->stream>>>(A.z, P + A.a_off, keep, mask, A.moff, A.train_scale,
                                                                       es, A.h, A.code, Bn, A.H, A.W, A.C);
  else
    dbr_act_fwd_kernel<1><<<grid_for(nout, 256), 256, 0, c->stream>>>(A.z, P + A.a_off, keep, mask, A.moff, A.train_scale,
                                                                       es, A.h, nullptr, Bn, A.H, A.W, A.C);
  LAUNCH_CHECK(c);
  return FG_OK;
}

int DBr::act_bwd(const Act& A, const float* dy, float* dz, float* G, int Bn) {
  fg_ctx* c = n->c;
  const float* keep = train && A.moff >= 0 ? masks : nullptr;
  const float es = train ? 1.f : A.eval_scale;
  const float* P = n->net.PD;
  float* ds = G ? G + A.a_off : nullptr;
  const int64_t nout = (int64_t)Bn * A.out_per();
  const int grid = grid_for(nout, 256, 132 * 8);
  FG_TRY(red_check(c, grid, 1));
  if (A.pool == 2)
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
  const float* P = n->net.PD;
  if (n->net.D_pack != pack_key(c)) {
    for (Layer* l : layers()) FG_TRY(convl_pack(c, l->L, P));
    n->net.D_pack = pack_key(c);
  }
  const int S = dd.side;
  if (xin != x) FG_CUDA(cudaMemcpyAsync(x, xin, sizeof(float) * (size_t)Bn * S * S * c->C, cudaMemcpyDeviceToDevice, c->stream));
  JoinArgs ja{};
  for (int k = 0; k < 3; ++k) {
    Branch& b = br[k];
    for (Layer& l : b.conv) {
      if (l.stride == 2) {  // stride 1, then every other pixel
        FG_TRY(convl_fwd(e, l.L, l.in, P, zfull, Bn));
        FG_TRY(k_subsample2(c, zfull, l.act.z, Bn, l.L.H, l.L.H, l.L.Cout));
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
  FG_TRY(convl_fwd(e, head.L, joint, P, head.act.z, Bn));
  FG_TRY(act_fwd(head.act, Bn, training));
  FG_TRY(k_gemv_fwd(c, head.act.h, P + JW, P + Jb, logit, Bn, head.act.C));
  B = Bn;
  train = training;
  valid = true;
  return FG_OK;
}

// want_dx: the image gradient is the sum of the three branches' (nn.ConcatTable backward), in branch order
int DBr::backward(bool want_wgrad, bool want_dx) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  if (!valid) {
    fg_set_error("D backward needs a preceding D forward");
    return FG_ERR_STATE;
  }
  const float* P = n->net.PD;
  float* G = want_wgrad ? n->net.gD : nullptr;
  const int hw = head.act.C;
  if (G) FG_TRY(k_gemv_wgrad_add(c, head.act.h, dlogit, G + JW, G + Jb, B, hw));
  FG_TRY(k_gemv_dgrad(c, dlogit, P + JW, ga, B, hw));
  FG_TRY(act_bwd(head.act, ga, gb, G, B));
  FG_TRY(convl_bwd(e, head.L, joint, gb, G, djoint, B));
  JoinArgs ja{};
  for (int k = 0; k < 3; ++k) {
    ja.p[k] = br[k].dsplit;
    ja.w[k] = br[k].out;
  }
  splitN_kernel<<<grid_for((int64_t)B * joint_w, 256), 256, 0, c->stream>>>(ja, djoint, B, joint_w);
  LAUNCH_CHECK(c);
  for (int k = 0; k < 3; ++k) {
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
      float* dz = next();
      FG_TRY(act_bwd(l.act, cur, dz, G, B));
      if (l.stride == 2) {  // the adjoint of the subsample: zeros at the odd pixels
        float* full = dz == t0 ? t1 : t0;
        FG_TRY(k_zero_insert2(c, dz, full, B, l.L.H, l.L.H, l.L.Cout));
        dz = full;
      }
      float* din = i == 0 ? (want_dx ? b.dxb : nullptr) : (dz == t0 ? t1 : t0);
      FG_TRY(convl_bwd(e, l.L, l.in, dz, G, din, B));
      cur = din;
    }
  }
  if (want_dx) {
    const int64_t nx = (int64_t)B * dd.side * dd.side * c->C;
    FG_TRY(k_add(c, dx, br[1].dxb, dx, nx));
    FG_TRY(k_add(c, dx, br[2].dxb, dx, nx));
  }
  return FG_OK;
}
}  // namespace

int dbr_side(int disc) {
  const DbrDesc* d = find_desc(disc);
  return d ? d->side : 0;
}
int64_t dbr_param_count(int disc, int C) {
  const DbrDesc* d = find_desc(disc);
  if (!d || (C != 1 && C != 3)) return -1;
  return DBr(*d).layout(C);
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
