// ConvL / UpsL: layer-level dispatch shared by the nets (see convl.h)
#include "convl.h"

#include <utility>

#include "k_conv_tc.h"
#include "k_misc.h"

int convl_dalloc(ConvLEnv& e, float** p, size_t elems) { return fg_dalloc(e.c, *e.allocs, p, elems); }

int ScalePairs::alloc(fg_ctx* c, std::vector<void*>& allocs, int pairs) {
  n = pairs;
  used = 0;
  return fg_dalloc(c, allocs, &base, 2 * (size_t)pairs);
}
int ScalePairs::take(float** pair) {
  if (used == n) {
    fg_set_error("a block of %d FP16 scale pairs is full", n);
    return FG_ERR_UNSUPPORTED;
  }
  *pair = base + 2 * used++;
  return FG_OK;
}
int ScalePairs::reset(fg_ctx* c) const {
  if (!tc_f16(c)) return FG_OK;
  FG_CUDA(cudaMemset2DAsync(base, 2 * sizeof(float), 0, sizeof(float), n, c->stream));
  return FG_OK;
}

namespace {
// option "mma_f16": the hi/lo buffers of a layer hold the 3xFP16 split (halves, half of each buffer used), activations and
// gradients scaled into fp16's range by a device-side power of two (TcOp::s: (max|x|, 1/scale) pairs); the tensor
// path then needs 64-channel K blocks, so a layer with Cin % 64 != 0 stays on the 3xTF32 kernels.
inline bool tc_f(const fg_ctx* c, const ConvL& L, int B) { return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(L.geom_k(B)); }
inline bool tc_d(const fg_ctx* c, const ConvL& L, int B) { return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(L.geom_d(B)); }
inline bool tc_w(const fg_ctx* c, const ConvL& L, int B) { return tc_f(c, L, B) && L.Cout % 128 == 0 && L.geom_k(B).Cin % 64 == 0; }
}  // namespace

bool convl_tc_fwd(const fg_ctx* c, const ConvL& L) { return tc_f(c, L, 1); }
bool convl_tc_bwd(const fg_ctx* c, const ConvL& L) { return tc_f(c, L, 1) && tc_d(c, L, 1); }
bool convl_tc_wgrad(const fg_ctx* c, const ConvL& L) { return tc_w(c, L, 1); }

bool wgrad_async(const fg_ctx* c, const ConvLEnv& e) {
  return c->bwd_streams && e.ws_w && c->world == 1 && !c->timing && !c->debug_keep;
}

namespace {
void swap_wgrad(fg_ctx* c, ConvLEnv& e) {
  fg_ctx::WgradWorkspaces& w = c->wgrad_ws;
  std::swap(c->stream, c->wgrad_stream);
  std::swap(c->splitk_ws, w.splitk_ws);
  std::swap(c->red_ws, w.red_ws);
  std::swap(c->red_ticket, w.red_ticket);
  std::swap(c->small_ws, w.small_ws);
  std::swap(e.ws, e.ws_w);
}
int wgrad_fork(fg_ctx* c) {
  if (!c->wgrad_stream) FG_CUDA(cudaStreamCreateWithFlags(&c->wgrad_stream, cudaStreamNonBlocking));
  if (!c->ev_wfork) FG_CUDA(cudaEventCreateWithFlags(&c->ev_wfork, cudaEventDisableTiming));
  if (!c->ev_wjoin) FG_CUDA(cudaEventCreateWithFlags(&c->ev_wjoin, cudaEventDisableTiming));
  FG_CUDA(cudaEventRecord(c->ev_wfork, c->stream));
  FG_CUDA(cudaStreamWaitEvent(c->wgrad_stream, c->ev_wfork, 0));
  c->wgrad_forked = true;
  return FG_OK;
}
}  // namespace

OnWgradStream::OnWgradStream(ConvLEnv& e_, bool on_) : e(e_), on(on_) {
  if (!on) return;
  r = wgrad_fork(e.c);
  if (r != FG_OK) on = false;
  else swap_wgrad(e.c, e);
}
OnWgradStream::~OnWgradStream() {
  if (on) swap_wgrad(e.c, e);
}

int wgrad_join(ConvLEnv& e) {
  fg_ctx* c = e.c;
  if (!c->wgrad_forked) return FG_OK;
  c->wgrad_forked = false;
  FG_CUDA(cudaEventRecord(c->ev_wjoin, c->wgrad_stream));
  FG_CUDA(cudaStreamWaitEvent(c->stream, c->ev_wjoin, 0));
  return FG_OK;
}

int tc_op_split(fg_ctx* c, TcOp& op, const float* x, int64_t n, bool f16) {
  if (!f16) {
    if (op.split_ready) {
      op.split_ready = false;
      return FG_OK;
    }
    return tc_split(c, x, op.hi, op.lo, n);
  }
  if (op.amax_ready) op.amax_ready = false;
  else FG_TRY(tc_amax(c, x, n, op.s));
  return tc_split_h(c, x, op.hi, op.lo, n, op.s);
}

int convl_alloc(ConvLEnv& e, ConvL& L) {
  const size_t nw = (size_t)L.k * L.k * L.Cout * L.Cin;
  FG_TRY(convl_dalloc(e, &L.Wp, nw));
  FG_TRY(convl_dalloc(e, &L.Wpd, nw));
  if (L.nA) FG_TRY(convl_dalloc(e, &L.bp, L.Cout));
  if (!e.dy.s) FG_TRY(convl_dalloc(e, &e.dy.s, 2));
  const bool tc = tc_conv_eligible(L.geom_k(e.maxB));
  if (tc) {
    const size_t nk = (size_t)L.k * L.k * L.Cout * L.geom_k(e.maxB).Cin;
    FG_TRY(convl_dalloc(e, &L.Wf_hi, nk));
    FG_TRY(convl_dalloc(e, &L.Wf_lo, nk));
    if (L.kpad) FG_TRY(convl_dalloc(e, &L.Wpad, nk));  // zero-filled: the pad columns stay zero
  }
  if (L.need_dgrad && tc_conv_eligible(L.geom_d(e.maxB))) {
    FG_TRY(convl_dalloc(e, &L.Wd_hi, nw));
    FG_TRY(convl_dalloc(e, &L.Wd_lo, nw));
  }
  // padded tensor-core variants (see ConvL)
  const int B = e.maxB;
  if (L.pad_out && !(tc_conv_eligible(ConvGeom{B, L.H, L.H, L.Cin, L.pad_out, L.k, 1}) &&
                     tc_conv_eligible(ConvGeom{B, L.H, L.H, L.pad_out, L.Cin, L.k, 1}) && L.Cin % 128 == 0))
    L.pad_out = 0;
  if (L.pad_dy && !(tc && tc_conv_eligible(ConvGeom{B, L.H, L.H, L.Cin, L.pad_dy, L.k, 1}) && L.Cin % 64 == 0))
    L.pad_dy = 0;
  if (L.pad_out) {
    const size_t nq = (size_t)L.k * L.k * L.pad_out * L.Cin;
    FG_TRY(convl_dalloc(e, &L.Wq_hi, nq));  // zero-initialised: the padding rows stay zero
    FG_TRY(convl_dalloc(e, &L.Wq_lo, nq));
  }
  return convl_alloc_x(e, L);
}

int convl_alloc_x(ConvLEnv& e, ConvL& L) {
  if (!L.x.s) FG_TRY(convl_dalloc(e, &L.x.s, 2));
  const bool tc = tc_conv_eligible(L.geom_k(e.maxB));
  if (!tc && !L.pad_out) return FG_OK;
  // a pad_out layer (Cout <= 4) is never eligible itself: its split holds the Cin input channels
  const size_t nx = (size_t)e.maxB * L.H * L.H * L.geom_k(e.maxB).Cin;
  FG_TRY(convl_dalloc(e, &L.x.hi, nx));
  FG_TRY(convl_dalloc(e, &L.x.lo, nx));
  if (tc && L.kpad) FG_TRY(convl_dalloc(e, &L.xpad, nx));  // zero-filled: the pad columns stay zero
  return FG_OK;
}

int convl_pack(fg_ctx* c, ConvL& L, const float* P) {
  const int KK = L.k * L.k;
  const bool tc_on = c->conv_impl != FG_CONV_SIMT;
  const bool h = tc_on && tc_f16(c) && L.geom_k(1).Cin % 64 == 0 && (L.Cout % 64 == 0 || L.pad_out);
  L.packed_f16 = h;
  // a convolution without permutations that runs on the tensor cores both ways: pack and split in one kernel, no fp32 packs
  if (KK > 1 && tc_on && !L.nA && !L.cA && !L.pad_out && !L.kpad && L.Wf_hi && (L.Wd_hi || !L.need_dgrad) && tc_f(c, L, 1) &&
      (!L.need_dgrad || tc_d(c, L, 1))) {
    if (h) return tc_pack_split_h(c, P + L.w_off, L.Wf_hi, L.Wf_lo, L.Wd_hi, L.Wd_lo, L.Cout, L.Cin, KK);
    return tc_pack_split(c, P + L.w_off, L.Wf_hi, L.Wf_lo, L.Wd_hi, L.Wd_lo, L.Cout, L.Cin, KK);
  }
  FG_TRY(k_pack_weights(c, P + L.w_off, L.Wp, L.need_dgrad ? L.Wpd : nullptr, L.Cout, L.Cin, KK, L.nA, L.nS, L.cA, L.cS));
  if (L.bp) FG_TRY(k_pack_weights(c, P + L.b_off, L.bp, nullptr, L.Cout, 1, 1, L.nA, L.nS, 0, 0));
  if (!tc_on) return FG_OK;
  if (L.kpad && L.Wf_hi) {  // [Cout][Cin] -> [Cout][kpad], then the split
    FG_CUDA(cudaMemcpy2DAsync(L.Wpad, L.kpad * sizeof(float), L.Wp, L.Cin * sizeof(float), L.Cin * sizeof(float), L.Cout,
                              cudaMemcpyDeviceToDevice, c->stream));
    if (h) return tc_split_h(c, L.Wpad, L.Wf_hi, L.Wf_lo, (int64_t)L.Cout * L.kpad);
    return tc_split(c, L.Wpad, L.Wf_hi, L.Wf_lo, (int64_t)L.Cout * L.kpad);
  }
  const int64_t nw = (int64_t)KK * L.Cout * L.Cin;
  if (h) {
    if (L.Wf_hi) FG_TRY(tc_split_h(c, L.Wp, L.Wf_hi, L.Wf_lo, nw));
    if (L.Wd_hi) FG_TRY(tc_split_h(c, L.Wpd, L.Wd_hi, L.Wd_lo, nw));
    if (L.pad_out) FG_TRY(k_pack_pad_split_h(c, P + L.w_off, L.Wq_hi, L.Wq_lo, L.Cout, L.pad_out, L.Cin, KK));
    return FG_OK;
  }
  if (L.Wf_hi) FG_TRY(tc_split(c, L.Wp, L.Wf_hi, L.Wf_lo, nw));
  if (L.Wd_hi) FG_TRY(tc_split(c, L.Wpd, L.Wd_hi, L.Wd_lo, nw));
  if (L.pad_out) FG_TRY(k_pack_pad_split(c, P + L.w_off, L.Wq_hi, L.Wq_lo, L.Cout, L.pad_out, L.Cin, KK));
  return FG_OK;
}

int convl_fwd(ConvLEnv& e, ConvL& L, const float* in, const float* P, float* out, int B) {
  fg_ctx* c = e.c;
  const ConvGeom g = L.geom(B);
  const float* bias = L.bp ? L.bp : P + L.b_off;
  const bool h = L.packed_f16;  // the weight packs decide: they were built for one operand format
  const float* os = h ? L.x.s + 1 : nullptr;
  if (L.pad_out && c->conv_impl != FG_CONV_SIMT) {
    FG_TRY(tc_op_split(c, L.x, in, (int64_t)B * L.H * L.H * L.Cin, h));
    {
      ScopedTimer t(c, L.tf);
      FG_TRY(tc_conv_fwd(c, L.x.hi, L.x.lo, L.Wq_hi, L.Wq_lo, nullptr, e.ga, ConvGeom{B, L.H, L.H, L.Cin, L.pad_out, L.k, 1}, 0,
                         nullptr, nullptr, h, os));
    }
    return k_compact_bias(c, e.ga, bias, out, (int64_t)B * L.H * L.H, L.Cout, L.pad_out);
  }
  if (tc_f(c, L, B)) {
    const ConvGeom gk = L.geom_k(B);
    if (L.kpad) {
      FG_CUDA(cudaMemcpy2DAsync(L.xpad, L.kpad * sizeof(float), in, L.Cin * sizeof(float), L.Cin * sizeof(float), (size_t)B * L.H * L.H,
                                cudaMemcpyDeviceToDevice, c->stream));
      in = L.xpad;
    }
    FG_TRY(tc_op_split(c, L.x, in, (int64_t)B * L.H * L.H * gk.Cin, h));
    ScopedTimer t(c, L.tf);
    return tc_conv_fwd(c, L.x.hi, L.x.lo, L.Wf_hi, L.Wf_lo, bias, out, gk, 0, nullptr, nullptr, h, os);
  }
  ScopedTimer t(c, L.tf);
  if (c->edge_impl && k_edge_eligible(g)) return k_conv_edge(c, in, L.Wp, bias, out, g);
  return k_small_eligible(g) ? k_conv_small(c, in, L.Wp, bias, out, g) : k_conv_simt(c, in, L.Wp, bias, out, g);
}

int convl_bwd(ConvLEnv& e, ConvL& L, const float* in, const float* dy, float* G, float* din, int B, bool wgrad_side) {
  fg_ctx* c = e.c;
  const ConvGeom g = L.geom(B), gd = L.geom_d(B);
  const bool w_tc = G && tc_w(c, L, B), d_tc = din && tc_d(c, L, B);
  const bool h = L.packed_f16;
  // what the producer of dY already did (TcOp): consumed here
  float* sdy = L.sdy ? L.sdy : e.dy.s;
  float *dy_hi = L.dy_hi ? L.dy_hi : e.dy.hi, *dy_lo = L.dy_lo ? L.dy_lo : e.dy.lo;
  const bool split_ready = e.dy.split_ready, amax_ready = e.dy.amax_ready, bias_ready = e.dy.bias_ready;
  e.dy.split_ready = e.dy.amax_ready = e.dy.bias_ready = false;
  const float *osy = h ? sdy + 1 : nullptr, *osx = h ? L.x.s + 1 : nullptr;
  const bool tc_on = c->conv_impl != FG_CONV_SIMT;
  const int64_t P = (int64_t)B * L.H * L.H;
  if (h && !amax_ready && (w_tc || d_tc || (G && tc_on && (L.pad_out || L.pad_dy)))) FG_TRY(tc_amax(c, dy, P * L.Cout, sdy));
  if (w_tc || d_tc) {
    if (h) FG_TRY(tc_split_h(c, dy, dy_hi, dy_lo, P * L.Cout, sdy));
    else if (!split_ready) FG_TRY(tc_split(c, dy, dy_hi, dy_lo, P * L.Cout));
  }
  if (G && tc_on && L.pad_out) {
    // swapped roles: Gt[t'][c][n] = sum_p X[p][c] * dYpad[p + off(t')][n]  ==  dW[KK-1-t'][n][c]
    if (h) FG_TRY(k_pad_split_h(c, dy, e.pad.hi, e.pad.lo, P, L.Cout, L.pad_out, sdy));
    else FG_TRY(k_pad_split(c, dy, e.pad.hi, e.pad.lo, P, L.Cout, L.pad_out));
    {
      ScopedTimer t(c, L.tw);
      FG_TRY(tc_conv_wgrad(c, e.pad.hi, e.pad.lo, L.x.hi, L.x.lo, e.ws, ConvGeom{B, L.H, L.H, L.pad_out, L.Cin, L.k, 1}, h, osy, osx));
    }
    FG_TRY(k_unpack_wgrad_swapped(c, e.ws, G + L.w_off, L.Cout, L.pad_out, L.Cin, L.k * L.k));
    if (!bias_ready) FG_TRY(k_colsum_add(c, dy, G + L.b_off, P, L.Cout, 0, 0));
  } else if (G && tc_on && L.pad_dy && !w_tc) {
    if (h) FG_TRY(k_pad_split_h(c, dy, e.pad.hi, e.pad.lo, P, L.Cout, L.pad_dy, sdy));
    else FG_TRY(k_pad_split(c, dy, e.pad.hi, e.pad.lo, P, L.Cout, L.pad_dy));
    {
      ScopedTimer t(c, L.tw);
      FG_TRY(tc_conv_wgrad(c, L.x.hi, L.x.lo, e.pad.hi, e.pad.lo, e.ws, ConvGeom{B, L.H, L.H, L.Cin, L.pad_dy, L.k, 1}, h, osy, osx));
    }
    FG_TRY(k_unpack_wgrad_pad(c, e.ws, G + L.w_off, L.Cout, L.pad_dy, L.Cin, L.k * L.k));
    if (!bias_ready) FG_TRY(k_colsum_add(c, dy, G + L.b_off, P, L.Cout, 0, 0));
  } else if (G) {
    OnWgradStream side(e, wgrad_side);
    FG_TRY(side.r);
    // kpad: the [Cout][kpad] gradient lands behind the [Cout][Cin] one, whose pad columns are dropped by the copy
    const int64_t koff = L.kpad && w_tc ? (int64_t)L.Cout * L.Cin : 0;
    {
      ScopedTimer t(c, L.tw);
      if (w_tc) FG_TRY(tc_conv_wgrad(c, L.x.hi, L.x.lo, dy_hi, dy_lo, e.ws + koff, L.geom_k(B), h, osy, osx));
      else if (k_small_eligible(g)) FG_TRY(k_wgrad_small(c, in, dy, e.ws, g));
      else FG_TRY(k_wgrad_simt(c, in, dy, e.ws, g));
    }
    if (koff)
      FG_CUDA(cudaMemcpy2DAsync(e.ws, L.Cin * sizeof(float), e.ws + koff, L.kpad * sizeof(float), L.Cin * sizeof(float), L.Cout,
                                cudaMemcpyDeviceToDevice, c->stream));
    FG_TRY(k_unpack_wgrad(c, e.ws, G + L.w_off, L.Cout, L.Cin, L.k * L.k, L.nA, L.nS, L.cA, L.cS));
    if (!bias_ready) FG_TRY(k_colsum_add(c, dy, G + L.b_off, P, L.Cout, L.nA, L.nS));
  }
  if (din) {
    ScopedTimer t(c, L.td);
    if (d_tc) return tc_conv_fwd(c, dy_hi, dy_lo, L.Wd_hi, L.Wd_lo, nullptr, din, gd, 0, nullptr, nullptr, h, osy);
    if (c->edge_impl && k_edge_eligible(gd)) return k_conv_edge(c, dy, L.Wpd, nullptr, din, gd);
    return k_small_eligible(gd) ? k_conv_small(c, dy, L.Wpd, nullptr, din, gd) : k_conv_simt(c, dy, L.Wpd, nullptr, din, gd);
  }
  return FG_OK;
}

bool upsl_tc(const fg_ctx* c, const UpsL& U) {
  return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(U.geom(1)) && U.Cout % 128 == 0 && U.Cin % 64 == 0;
}

int upsl_alloc(ConvLEnv& e, UpsL& U) {
  const size_t nw25 = (size_t)25 * U.Cout * U.Cin, nw36 = (size_t)36 * U.Cout * U.Cin;
  FG_TRY(convl_dalloc(e, &U.Wp, nw25));
  FG_TRY(convl_dalloc(e, &U.Wpd, nw25));
  FG_TRY(convl_dalloc(e, &U.Wf_hi, nw36));
  FG_TRY(convl_dalloc(e, &U.Wf_lo, nw36));
  FG_TRY(convl_dalloc(e, &U.Wd_hi, nw36));
  FG_TRY(convl_dalloc(e, &U.Wd_lo, nw36));
  FG_TRY(convl_dalloc(e, &U.Wx_hi, nw25));
  FG_TRY(convl_dalloc(e, &U.Wx_lo, nw25));
  return upsl_alloc_x(e, U);
}

int upsl_alloc_x(ConvLEnv& e, UpsL& U) {
  const size_t nx = (size_t)e.maxB * (U.H / 2) * (U.H / 2) * U.Cin;
  FG_TRY(convl_dalloc(e, &U.x.hi, nx));
  FG_TRY(convl_dalloc(e, &U.x.lo, nx));
  if (!U.x.s) FG_TRY(convl_dalloc(e, &U.x.s, 2));
  return FG_OK;
}

int upsl_pack(fg_ctx* c, UpsL& U, const float* P) {
  const float* W = P + U.w_off;
  if (!upsl_tc(c, U)) return k_pack_weights(c, W, U.Wp, U.Wpd, U.Cout, U.Cin, 25, 0, 0, 0, 0);
  if (tc_f16(c)) FG_TRY(tc_pack_collapsed_h(c, W, U.Wf_hi, U.Wf_lo, U.Wd_hi, U.Wd_lo, U.Cout, U.Cin));
  else FG_TRY(tc_pack_collapsed(c, W, U.Wf_hi, U.Wf_lo, U.Wd_hi, U.Wd_lo, U.Cout, U.Cin));
  // conv_impl 1 runs the forward on the dense 25-tap pack; the backward always uses the collapsed dgrad pack
  if (c->conv_impl == FG_CONV_TC_DENSE) FG_TRY(tc_pack_split(c, W, U.Wx_hi, U.Wx_lo, nullptr, nullptr, U.Cout, U.Cin, 25));
  return FG_OK;
}

int upsl_fwd(ConvLEnv& e, UpsL& U, const float* h, const float* P, float* z, int B, int* parts) {
  fg_ctx* c = e.c;
  const ConvGeom g = U.geom(B);
  const bool want = parts && *parts;
  if (parts) *parts = 0;
  const float* bias = P + U.b_off;
  if (!upsl_tc(c, U)) {
    ScopedTimer t(c, U.tf);
    return k_conv_simt(c, h, U.Wp, bias, z, g);
  }
  const bool f16 = tc_f16(c);
  FG_TRY(tc_op_split(c, U.x, h, (int64_t)B * (U.H / 2) * (U.H / 2) * U.Cin, f16));  // kept for the weight gradient
  ScopedTimer t(c, U.tf);
  float* st = want && c->bn_epilogue ? c->bn_parts : nullptr;
  const bool dense = c->conv_impl == FG_CONV_TC_DENSE;
  return tc_conv_fwd(c, U.x.hi, U.x.lo, dense ? U.Wx_hi : U.Wf_hi, dense ? U.Wx_lo : U.Wf_lo, bias, z, g, dense ? 1 : 2, st,
                     st ? parts : nullptr, f16, f16 ? U.x.s + 1 : nullptr);
}

int upsl_bwd(ConvLEnv& e, UpsL& U, TcOp& dy, const float* h, const float* dz, float* G, float* dh, int B, bool* pooled,
             bool wgrad_side) {
  fg_ctx* c = e.c;
  const ConvGeom g = U.geom(B);
  float* dW = G + U.w_off;
  *pooled = upsl_tc(c, U);
  if (!*pooled) {
    {
      ScopedTimer t(c, U.tw);
      FG_TRY(k_wgrad_simt(c, h, dz, e.ws, g));
    }
    FG_TRY(k_unpack_wgrad(c, e.ws, dW, U.Cout, U.Cin, 25, 0, 0, 0, 0));
    ScopedTimer t(c, U.td);
    return k_conv_simt(c, dz, U.Wpd, nullptr, dh, ConvGeom{B, U.H, U.H, U.Cout, U.Cin, 5, 1});
  }
  const bool f16 = tc_f16(c);
  FG_TRY(tc_op_split(c, dy, dz, (int64_t)B * U.H * U.H * U.Cout, f16));
  const float *sy = f16 ? dy.s + 1 : nullptr, *sx = f16 ? U.x.s + 1 : nullptr;
  // 3xFP16 with option bwd_merge: wgrad and dgrad as ONE persistent launch (the dgrad tiles fill the SMs a narrow weight
  // gradient leaves idle; same bits as two launches)
  if (f16 && U.tb && (c->bwd_merge == 2 ? tc_bwd_pair_eligible(c, g) : c->bwd_merge == 1 && tc_bwd_pair_pays(c, g))) {
    {
      ScopedTimer t(c, U.tb);
      FG_TRY(tc_conv_bwd_ups(c, U.x.hi, U.x.lo, dy.hi, dy.lo, U.Wd_hi, U.Wd_lo, e.ws, dh, g, sy, sx));
    }
    return tc_combine_collapsed_wgrad(c, e.ws, dW, U.Cout, U.Cin);
  }
  {
    // wgrad_side: the weight gradient and its combine on the wgrad stream, beside the data gradient (G.C1's 72 CTAs
    // leave 60 SMs to the data-gradient tiles)
    OnWgradStream side(e, wgrad_side);
    FG_TRY(side.r);
    {
      ScopedTimer t(c, U.tw);
      FG_TRY(tc_conv_wgrad(c, U.x.hi, U.x.lo, dy.hi, dy.lo, e.ws, g, f16, sy, sx));
    }
    FG_TRY(tc_combine_collapsed_wgrad(c, e.ws, dW, U.Cout, U.Cin));
  }
  ScopedTimer t(c, U.td);
  return tc_conv_dgrad_ups(c, dy.hi, dy.lo, U.Wd_hi, U.Wd_lo, dh, g, f16, sy);
}
