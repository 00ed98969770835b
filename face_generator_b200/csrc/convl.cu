// ConvL: layer-level dispatch shared by nets_c2f.cu and nets_s16.cu (see convl.h)
#include "convl.h"

#include "k_conv_tc.h"
#include "k_misc.h"

int convl_dalloc(ConvLEnv& e, float** p, size_t elems) { return fg_dalloc(e.c, *e.allocs, p, elems); }

namespace {
// option "mma_f16": the hi/lo buffers of a layer hold the 3xFP16 split (halves, half of each buffer used), activations and
// gradients scaled into fp16's range by a device-side power of two (L.sx / env.sdy: (max|x|, 1/scale) pairs); the tensor
// path then needs 64-channel K blocks, so a layer with Cin % 64 != 0 stays on the 3xTF32 kernels.
inline bool f16_on(const fg_ctx* c) { return c->mma_f16 && c->conv_impl == FG_CONV_TC_COLLAPSED; }
inline bool tc_f(const fg_ctx* c, const ConvL& L, int B) { return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(L.geom(B)); }
inline bool tc_d(const fg_ctx* c, const ConvL& L, int B) { return c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(L.geom_d(B)); }
inline bool tc_w(const fg_ctx* c, const ConvL& L, int B) { return tc_f(c, L, B) && L.Cout % 128 == 0 && L.Cin % 64 == 0; }
int split_x(ConvLEnv& e, ConvL& L, const float* in, int64_t n, bool f16) {
  if (!f16) return tc_split(e.c, in, L.x_hi, L.x_lo, n);
  FG_TRY(tc_amax(e.c, in, n, L.sx));
  return tc_split_h(e.c, in, L.x_hi, L.x_lo, n, L.sx);
}
}  // namespace

int convl_alloc(ConvLEnv& e, ConvL& L) {
  const size_t nw = (size_t)L.k * L.k * L.Cout * L.Cin;
  FG_TRY(convl_dalloc(e, &L.Wp, nw));
  FG_TRY(convl_dalloc(e, &L.Wpd, nw));
  if (L.nA) FG_TRY(convl_dalloc(e, &L.bp, L.Cout));
  FG_TRY(convl_dalloc(e, &L.sx, 2));
  if (!e.sdy) FG_TRY(convl_dalloc(e, &e.sdy, 2));
  if (tc_conv_eligible(L.geom(e.maxB))) {
    FG_TRY(convl_dalloc(e, &L.Wf_hi, nw));
    FG_TRY(convl_dalloc(e, &L.Wf_lo, nw));
    const size_t nx = (size_t)e.maxB * L.H * L.H * L.Cin;
    FG_TRY(convl_dalloc(e, &L.x_hi, nx));
    FG_TRY(convl_dalloc(e, &L.x_lo, nx));
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
  if (L.pad_dy && !(L.x_hi && tc_conv_eligible(ConvGeom{B, L.H, L.H, L.Cin, L.pad_dy, L.k, 1}) && L.Cin % 64 == 0))
    L.pad_dy = 0;
  if (L.pad_out) {
    const size_t nq = (size_t)L.k * L.k * L.pad_out * L.Cin;
    FG_TRY(convl_dalloc(e, &L.Wq_hi, nq));  // zero-initialised: the padding rows stay zero
    FG_TRY(convl_dalloc(e, &L.Wq_lo, nq));
    const size_t nx = (size_t)B * L.H * L.H * L.Cin;
    FG_TRY(convl_dalloc(e, &L.x_hi, nx));
    FG_TRY(convl_dalloc(e, &L.x_lo, nx));
  }
  return FG_OK;
}

int convl_pack(fg_ctx* c, ConvL& L, const float* P) {
  const int KK = L.k * L.k;
  FG_TRY(k_pack_weights(c, P + L.w_off, L.Wp, L.need_dgrad ? L.Wpd : nullptr, L.Cout, L.Cin, KK, L.nA, L.nS, L.cA, L.cS));
  if (L.bp) FG_TRY(k_pack_weights(c, P + L.b_off, L.bp, nullptr, L.Cout, 1, 1, L.nA, L.nS, 0, 0));
  if (c->conv_impl == FG_CONV_SIMT) return FG_OK;
  const int64_t nw = (int64_t)KK * L.Cout * L.Cin;
  const bool h = f16_on(c) && L.Cin % 64 == 0 && (L.Cout % 64 == 0 || L.pad_out);
  L.packed_f16 = h;
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
  const float* os = h ? L.sx + 1 : nullptr;
  if (L.pad_out && c->conv_impl != FG_CONV_SIMT) {
    FG_TRY(split_x(e, L, in, (int64_t)B * L.H * L.H * L.Cin, h));
    {
      ScopedTimer t(c, L.tf);
      FG_TRY(tc_conv_fwd(c, L.x_hi, L.x_lo, L.Wq_hi, L.Wq_lo, nullptr, e.ga, ConvGeom{B, L.H, L.H, L.Cin, L.pad_out, L.k, 1}, 0,
                         nullptr, nullptr, h, os));
    }
    return k_compact_bias(c, e.ga, bias, out, (int64_t)B * L.H * L.H, L.Cout, L.pad_out);
  }
  if (tc_f(c, L, B)) {
    FG_TRY(split_x(e, L, in, (int64_t)B * L.H * L.H * L.Cin, h));
    ScopedTimer t(c, L.tf);
    return tc_conv_fwd(c, L.x_hi, L.x_lo, L.Wf_hi, L.Wf_lo, bias, out, g, 0, nullptr, nullptr, h, os);
  }
  ScopedTimer t(c, L.tf);
  if (c->edge_impl && k_edge_eligible(g)) return k_conv_edge(c, in, L.Wp, bias, out, g);
  return k_small_eligible(g) ? k_conv_small(c, in, L.Wp, bias, out, g) : k_conv_simt(c, in, L.Wp, bias, out, g);
}

int convl_bwd(ConvLEnv& e, ConvL& L, const float* in, const float* dy, float* G, float* din, int B) {
  fg_ctx* c = e.c;
  const ConvGeom g = L.geom(B), gd = L.geom_d(B);
  const bool w_tc = G && tc_w(c, L, B), d_tc = din && tc_d(c, L, B);
  const bool h = L.packed_f16;
  const float *osy = h ? e.sdy + 1 : nullptr, *osx = h ? L.sx + 1 : nullptr;
  const bool tc_on = c->conv_impl != FG_CONV_SIMT;
  const int64_t P = (int64_t)B * L.H * L.H;
  if (h && (w_tc || d_tc || (G && tc_on && (L.pad_out || L.pad_dy)))) FG_TRY(tc_amax(c, dy, P * L.Cout, e.sdy));
  if (w_tc || d_tc) {
    if (h) FG_TRY(tc_split_h(c, dy, e.dy_hi, e.dy_lo, P * L.Cout, e.sdy));
    else FG_TRY(tc_split(c, dy, e.dy_hi, e.dy_lo, P * L.Cout));
  }
  if (G && tc_on && L.pad_out) {
    // swapped roles: Gt[t'][c][n] = sum_p X[p][c] * dYpad[p + off(t')][n]  ==  dW[KK-1-t'][n][c]
    if (h) FG_TRY(k_pad_split_h(c, dy, e.pad_hi, e.pad_lo, P, L.Cout, L.pad_out, e.sdy));
    else FG_TRY(k_pad_split(c, dy, e.pad_hi, e.pad_lo, P, L.Cout, L.pad_out));
    {
      ScopedTimer t(c, L.tw);
      FG_TRY(tc_conv_wgrad(c, e.pad_hi, e.pad_lo, L.x_hi, L.x_lo, e.ws, ConvGeom{B, L.H, L.H, L.pad_out, L.Cin, L.k, 1}, h, osy, osx));
    }
    FG_TRY(k_unpack_wgrad_swapped(c, e.ws, G + L.w_off, L.Cout, L.pad_out, L.Cin, L.k * L.k));
    FG_TRY(k_colsum_add(c, dy, G + L.b_off, P, L.Cout, 0, 0));
  } else if (G && tc_on && L.pad_dy && !w_tc) {
    if (h) FG_TRY(k_pad_split_h(c, dy, e.pad_hi, e.pad_lo, P, L.Cout, L.pad_dy, e.sdy));
    else FG_TRY(k_pad_split(c, dy, e.pad_hi, e.pad_lo, P, L.Cout, L.pad_dy));
    {
      ScopedTimer t(c, L.tw);
      FG_TRY(tc_conv_wgrad(c, L.x_hi, L.x_lo, e.pad_hi, e.pad_lo, e.ws, ConvGeom{B, L.H, L.H, L.Cin, L.pad_dy, L.k, 1}, h, osy, osx));
    }
    FG_TRY(k_unpack_wgrad_pad(c, e.ws, G + L.w_off, L.Cout, L.pad_dy, L.Cin, L.k * L.k));
    FG_TRY(k_colsum_add(c, dy, G + L.b_off, P, L.Cout, 0, 0));
  } else if (G) {
    {
      ScopedTimer t(c, L.tw);
      if (w_tc) FG_TRY(tc_conv_wgrad(c, L.x_hi, L.x_lo, e.dy_hi, e.dy_lo, e.ws, g, h, osy, osx));
      else if (k_small_eligible(g)) FG_TRY(k_wgrad_small(c, in, dy, e.ws, g));
      else FG_TRY(k_wgrad_simt(c, in, dy, e.ws, g));
    }
    FG_TRY(k_unpack_wgrad(c, e.ws, G + L.w_off, L.Cout, L.Cin, L.k * L.k, L.nA, L.nS, L.cA, L.cS));
    FG_TRY(k_colsum_add(c, dy, G + L.b_off, P, L.Cout, L.nA, L.nS));
  }
  if (din) {
    ScopedTimer t(c, L.td);
    if (d_tc) return tc_conv_fwd(c, e.dy_hi, e.dy_lo, L.Wd_hi, L.Wd_lo, nullptr, din, gd, 0, nullptr, nullptr, h, osy);
    if (c->edge_impl && k_edge_eligible(gd)) return k_conv_edge(c, dy, L.Wpd, nullptr, din, gd);
    return k_small_eligible(gd) ? k_conv_small(c, dy, L.Wpd, nullptr, din, gd) : k_conv_simt(c, dy, L.Wpd, nullptr, din, gd);
  }
  return FG_OK;
}
