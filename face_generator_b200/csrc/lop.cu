// L-op level of the C ABI: single layers at the nn.Module boundary (NCHW fp32, host or device
// pointers).  These are what the Lua `b200.*` nn.Module shims call from updateOutput /
// updateGradInput / accGradParameters; they reuse the same kernels as the fused nets and convert
// NCHW <-> NHWC around them (the fused L-net / L-step paths never pay that conversion).
#include <cstring>

#include "fg_internal.h"
#include "k_conv_tc.h"
#include "k_misc.h"

namespace {
int scratch(fg_ctx* c, int slot, size_t n, float** out) {
  if (c->scratch_elems[slot] < n) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    if (c->scratch[slot]) FG_CUDA(cudaFree(c->scratch[slot]));
    c->scratch[slot] = nullptr;
    c->scratch_elems[slot] = 0;
    FG_CUDA(cudaMalloc((void**)&c->scratch[slot], n * sizeof(float)));
    c->scratch_elems[slot] = n;
  }
  *out = c->scratch[slot];
  return FG_OK;
}
// device copy of a user tensor (slot used only for host pointers)
int in_dev(fg_ctx* c, const float* p, size_t n, int slot, const float** out) {
  if (fg_is_dev(p)) {
    *out = p;
    return FG_OK;
  }
  float* s;
  FG_TRY(scratch(c, slot, n, &s));
  FG_CUDA(cudaMemcpyAsync(s, p, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  *out = s;
  return FG_OK;
}
// device buffer to produce a user output in; finish with out_done()
int out_dev(fg_ctx* c, float* user, size_t n, int slot, float** dev, bool load) {
  if (fg_is_dev(user)) {
    *dev = user;
    return FG_OK;
  }
  FG_TRY(scratch(c, slot, n, dev));
  if (load) FG_CUDA(cudaMemcpyAsync(*dev, user, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  return FG_OK;
}
int out_done(fg_ctx* c, float* user, const float* dev, size_t n) {
  if (user == dev) return FG_OK;
  FG_CUDA(cudaMemcpyAsync(user, dev, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
}  // namespace

#define ENTER(c)                                      \
  do {                                                \
    if (!(c)) {                                       \
      fg_set_error("null fg_ctx");                    \
      return FG_ERR_INVALID;                          \
    }                                                 \
    FG_CUDA(cudaSetDevice((c)->device));              \
    note_conv((c), FG_KERNEL_NONE, 0, 0, 0, 0);       \
  } while (0)
// the shape every convolution entry point accepts: positive sizes, an odd kernel ("same" padding (k-1)/2)
#define CONV_SHAPE_OK (N > 0 && Cin > 0 && Cout > 0 && H > 0 && W > 0 && k >= 1 && (k & 1))

extern "C" {

int fg_conv2d_forward(fg_ctx* c, const float* x, const float* w, const float* b, float* y, int N, int Cin, int H, int W,
                      int Cout, int k) {
  ENTER(c);
  FG_REQUIRE(x && w && y && CONV_SHAPE_OK,
             "fg_conv2d_forward: bad arguments (odd kernel sizes only: same padding (k-1)/2)");
  const size_t nx = (size_t)N * Cin * H * W, ny = (size_t)N * Cout * H * W, nw = (size_t)Cout * Cin * k * k;
  const float *xd, *wd, *bd = nullptr;
  FG_TRY(in_dev(c, x, nx, 0, &xd));
  FG_TRY(in_dev(c, w, nw, 1, &wd));
  if (b) FG_TRY(in_dev(c, b, Cout, 2, &bd));
  float *xn, *wp, *yn, *yd;
  FG_TRY(scratch(c, 3, nx, &xn));
  FG_TRY(scratch(c, 4, nw, &wp));
  FG_TRY(scratch(c, 5, ny, &yn));
  FG_TRY(k_nchw_to_nhwc(c, xd, xn, N, Cin, H * W));
  const ConvGeom g{N, H, W, Cin, Cout, k, 1};
  if (c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(g) && c->mma_f16 && Cin % 64 == 0 && nx % 4 == 0) {
    float *xs, *ws;  // FP16 split: nx (nw) halves each for hi and lo = nx (nw) floats of scratch
    FG_TRY(scratch(c, 4, nx, &xs));
    FG_TRY(scratch(c, 7, nw, &ws));
    FG_TRY(tc_amax(c, xn, (int64_t)nx, c->lop_sx));  // activations are scaled into fp16's range as well
    FG_TRY(tc_split_h(c, xn, xs, xs + nx / 2, (int64_t)nx, c->lop_sx));
    FG_TRY(tc_pack_split_h(c, wd, ws, ws + nw / 2, nullptr, nullptr, Cout, Cin, k * k));
    FG_TRY(tc_conv_fwd(c, xs, xs + nx / 2, ws, ws + nw / 2, bd, yn, g, 0, nullptr, nullptr, 1, c->lop_sx + 1));
  } else if (c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(g)) {
    float *xs, *ws;
    FG_TRY(scratch(c, 4, 2 * nx, &xs));
    FG_TRY(scratch(c, 7, 2 * nw, &ws));
    FG_TRY(tc_split(c, xn, xs, xs + nx, (int64_t)nx));
    FG_TRY(tc_pack_split(c, wd, ws, ws + nw, nullptr, nullptr, Cout, Cin, k * k));
    FG_TRY(tc_conv_fwd(c, xs, xs + nx, ws, ws + nw, bd, yn, g, 0));
  } else {
    FG_TRY(k_pack_weights(c, wd, wp, nullptr, Cout, Cin, k * k, 0, 0, 0, 0));
    if (c->edge_impl && k_edge_eligible(g)) FG_TRY(k_conv_edge(c, xn, wp, bd, yn, g));  // 3-channel image edge
    else FG_TRY(k_conv_simt(c, xn, wp, bd, yn, g));
  }
  FG_TRY(out_dev(c, y, ny, 6, &yd, false));
  FG_TRY(k_nhwc_to_nchw(c, yn, yd, N, Cout, H * W));
  return out_done(c, y, yd, ny);
}

int fg_conv2d_backward_data(fg_ctx* c, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W, int Cout,
                            int k) {
  ENTER(c);
  FG_REQUIRE(dy && w && dx && CONV_SHAPE_OK, "fg_conv2d_backward_data: bad arguments (N %d, Cin %d, %dx%d, Cout %d, k %d)",
             N, Cin, H, W, Cout, k);
  const size_t nx = (size_t)N * Cin * H * W, ny = (size_t)N * Cout * H * W, nw = (size_t)Cout * Cin * k * k;
  const float *dyd, *wd;
  FG_TRY(in_dev(c, dy, ny, 0, &dyd));
  FG_TRY(in_dev(c, w, nw, 1, &wd));
  float *dyn, *wpd, *dxn, *dxd;
  FG_TRY(scratch(c, 3, ny, &dyn));
  FG_TRY(scratch(c, 4, nw, &wpd));
  FG_TRY(scratch(c, 5, nx, &dxn));
  FG_TRY(k_nchw_to_nhwc(c, dyd, dyn, N, Cout, H * W));
  const ConvGeom gd{N, H, W, Cout, Cin, k, 1};
  if (c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(gd) && c->mma_f16 && Cout % 64 == 0 && ny % 4 == 0 && nw % 2 == 0) {
    float *ys, *ws;  // the gradient is scaled by a power of two into fp16's range first (tc_amax), the kernel undoes it
    FG_TRY(scratch(c, 2, ny, &ys));
    FG_TRY(scratch(c, 7, 2 * nw, &ws));
    FG_TRY(tc_amax(c, dyn, (int64_t)ny, c->lop_sy));
    FG_TRY(tc_split_h(c, dyn, ys, ys + ny / 2, (int64_t)ny, c->lop_sy));
    FG_TRY(tc_pack_split_h(c, wd, ws, ws + nw / 2, ws + nw, ws + nw + nw / 2, Cout, Cin, k * k));
    FG_TRY(tc_conv_fwd(c, ys, ys + ny / 2, ws + nw, ws + nw + nw / 2, nullptr, dxn, gd, 0, nullptr, nullptr, 1, c->lop_sy + 1));
  } else if (c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(gd)) {
    float *ys, *ws;
    FG_TRY(scratch(c, 2, 2 * ny, &ys));
    FG_TRY(scratch(c, 7, 4 * nw, &ws));
    FG_TRY(tc_split(c, dyn, ys, ys + ny, (int64_t)ny));
    FG_TRY(tc_pack_split(c, wd, ws, ws + nw, ws + 2 * nw, ws + 3 * nw, Cout, Cin, k * k));
    FG_TRY(tc_conv_fwd(c, ys, ys + ny, ws + 2 * nw, ws + 3 * nw, nullptr, dxn, gd, 0));
  } else {
    FG_TRY(k_pack_weights(c, wd, nullptr, wpd, Cout, Cin, k * k, 0, 0, 0, 0));
    if (c->edge_impl && k_edge_eligible(gd)) FG_TRY(k_conv_edge(c, dyn, wpd, nullptr, dxn, gd));
    else FG_TRY(k_conv_simt(c, dyn, wpd, nullptr, dxn, gd));
  }
  FG_TRY(out_dev(c, dx, nx, 6, &dxd, false));
  FG_TRY(k_nhwc_to_nchw(c, dxn, dxd, N, Cin, H * W));
  return out_done(c, dx, dxd, nx);
}

int fg_conv2d_backward_filter(fg_ctx* c, const float* x, const float* dy, float* dw, float* db, int N, int Cin, int H,
                              int W, int Cout, int k) {
  ENTER(c);
  FG_REQUIRE(x && dy && dw && CONV_SHAPE_OK, "fg_conv2d_backward_filter: bad arguments (N %d, Cin %d, %dx%d, Cout %d, k %d)",
             N, Cin, H, W, Cout, k);
  const size_t nx = (size_t)N * Cin * H * W, ny = (size_t)N * Cout * H * W, nw = (size_t)Cout * Cin * k * k;
  const float *xd, *dyd;
  FG_TRY(in_dev(c, x, nx, 0, &xd));
  FG_TRY(in_dev(c, dy, ny, 1, &dyd));
  float *xn, *dyn, *ws, *dwd, *dbd = nullptr;
  FG_TRY(scratch(c, 3, nx, &xn));
  FG_TRY(scratch(c, 4, ny, &dyn));
  FG_TRY(scratch(c, 5, nw, &ws));
  FG_TRY(k_nchw_to_nhwc(c, xd, xn, N, Cin, H * W));
  FG_TRY(k_nchw_to_nhwc(c, dyd, dyn, N, Cout, H * W));
  const ConvGeom gw{N, H, W, Cin, Cout, k, 1};
  if (c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(gw) && Cout % 128 == 0 && Cin % 64 == 0 && c->mma_f16 && nx % 8 == 0 &&
      ny % 8 == 0) {
    float *xs, *ys;  // FP16 split; dY scaled into range by a power of two that the kernel undoes
    FG_TRY(scratch(c, 2, nx, &xs));
    FG_TRY(scratch(c, 7, ny, &ys));
    FG_TRY(tc_amax(c, xn, (int64_t)nx, c->lop_sx));
    FG_TRY(tc_split_h(c, xn, xs, xs + nx / 2, (int64_t)nx, c->lop_sx));
    FG_TRY(tc_amax(c, dyn, (int64_t)ny, c->lop_sy));
    FG_TRY(tc_split_h(c, dyn, ys, ys + ny / 2, (int64_t)ny, c->lop_sy));
    FG_TRY(tc_conv_wgrad(c, xs, xs + nx / 2, ys, ys + ny / 2, ws, gw, 1, c->lop_sy + 1, c->lop_sx + 1));
  } else if (c->conv_impl != FG_CONV_SIMT && tc_conv_eligible(gw) && Cout % 128 == 0 && Cin % 64 == 0) {
    float *xs, *ys;
    FG_TRY(scratch(c, 2, 2 * nx, &xs));
    FG_TRY(scratch(c, 7, 2 * ny, &ys));
    FG_TRY(tc_split(c, xn, xs, xs + nx, (int64_t)nx));
    FG_TRY(tc_split(c, dyn, ys, ys + ny, (int64_t)ny));
    FG_TRY(tc_conv_wgrad(c, xs, xs + nx, ys, ys + ny, ws, gw));
  } else {
    FG_TRY(k_wgrad_simt(c, xn, dyn, ws, gw));
  }
  FG_TRY(out_dev(c, dw, nw, 6, &dwd, true));
  FG_TRY(k_unpack_wgrad(c, ws, dwd, Cout, Cin, k * k, 0, 0, 0, 0));
  if (db) {
    FG_TRY(out_dev(c, db, Cout, 7, &dbd, true));
    FG_TRY(k_colsum_add(c, dyn, dbd, (int64_t)N * H * W, Cout, 0, 0));
  }
  FG_TRY(out_done(c, dw, dwd, nw));
  if (db) FG_TRY(out_done(c, db, dbd, Cout));
  return FG_OK;
}

// cudnn.SpatialConvolutionUpsample (layers/cudnnSpatialConvolutionUpsample.lua): parent.__init(nInputPlane,
// nOutputPlane*factor*factor, ...) at :14-15, and every pass only re-views the contiguous output / gradOutput between
// [N][nOut*f*f][h][w] and [N][nOut][h*f][w*f] (:18-30, :32-58) -- the bytes do not move, so the layer IS the
// convolution with nOut*f*f planes on the caller's buffer.
static int scu_planes(fg_ctx* c, int nOutputPlane, int factor, int* planes) {
  if (c) note_conv(c, FG_KERNEL_NONE, 0, 0, 0, 0);  // a refusal here does not report the previous call's kernel
  FG_REQUIRE(nOutputPlane > 0 && factor >= 1 && (int64_t)nOutputPlane * factor * factor < (1 << 20),
             "SpatialConvolutionUpsample: bad nOutputPlane %d / factor %d", nOutputPlane, factor);
  *planes = nOutputPlane * factor * factor;
  return FG_OK;
}
int fg_scu_forward(fg_ctx* c, const float* x, const float* w, const float* b, float* y, int N, int Cin, int H, int W,
                   int nOutputPlane, int k, int factor) {
  int planes;
  FG_TRY(scu_planes(c, nOutputPlane, factor, &planes));
  return fg_conv2d_forward(c, x, w, b, y, N, Cin, H, W, planes, k);
}
int fg_scu_backward_data(fg_ctx* c, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W,
                         int nOutputPlane, int k, int factor) {
  int planes;
  FG_TRY(scu_planes(c, nOutputPlane, factor, &planes));
  return fg_conv2d_backward_data(c, dy, w, dx, N, Cin, H, W, planes, k);
}
int fg_scu_backward_filter(fg_ctx* c, const float* x, const float* dy, float* dw, float* db, int N, int Cin, int H, int W,
                           int nOutputPlane, int k, int factor) {
  int planes;
  FG_TRY(scu_planes(c, nOutputPlane, factor, &planes));
  return fg_conv2d_backward_filter(c, x, dy, dw, db, N, Cin, H, W, planes, k);
}

int fg_linear_forward(fg_ctx* c, const float* x, const float* w, const float* b, float* y, int N, int in, int out) {
  ENTER(c);
  FG_REQUIRE(x && w && y && N > 0 && in > 0 && out > 0, "fg_linear_forward: bad arguments");
  const float *xd, *wd, *bd = nullptr;
  FG_TRY(in_dev(c, x, (size_t)N * in, 0, &xd));
  FG_TRY(in_dev(c, w, (size_t)out * in, 1, &wd));
  if (b) FG_TRY(in_dev(c, b, out, 2, &bd));
  float* yd;
  FG_TRY(out_dev(c, y, (size_t)N * out, 6, &yd, false));
  FG_TRY(k_conv_simt(c, xd, wd, bd, yd, ConvGeom{N, 1, 1, in, out, 1, 1}));  // W[out][in] is already [n][c]
  return out_done(c, y, yd, (size_t)N * out);
}

int fg_linear_backward(fg_ctx* c, const float* x, const float* w, const float* dy, float* dx, float* dw, float* db, int N,
                       int in, int out) {
  ENTER(c);
  FG_REQUIRE(x && w && dy && N > 0 && in > 0 && out > 0, "fg_linear_backward: bad arguments");
  const float *xd, *wd, *dyd;
  FG_TRY(in_dev(c, x, (size_t)N * in, 0, &xd));
  FG_TRY(in_dev(c, w, (size_t)out * in, 1, &wd));
  FG_TRY(in_dev(c, dy, (size_t)N * out, 2, &dyd));
  if (dx) {
    float *wpd, *dxd;
    FG_TRY(scratch(c, 3, (size_t)out * in, &wpd));
    FG_TRY(k_pack_weights(c, wd, nullptr, wpd, out, in, 1, 0, 0, 0, 0));
    FG_TRY(out_dev(c, dx, (size_t)N * in, 6, &dxd, false));
    FG_TRY(k_conv_simt(c, dyd, wpd, nullptr, dxd, ConvGeom{N, 1, 1, out, in, 1, 1}));
    FG_TRY(out_done(c, dx, dxd, (size_t)N * in));
  }
  if (dw) {
    float *ws, *dwd;
    FG_TRY(scratch(c, 4, (size_t)out * in, &ws));
    FG_TRY(k_wgrad_simt(c, xd, dyd, ws, ConvGeom{N, 1, 1, in, out, 1, 1}));
    FG_TRY(out_dev(c, dw, (size_t)out * in, 6, &dwd, true));
    FG_TRY(k_unpack_wgrad(c, ws, dwd, out, in, 1, 0, 0, 0, 0));
    FG_TRY(out_done(c, dw, dwd, (size_t)out * in));
  }
  if (db) {
    float* dbd;
    FG_TRY(out_dev(c, db, out, 7, &dbd, true));
    FG_TRY(k_colsum_add(c, dyd, dbd, N, out, 0, 0));
    FG_TRY(out_done(c, db, dbd, out));
  }
  return FG_OK;
}

int fg_bn_forward_train(fg_ctx* c, const float* x, const float* gamma, const float* beta, float* y, float* save_mean,
                        float* save_istd, float* run_mean, float* run_var, int N, int C, int HW) {
  ENTER(c);
  FG_REQUIRE(x && gamma && beta && y && save_mean && save_istd && N > 0 && C > 0 && C <= 1024,
             "fg_bn_forward_train: bad arguments (C <= 1024)");
  const size_t n = (size_t)N * C * HW;
  const float *xd, *gd, *bd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, gamma, C, 1, &gd));
  FG_TRY(in_dev(c, beta, C, 2, &bd));
  float *xn, *yn, *small, *yd;
  FG_TRY(scratch(c, 3, n, &xn));
  FG_TRY(scratch(c, 4, n, &yn));
  FG_TRY(scratch(c, 5, (size_t)8 * C + 16, &small));  // [acc 2C doubles = 4C floats][mean C][istd C][rm C][rv C]
  double* acc = (double*)small;
  float *mean = small + 4 * C, *istd = mean + C, *rm = istd + C, *rv = rm + C;
  if (run_mean) FG_CUDA(cudaMemcpyAsync(rm, run_mean, C * sizeof(float), cudaMemcpyDefault, c->stream));
  if (run_var) FG_CUDA(cudaMemcpyAsync(rv, run_var, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_TRY(k_nchw_to_nhwc(c, xd, xn, N, C, HW));
  FG_TRY(k_bn_stats(c, xn, acc, (int64_t)N * HW, C));
  FG_TRY(k_bn_finalize(c, acc, mean, istd, run_mean ? rm : nullptr, run_var ? rv : nullptr, (int64_t)N * HW, C));
  FG_TRY(k_bn_prelu_apply(c, xn, mean, istd, gd, bd, nullptr, yn, (int64_t)N * HW, C));
  FG_TRY(out_dev(c, y, n, 6, &yd, false));
  FG_TRY(k_nhwc_to_nchw(c, yn, yd, N, C, HW));
  FG_TRY(out_done(c, y, yd, n));
  FG_CUDA(cudaMemcpyAsync(save_mean, mean, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemcpyAsync(save_istd, istd, C * sizeof(float), cudaMemcpyDefault, c->stream));
  if (run_mean) FG_CUDA(cudaMemcpyAsync(run_mean, rm, C * sizeof(float), cudaMemcpyDefault, c->stream));
  if (run_var) FG_CUDA(cudaMemcpyAsync(run_var, rv, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int fg_bn_backward(fg_ctx* c, const float* x, const float* gamma, const float* save_mean, const float* save_istd,
                   const float* dy, float* dx, float* dgamma, float* dbeta, int N, int C, int HW) {
  ENTER(c);
  FG_REQUIRE(x && gamma && save_mean && save_istd && dy && dx && N > 0 && C > 0 && C <= 1024,
             "fg_bn_backward: bad arguments (C <= 1024)");
  const size_t n = (size_t)N * C * HW;
  const float *xd, *dyd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, dy, n, 1, &dyd));
  float *xn, *dyn, *dxn, *small, *dxd;
  FG_TRY(scratch(c, 2, n, &xn));
  FG_TRY(scratch(c, 3, n, &dyn));
  FG_TRY(scratch(c, 4, n, &dxn));
  FG_TRY(scratch(c, 5, (size_t)12 * C + 16, &small));
  double* acc = (double*)small;
  float *gd = small + 4 * C, *mean = gd + C, *istd = mean + C, *mg = istd + C, *dg = mg + 2 * C, *db = dg + C,
        *zero = db + C;
  FG_CUDA(cudaMemcpyAsync(gd, gamma, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemcpyAsync(mean, save_mean, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemcpyAsync(istd, save_istd, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemsetAsync(zero, 0, C * sizeof(float), c->stream));
  if (dgamma) FG_CUDA(cudaMemcpyAsync(dg, dgamma, C * sizeof(float), cudaMemcpyDefault, c->stream));
  if (dbeta) FG_CUDA(cudaMemcpyAsync(db, dbeta, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_TRY(k_nchw_to_nhwc(c, xd, xn, N, C, HW));
  FG_TRY(k_nchw_to_nhwc(c, dyd, dyn, N, C, HW));
  // H=HW, W=1 flattening is fine: no pooling here
  FG_TRY(k_bn_prelu_bwd_reduce(c, dyn, xn, mean, istd, gd, zero, nullptr, acc, nullptr, N, HW, 1, C, 0));
  FG_TRY(k_bn_bwd_finalize(c, acc, mg, dgamma ? dg : nullptr, dbeta ? db : nullptr, (int64_t)N * HW, C));
  FG_TRY(k_bn_prelu_bwd_apply(c, dyn, xn, mean, istd, gd, zero, nullptr, mg, dxn, N, HW, 1, C, 0));
  FG_TRY(out_dev(c, dx, n, 6, &dxd, false));
  FG_TRY(k_nhwc_to_nchw(c, dxn, dxd, N, C, HW));
  FG_TRY(out_done(c, dx, dxd, n));
  if (dgamma) FG_CUDA(cudaMemcpyAsync(dgamma, dg, C * sizeof(float), cudaMemcpyDefault, c->stream));
  if (dbeta) FG_CUDA(cudaMemcpyAsync(dbeta, db, C * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int fg_prelu_forward(fg_ctx* c, const float* x, const float* slope, float* y, int64_t n) {
  ENTER(c);
  FG_REQUIRE(x && slope && y && n > 0, "fg_prelu_forward: bad arguments");
  const float *xd, *sd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, slope, 1, 1, &sd));
  float* yd;
  FG_TRY(out_dev(c, y, n, 6, &yd, false));
  FG_TRY(k_prelu_fwd(c, xd, sd, yd, n));
  return out_done(c, y, yd, n);
}
int fg_prelu_backward(fg_ctx* c, const float* x, const float* slope, const float* dy, float* dx, float* dslope, int64_t n) {
  ENTER(c);
  FG_REQUIRE(x && slope && dy && dx && n > 0 && n < (int64_t)1 << 31, "fg_prelu_backward: bad arguments");
  const float *xd, *sd, *dyd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, slope, 1, 1, &sd));
  FG_TRY(in_dev(c, dy, n, 2, &dyd));
  float *dxd, *dsd = nullptr;
  FG_TRY(out_dev(c, dx, n, 6, &dxd, false));
  if (dslope) FG_TRY(out_dev(c, dslope, 1, 7, &dsd, true));
  FG_TRY(k_prelu_bwd(c, dyd, xd, sd, dxd, dsd, 1, (int)n, 1, 1, 0));
  FG_TRY(out_done(c, dx, dxd, n));
  if (dslope) FG_TRY(out_done(c, dslope, dsd, 1));
  return FG_OK;
}

// ---- resampling / pooling / dropout / sigmoid: NCHW kernels, no layout round trip --------------------
// shared shape: one input of nin floats, one output of nout floats
#define UNARY_LOP(NAME, IN, OUT, NIN, NOUT, CALL)                                   \
  ENTER(c);                                                                         \
  FG_REQUIRE(IN && OUT && N > 0 && C > 0 && H > 0 && W > 0, NAME ": bad arguments"); \
  const size_t nin = (NIN), nout = (NOUT);                                          \
  const float* ind;                                                                 \
  float* outd;                                                                      \
  FG_TRY(in_dev(c, IN, nin, 0, &ind));                                              \
  FG_TRY(out_dev(c, OUT, nout, 6, &outd, false));                                   \
  FG_TRY(CALL);                                                                     \
  return out_done(c, OUT, outd, nout)

int fg_upsample2_forward(fg_ctx* c, const float* x, float* y, int N, int C, int H, int W) {
  UNARY_LOP("fg_upsample2_forward", x, y, (size_t)N * C * H * W, (size_t)N * C * H * W * 4,
            k_up2_fwd_nchw(c, ind, outd, (int64_t)N * C, H, W));
}
int fg_upsample2_backward(fg_ctx* c, const float* dy, float* dx, int N, int C, int H, int W) {
  UNARY_LOP("fg_upsample2_backward", dy, dx, (size_t)N * C * H * W * 4, (size_t)N * C * H * W,
            k_up2_bwd_nchw(c, ind, outd, (int64_t)N * C, H, W));
}
int fg_avgpool2_forward(fg_ctx* c, const float* x, float* y, int N, int C, int H, int W) {
  UNARY_LOP("fg_avgpool2_forward", x, y, (size_t)N * C * H * W, (size_t)N * C * (H / 2) * (W / 2),
            k_avgpool2_fwd_nchw(c, ind, outd, (int64_t)N * C, H, W));
}
int fg_avgpool2_backward(fg_ctx* c, const float* dy, float* dx, int N, int C, int H, int W) {
  UNARY_LOP("fg_avgpool2_backward", dy, dx, (size_t)N * C * (H / 2) * (W / 2), (size_t)N * C * H * W,
            k_avgpool2_bwd_nchw(c, ind, outd, (int64_t)N * C, H, W));
}
int fg_maxpool2_forward(fg_ctx* c, const float* x, float* y, int N, int C, int H, int W) {
  UNARY_LOP("fg_maxpool2_forward", x, y, (size_t)N * C * H * W, (size_t)N * C * (H / 2) * (W / 2),
            k_maxpool2_fwd_nchw(c, ind, outd, (int64_t)N * C, H, W));
}
#undef UNARY_LOP
int fg_maxpool2_backward(fg_ctx* c, const float* x, const float* dy, float* dx, int N, int C, int H, int W) {
  ENTER(c);
  FG_REQUIRE(x && dy && dx && N > 0 && C > 0 && H > 0 && W > 0, "fg_maxpool2_backward: bad arguments");
  const size_t nx = (size_t)N * C * H * W, ny = (size_t)N * C * (H / 2) * (W / 2);
  const float *xd, *dyd;
  float* dxd;
  FG_TRY(in_dev(c, x, nx, 0, &xd));
  FG_TRY(in_dev(c, dy, ny, 1, &dyd));
  FG_TRY(out_dev(c, dx, nx, 6, &dxd, false));
  FG_TRY(k_maxpool2_bwd_nchw(c, xd, dyd, dxd, (int64_t)N * C, H, W));
  return out_done(c, dx, dxd, nx);
}

static int dropout_apply(fg_ctx* c, const char* who, const float* x, const float* mask, float p, int spatial, float* y, int N,
                         int C, int HW) {
  ENTER(c);
  FG_REQUIRE(x && y && N > 0 && C > 0 && HW > 0 && p >= 0.f && p < 1.f, "%s: bad arguments", who);
  const size_t n = (size_t)N * C * HW, nm = spatial ? (size_t)N * C : n;
  const float *xd, *md = nullptr;
  float* yd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  if (mask) FG_TRY(in_dev(c, mask, nm, 1, &md));
  FG_TRY(out_dev(c, y, n, 6, &yd, false));
  // training: nn.Dropout rescales by 1/(1-p), nn.SpatialDropout does not; evaluate(): identity resp. (1-p)
  const float scale = mask ? (spatial ? 1.f : 1.f / (1.f - p)) : (spatial ? 1.f - p : 1.f);
  FG_TRY(k_dropout_nchw(c, xd, md, scale, spatial ? HW : 1, yd, (int64_t)n));
  return out_done(c, y, yd, n);
}
int fg_dropout_forward(fg_ctx* c, const float* x, const float* mask, float p, int spatial, float* y, int N, int C, int HW) {
  return dropout_apply(c, "fg_dropout_forward", x, mask, p, spatial, y, N, C, HW);
}
int fg_dropout_backward(fg_ctx* c, const float* dy, const float* mask, float p, int spatial, float* dx, int N, int C,
                        int HW) {
  return dropout_apply(c, "fg_dropout_backward", dy, mask, p, spatial, dx, N, C, HW);
}
int fg_dropout_mask(fg_ctx* c, float* mask_dev, int64_t n, float p, uint64_t seed) {
  ENTER(c);
  FG_REQUIRE(mask_dev && n > 0 && fg_is_dev(mask_dev), "fg_dropout_mask: needs a device buffer");
  return k_bernoulli_keep(c, mask_dev, n, seed, p);
}

int fg_sigmoid_forward(fg_ctx* c, const float* x, float* y, int64_t n) {
  ENTER(c);
  FG_REQUIRE(x && y && n > 0, "fg_sigmoid_forward: bad arguments");
  const float* xd;
  float* yd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(out_dev(c, y, n, 6, &yd, false));
  FG_TRY(k_sigmoid_fwd(c, xd, yd, n));
  return out_done(c, y, yd, n);
}
int fg_sigmoid_backward(fg_ctx* c, const float* y, const float* dy, float* dx, int64_t n) {
  ENTER(c);
  FG_REQUIRE(y && dy && dx && n > 0, "fg_sigmoid_backward: bad arguments");
  const float *yd, *dyd;
  float* dxd;
  FG_TRY(in_dev(c, y, n, 0, &yd));
  FG_TRY(in_dev(c, dy, n, 1, &dyd));
  FG_TRY(out_dev(c, dx, n, 6, &dxd, false));
  FG_TRY(k_sigmoid_bwd(c, dyd, yd, dxd, n));
  return out_done(c, dx, dxd, n);
}


// nn.ReLU, nn.Tanh and nn.AbsCriterion (the layers of train_autoencoder.lua's net), flat tensors of n floats
int fg_relu_forward(fg_ctx* c, const float* x, float* y, int64_t n) {
  ENTER(c);
  FG_REQUIRE(x && y && n > 0, "fg_relu_forward: bad arguments");
  const float* xd;
  float* yd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(out_dev(c, y, n, 6, &yd, false));
  FG_TRY(k_relu_fwd(c, xd, yd, n));
  return out_done(c, y, yd, n);
}
int fg_relu_backward(fg_ctx* c, const float* x, const float* dy, float* dx, int64_t n) {
  ENTER(c);
  FG_REQUIRE(x && dy && dx && n > 0, "fg_relu_backward: bad arguments");
  const float *xd, *dyd;
  float* dxd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, dy, n, 1, &dyd));
  FG_TRY(out_dev(c, dx, n, 6, &dxd, false));
  FG_TRY(k_relu_bwd(c, dyd, xd, dxd, n));
  return out_done(c, dx, dxd, n);
}
int fg_tanh_forward(fg_ctx* c, const float* x, float* y, int64_t n) {
  ENTER(c);
  FG_REQUIRE(x && y && n > 0, "fg_tanh_forward: bad arguments");
  const float* xd;
  float* yd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(out_dev(c, y, n, 6, &yd, false));
  FG_TRY(k_tanh_dropout_fwd(c, xd, nullptr, nullptr, 0.f, yd, nullptr, nullptr, n));
  return out_done(c, y, yd, n);
}
int fg_tanh_backward(fg_ctx* c, const float* y, const float* dy, float* dx, int64_t n) {
  ENTER(c);
  FG_REQUIRE(y && dy && dx && n > 0, "fg_tanh_backward: bad arguments");
  const float *yd, *dyd;
  float* dxd;
  FG_TRY(in_dev(c, y, n, 0, &yd));
  FG_TRY(in_dev(c, dy, n, 1, &dyd));
  FG_TRY(out_dev(c, dx, n, 6, &dxd, false));
  FG_TRY(k_tanh_dropout_bwd(c, dyd, nullptr, 0.f, yd, dxd, n));
  return out_done(c, dx, dxd, n);
}
int fg_abs_forward(fg_ctx* c, const float* x, const float* t, int64_t n, float* loss_out) {
  ENTER(c);
  FG_REQUIRE(x && t && loss_out && n > 0, "fg_abs_forward: bad arguments");
  const float *xd, *td;
  float* ld;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, t, n, 1, &td));
  FG_TRY(out_dev(c, loss_out, 1, 6, &ld, false));
  FG_TRY(k_abs_criterion(c, false, xd, td, nullptr, nullptr, n, ld));
  return out_done(c, loss_out, ld, 1);
}
int fg_abs_backward(fg_ctx* c, const float* x, const float* t, int64_t n, float* dx) {
  ENTER(c);
  FG_REQUIRE(x && t && dx && n > 0, "fg_abs_backward: bad arguments");
  const float *xd, *td;
  float* dxd;
  FG_TRY(in_dev(c, x, n, 0, &xd));
  FG_TRY(in_dev(c, t, n, 1, &td));
  FG_TRY(out_dev(c, dx, n, 6, &dxd, false));
  FG_TRY(k_abs_criterion(c, false, xd, td, nullptr, dxd, n, nullptr));
  return out_done(c, dx, dxd, n);
}

}  // extern "C"
