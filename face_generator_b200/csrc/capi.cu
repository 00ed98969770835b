// C ABI of libfg_b200.so (include/fg_b200.h).  Thin: argument checking, host/device pointer
// classification, NCHW<->NHWC at the boundary, then nets.cu / kernels.
#include <cstdarg>
#include <cstdlib>
#include <cstring>

#include "fg_internal.h"
#include "k_conv_tc.h"

static thread_local char g_err[1024] = "";
void fg_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

#define ENTER(c)                                      \
  do {                                                \
    if (!(c)) {                                       \
      fg_set_error("null fg_ctx");                    \
      return FG_ERR_INVALID;                          \
    }                                                 \
    FG_CUDA(cudaSetDevice((c)->device));              \
  } while (0)

namespace {
bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
// returns a device pointer holding n floats of `p` (p itself when already on the device)
int to_dev(fg_ctx* c, const float* p, size_t n, float* staging, const float** out) {
  if (is_device_ptr(p)) {
    *out = p;
    return FG_OK;
  }
  FG_CUDA(cudaMemcpyAsync(staging, p, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  *out = staging;
  return FG_OK;
}
// copy n floats from a device buffer to a user pointer (host => synchronise so it is valid on return)
int to_user(fg_ctx* c, float* dst, const float* src_dev, size_t n) {
  if (dst == src_dev) return FG_OK;
  const bool dev = is_device_ptr(dst);
  FG_CUDA(cudaMemcpyAsync(dst, src_dev, n * sizeof(float), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                          c->stream));
  if (!dev) FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
}  // namespace

extern "C" {

const char* fg_version(void) { return "fg_b200 0.1 (sm_90a)"; }
const char* fg_last_error(void) { return g_err; }

void fg_hyper_default(fg_hyper* h) {
  if (!h) return;
  h->lr_D = 1e-3f; h->lr_G = 1e-3f;
  h->beta1 = 0.9f; h->beta2 = 0.999f; h->eps = 1e-8f;
  h->D_L1 = 0.f; h->D_L2 = 1e-4f;
  h->G_L1 = 0.f; h->G_L2 = 0.f;
  h->D_clamp = 1.f; h->G_clamp = 5.f;
  h->D_maxAcc = 1.01f;
  h->accs_interval = 20;
  h->p_spatial = 0.2f; h->p_drop = 0.5f;
}

int fg_create(fg_ctx** out, int device, int max_batch, int channels) {
  if (!out) { fg_set_error("fg_create: out is null"); return FG_ERR_INVALID; }
  *out = nullptr;
  FG_REQUIRE(channels == 1 || channels == 3, "fg_create: channels must be 1 or 3 (got %d)", channels);
  FG_REQUIRE(max_batch >= 4 && max_batch % 2 == 0, "fg_create: max_batch must be even and >= 4 (got %d)", max_batch);
  int ndev = 0;
  FG_CUDA(cudaGetDeviceCount(&ndev));
  FG_REQUIRE(device >= 0 && device < ndev, "fg_create: device %d not present (%d CUDA devices); there is no CPU fallback",
             device, ndev);
  FG_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  FG_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    fg_set_error("fg_create: device %d is sm_%d%d; this library only contains sm_90a code", device, prop.major, prop.minor);
    return FG_ERR_UNSUPPORTED;
  }
  fg_ctx* c = new fg_ctx();
  c->device = device;
  c->maxB = max_batch;
  c->C = channels;
  c->sm_count = prop.multiProcessorCount;
  if (const char* e = getenv("FG_MMA_F16")) c->mma_f16 = atoi(e) != 0;  // experiment switch for option "mma_f16"
  if (const char* e = getenv("FG_DP_OVERLAP")) c->dp_overlap = atoi(e) != 0;
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    fg_set_error("fg_create: cudaStreamCreate failed");
    delete c;
    return FG_ERR_CUDA;
  }
  int r = net_alloc(c);
  if (r == FG_OK) r = tc_init(c);
  if (r != FG_OK) {
    net_free(c);
    cudaStreamDestroy(c->stream);
    delete c;
    return r;
  }
  *out = c;
  return FG_OK;
}

int fg_destroy(fg_ctx* c) {
  if (!c) return FG_OK;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  net_graphs_clear(c);
  if (c->comm_stream) {
    cudaStreamSynchronize(c->comm_stream);
    cudaStreamDestroy(c->comm_stream);
    cudaEventDestroy(c->ev_fork);
    cudaEventDestroy(c->ev_join);
  }
  tc_destroy(c);
  net_free(c);
  for (auto& kv : c->timers)
    for (auto& pr : kv.second.pending) {
      cudaEventDestroy(pr.first);
      cudaEventDestroy(pr.second);
    }
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return FG_OK;
}

int fg_set_stream(fg_ctx* c, void* s) {
  ENTER(c);
  c->graph_epoch++;
  FG_CUDA(cudaStreamSynchronize(c->stream));
  if (s) {
    if (c->own_stream) cudaStreamDestroy(c->stream);
    c->stream = (cudaStream_t)s;
    c->own_stream = false;
  } else if (!c->own_stream) {
    FG_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  return FG_OK;
}
int fg_sync(fg_ctx* c) {
  ENTER(c);
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int fg_set_option(fg_ctx* c, const char* key, int64_t v) {
  ENTER(c);
  c->graph_epoch++;  // a captured step bakes the options in
  if (!strcmp(key, "conv_impl")) {
    FG_REQUIRE(v >= 0 && v <= 2, "conv_impl must be 0 (simt), 1 (tc dense) or 2 (tc collapsed)");
    c->conv_impl = (int)v;
    c->G_packed = c->D_packed = false;
    return FG_OK;
  }
  if (!strcmp(key, "params_dirty")) {
    c->G_packed = c->D_packed = false;
    return FG_OK;
  }
  if (!strcmp(key, "edge_impl")) {  // 1 (default): k_conv_edge.cu for the 3-channel-side convolutions; 0: k_conv_small.cu
    c->edge_impl = v != 0;
    return FG_OK;
  }
  if (!strcmp(key, "bn_epilogue")) {  // 1 (default): BatchNorm statistics from the tensor-core conv epilogue; 0: separate pass
    c->bn_epilogue = v != 0;
    return FG_OK;
  }
  if (!strcmp(key, "mma_f16")) {  // 1: K-major tensor-core kernels (forward, dgrad) use the 3xFP16 split + f16 MMAs
    c->mma_f16 = v != 0;
    c->G_packed = c->D_packed = false;
    return FG_OK;
  }
  if (!strcmp(key, "use_graph")) {  // 1 (default): fg_train_step replays a captured CUDA graph of the step
    c->use_graph = v != 0;
    c->graph_epoch++;
    return FG_OK;
  }
  if (!strcmp(key, "dp_overlap")) {  // 1 (default): D's all-reduce + optimizer overlap the G step's G forward (data parallel only)
    c->dp_overlap = v != 0;
    return FG_OK;
  }
  if (!strcmp(key, "debug_keep")) {  // keep the D step's pre-activations of fg_train_step ("Dstep.*" debug tensors)
    c->debug_keep = v != 0;
    return FG_OK;
  }
  if (!strcmp(key, "optimizer_D") || !strcmp(key, "optimizer_G")) {  // OPT.D_optmethod / OPT.G_optmethod (train.lua:38-39)
    FG_REQUIRE(v >= FG_OPT_ADAM && v <= FG_OPT_SGD, "%s must be 0 (adam), 1 (adagrad) or 2 (sgd)", key);
    (key[10] == 'D' ? c->opt_D : c->opt_G) = (int)v;
    return FG_OK;
  }
  fg_set_error("fg_set_option: unknown key '%s'", key);
  return FG_ERR_INVALID;
}
int fg_set_option_f(fg_ctx* c, const char* key, double v) {
  ENTER(c);
  c->graph_epoch++;
  if (!strcmp(key, "sgd_momentum_D") || !strcmp(key, "sgd_momentum_G")) {  // OPT.D_SGD_momentum / G_SGD_momentum (train.lua:23,25)
    FG_REQUIRE(v >= 0.0 && v < 1.0, "%s must be in [0, 1)", key);
    (key[13] == 'D' ? c->sgd_mom_D : c->sgd_mom_G) = (float)v;
    return FG_OK;
  }
  fg_set_error("fg_set_option_f: unknown key '%s'", key);
  return FG_ERR_INVALID;
}
int64_t fg_get_option(fg_ctx* c, const char* key) {
  if (!c || !key) return -1;
  if (!strcmp(key, "conv_impl")) return c->conv_impl;
  if (!strcmp(key, "max_batch")) return c->maxB;
  if (!strcmp(key, "channels")) return c->C;
  if (!strcmp(key, "sm_count")) return c->sm_count;
  if (!strcmp(key, "bn_epilogue")) return c->bn_epilogue;
  if (!strcmp(key, "edge_impl")) return c->edge_impl;
  if (!strcmp(key, "mma_f16")) return c->mma_f16;
  if (!strcmp(key, "dp_overlap")) return c->dp_overlap;
  if (!strcmp(key, "use_graph")) return c->use_graph;
  if (!strcmp(key, "optimizer_D")) return c->opt_D;
  if (!strcmp(key, "optimizer_G")) return c->opt_G;
  return -1;
}

int64_t fg_param_count(int net, int channels) {
  if (channels != 1 && channels != 3) return -1;
  return net == FG_NET_G ? make_g_layout(channels).total : net == FG_NET_D ? make_d_layout(channels).total : -1;
}
static int net_bufs(fg_ctx* c, int net, float** p, float** g, float** m, float** v, int64_t* n) {
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  const bool d = net == FG_NET_D;
  if (p) *p = d ? c->PD : c->PG;
  if (g) *g = d ? c->gD : c->gG;
  if (m) *m = d ? c->mD : c->mG;
  if (v) *v = d ? c->vD : c->vG;
  if (n) *n = d ? c->dl.total : c->gl.total;
  return FG_OK;
}
int fg_set_params(fg_ctx* c, int net, const float* src) {
  ENTER(c);
  float* p; int64_t n;
  FG_TRY(net_bufs(c, net, &p, nullptr, nullptr, nullptr, &n));
  FG_CUDA(cudaMemcpyAsync(p, src, n * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  c->G_packed = c->D_packed = false;
  return FG_OK;
}
int fg_get_params(fg_ctx* c, int net, float* dst) {
  ENTER(c);
  float* p; int64_t n;
  FG_TRY(net_bufs(c, net, &p, nullptr, nullptr, nullptr, &n));
  return to_user(c, dst, p, n);
}
int fg_get_grads(fg_ctx* c, int net, float* dst) {
  ENTER(c);
  float* g; int64_t n;
  FG_TRY(net_bufs(c, net, nullptr, &g, nullptr, nullptr, &n));
  return to_user(c, dst, g, n);
}
int fg_zero_grads(fg_ctx* c, int net) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return net_zero_grads(c, net);
}
// Borrow caller-owned DEVICE buffers as the flat parameter / gradient vectors of `net` (see include/fg_b200.h).
int fg_bind_params(fg_ctx* c, int net, float* params_dev, float* grads_dev) {
  ENTER(c);
  c->graph_epoch++;
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  for (const float* p : {params_dev, grads_dev}) {
    if (!p) continue;
    cudaPointerAttributes a;
    const bool dev = cudaPointerGetAttributes(&a, p) == cudaSuccess && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged);
    if (!dev) cudaGetLastError();
    FG_REQUIRE(dev, "fg_bind_params: buffers must be DEVICE memory (CudaTensor:data())");
    FG_REQUIRE(reinterpret_cast<uintptr_t>(p) % 16 == 0, "fg_bind_params: buffers must be 16-byte aligned");
  }
  FG_CUDA(cudaStreamSynchronize(c->stream));
  const bool d = net == FG_NET_D;
  (d ? c->PD : c->PG) = params_dev ? params_dev : (d ? c->ownPD : c->ownPG);
  float* own_g = d ? c->ownGD : c->ownGG;
  const int64_t n = d ? c->dl.total : c->gl.total;
  (d ? c->gD : c->gG) = grads_dev ? grads_dev : own_g;
  (d ? c->tailD : c->tailG) = grads_dev ? c->tail_sep + (d ? kGradTail : 0) : own_g + n;
  c->G_packed = c->D_packed = false;
  return FG_OK;
}
float* fg_params_ptr(fg_ctx* c, int net) { return !c ? nullptr : net == FG_NET_D ? c->PD : net == FG_NET_G ? c->PG : nullptr; }
float* fg_grads_ptr(fg_ctx* c, int net) { return !c ? nullptr : net == FG_NET_D ? c->gD : net == FG_NET_G ? c->gG : nullptr; }

int fg_set_adam_state(fg_ctx* c, int net, const float* m, const float* v, int t) {
  ENTER(c);
  float *dm, *dv; int64_t n;
  FG_TRY(net_bufs(c, net, nullptr, nullptr, &dm, &dv, &n));
  if (m) FG_CUDA(cudaMemcpyAsync(dm, m, n * sizeof(float), cudaMemcpyDefault, c->stream));
  if (v) FG_CUDA(cudaMemcpyAsync(dv, v, n * sizeof(float), cudaMemcpyDefault, c->stream));
  int* tp = net == FG_NET_D ? &c->dstats->t_D : &c->dstats->t_G;
  FG_CUDA(cudaMemcpyAsync(tp, &t, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int fg_get_adam_state(fg_ctx* c, int net, float* m, float* v, int* t) {
  ENTER(c);
  float *dm, *dv; int64_t n;
  FG_TRY(net_bufs(c, net, nullptr, nullptr, &dm, &dv, &n));
  if (m) FG_TRY(to_user(c, m, dm, n));
  if (v) FG_TRY(to_user(c, v, dv, n));
  if (t) {
    const int* tp = net == FG_NET_D ? &c->dstats->t_D : &c->dstats->t_G;
    FG_CUDA(cudaMemcpyAsync(t, tp, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  return FG_OK;
}
int fg_set_bn_state(fg_ctx* c, const float* src) {
  ENTER(c);
  FG_CUDA(cudaMemcpyAsync(c->bnG, src, 768 * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int fg_get_bn_state(fg_ctx* c, float* dst) {
  ENTER(c);
  return to_user(c, dst, c->bnG, 768);
}

// ---- L-net ------------------------------------------------------------------------------------------
int fg_G_forward(fg_ctx* c, const float* noise, int B, int training, float* images_out) {
  ENTER(c);
  FG_REQUIRE(noise && B >= 1 && B <= c->maxB, "fg_G_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  c->G_packed = false;  // parameters may have been edited through fg_params_ptr()
  const float* nd;
  FG_TRY(to_dev(c, noise, (size_t)B * kNoiseDim, c->in_noiseG, &nd));
  FG_TRY(net_G_forward(c, nd, B, training != 0));
  if (images_out) {
    FG_TRY(k_nhwc_to_nchw(c, c->G_y, c->io_dev, B, c->C, 1024));
    FG_TRY(to_user(c, images_out, c->io_dev, (size_t)B * c->C * 1024));
  }
  return FG_OK;
}
int fg_G_backward(fg_ctx* c, const float* d_images, float* d_noise) {
  ENTER(c);
  FG_REQUIRE(d_images, "fg_G_backward: d_images is null");
  const int B = c->G_B;
  const float* dd;
  FG_TRY(to_dev(c, d_images, (size_t)B * c->C * 1024, c->io_dev, &dd));
  FG_TRY(k_nchw_to_nhwc(c, dd, c->io_dev2, B, c->C, 1024));
  float* dn = nullptr;
  if (d_noise) dn = is_device_ptr(d_noise) ? d_noise : c->in_noiseD;
  FG_TRY(net_G_backward(c, c->io_dev2, dn));
  if (d_noise && dn != d_noise) FG_TRY(to_user(c, d_noise, dn, (size_t)B * kNoiseDim));
  return FG_OK;
}
int fg_D_forward(fg_ctx* c, const float* images, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(c);
  FG_REQUIRE(images && B >= 1 && B <= c->maxB, "fg_D_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  c->D_packed = false;
  fg_hyper h;
  fg_hyper_default(&h);
  const float* xd;
  FG_TRY(to_dev(c, images, (size_t)B * c->C * 1024, c->io_dev, &xd));
  FG_TRY(k_nchw_to_nhwc(c, xd, c->D_x, B, c->C, 1024));
  if (training) {
    if (masks) {
      FG_CUDA(cudaMemcpyAsync(c->D_masks, masks, sizeof(float) * (size_t)B * kMaskPerSample, cudaMemcpyDefault, c->stream));
    } else {
      FG_TRY(k_masks_generate(c, c->D_masks, B, seed, h.p_spatial, h.p_drop));
    }
  }
  FG_TRY(net_D_forward(c, c->D_x, B, training != 0, &h));
  FG_TRY(k_sigmoid_fwd(c, c->D_logit, c->D_out, B));
  if (out) FG_TRY(to_user(c, out, c->D_out, B));
  return FG_OK;
}
int fg_D_backward(fg_ctx* c, const float* d_out, int want_wgrad, float* d_images) {
  ENTER(c);
  FG_REQUIRE(d_out, "fg_D_backward: d_out is null");
  const int B = c->D_B;
  const float* dd;
  FG_TRY(to_dev(c, d_out, B, c->D_targets, &dd));
  FG_TRY(k_sigmoid_grad_mul(c, dd, c->D_out, c->D_dlogit, B));
  FG_TRY(net_D_backward(c, c->D_dlogit, want_wgrad != 0, d_images != nullptr));
  if (d_images) {
    FG_TRY(k_nhwc_to_nchw(c, c->D_dx, c->io_dev, B, c->C, 1024));
    FG_TRY(to_user(c, d_images, c->io_dev, (size_t)B * c->C * 1024));
  }
  return FG_OK;
}
int fg_bce_forward(fg_ctx* c, const float* x, const float* t, int n, float* loss_out) {
  ENTER(c);
  FG_REQUIRE(x && t && loss_out && n > 0 && n <= c->maxB, "fg_bce_forward: bad arguments");
  const float *xd, *td;
  FG_TRY(to_dev(c, x, n, c->io_dev, &xd));
  FG_TRY(to_dev(c, t, n, c->io_dev2, &td));
  FG_TRY(k_bce_fwd(c, xd, td, n, c->D_targets));
  return to_user(c, loss_out, c->D_targets, 1);
}
int fg_bce_backward(fg_ctx* c, const float* x, const float* t, int n, float* dx) {
  ENTER(c);
  FG_REQUIRE(x && t && dx && n > 0 && n <= c->maxB, "fg_bce_backward: bad arguments");
  const float *xd, *td;
  FG_TRY(to_dev(c, x, n, c->io_dev, &xd));
  FG_TRY(to_dev(c, t, n, c->io_dev2, &td));
  FG_TRY(k_bce_bwd(c, xd, td, n, c->D_targets));
  return to_user(c, dx, c->D_targets, n);
}
int fg_optim_step(fg_ctx* c, int net, const fg_hyper* h, float grad_scale) {
  ENTER(c);
  FG_REQUIRE(h && (net == FG_NET_G || net == FG_NET_D), "fg_optim_step: bad arguments");
  // no accuracy information at this level: force the gate open by clearing the history influence
  fg_hyper hh = *h;
  hh.D_maxAcc = 2.0f;
  float* g = net == FG_NET_D ? c->tailD : c->tailG;
  FG_TRY(k_gate_and_prep(c, net, &hh, g, 1, 1.0f));
  return net_optim(c, net, h, grad_scale, false);
}
int fg_adam_step(fg_ctx* c, float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                 float eps, int t, float l1_grad, float l2, float clampv, float grad_scale) {
  ENTER(c);
  FG_REQUIRE(p && g && m && v && n > 0 && t >= 1, "fg_adam_step: bad arguments");
  const double step = (double)lr * sqrt(1.0 - pow((double)beta2, t)) / (1.0 - pow((double)beta1, t));
  return k_adam(c, p, g, m, v, n, beta1, beta2, eps, l1_grad, l2, clampv, grad_scale, nullptr, nullptr, (float)step,
                nullptr);
}

// ---- L-step -----------------------------------------------------------------------------------------
int fg_train_step(fg_ctx* c, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                  const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  ENTER(c);
  FG_REQUIRE(h && real && noise_D && noise_G, "fg_train_step: null input");
  FG_REQUIRE(B >= 4 && B % 2 == 0 && B <= c->maxB, "fg_train_step: batch %d must be even, >= 4 and <= max_batch %d", B,
             c->maxB);
  const float *r, *nd, *ng, *md = nullptr, *mg = nullptr;
  FG_TRY(to_dev(c, real, (size_t)(B / 2) * c->C * 1024, c->in_real, &r));
  FG_TRY(to_dev(c, noise_D, (size_t)(B / 2) * kNoiseDim, c->in_noiseD, &nd));
  FG_TRY(to_dev(c, noise_G, (size_t)B * kNoiseDim, c->in_noiseG, &ng));
  if (masks_D) FG_TRY(to_dev(c, masks_D, (size_t)B * kMaskPerSample, c->in_masksD, &md));
  if (masks_G) FG_TRY(to_dev(c, masks_G, (size_t)B * kMaskPerSample, c->in_masksG, &mg));
  FG_TRY(net_train_step(c, h, B, r, nd, ng, md, mg, seed, true));
  if (stats) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    const DeviceStats& s = *c->hstats;
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

int fg_sample(fg_ctx* c, const float* noise, int N, int chunk, float* images_out) {
  ENTER(c);
  FG_REQUIRE(noise && images_out && N >= 1 && chunk >= 1 && chunk <= c->maxB, "fg_sample: bad arguments (chunk %d, max %d)",
             chunk, c->maxB);
  const bool out_dev = is_device_ptr(images_out);
  const size_t img = (size_t)c->C * 1024;
  c->G_packed = false;
  for (int s = 0; s < N; s += chunk) {
    const int b = std::min(chunk, N - s);
    const float* nd;
    FG_TRY(to_dev(c, noise + (size_t)s * kNoiseDim, (size_t)b * kNoiseDim, c->in_noiseG, &nd));
    // sample.lua never calls :evaluate() => BatchNorm uses the statistics of each chunk (SURVEY 3.4)
    FG_TRY(net_G_forward(c, nd, b, true));
    float* dst = images_out + (size_t)s * img;
    if (out_dev) {
      FG_TRY(k_nhwc_to_nchw(c, c->G_y, dst, b, c->C, 1024));
    } else {
      FG_TRY(k_nhwc_to_nchw(c, c->G_y, c->io_dev, b, c->C, 1024));
      FG_CUDA(cudaMemcpyAsync(dst, c->io_dev, b * img * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
      if (s + chunk < N) FG_CUDA(cudaStreamSynchronize(c->stream));  // io_dev is reused by the next chunk
    }
  }
  if (!out_dev) FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

// ---- helpers ----------------------------------------------------------------------------------------
void* fg_dev_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    fg_set_error("fg_dev_alloc(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  return p;
}
int fg_dev_free(void* p) {
  FG_CUDA(cudaFree(p));
  return FG_OK;
}
void* fg_host_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) {
    fg_set_error("fg_host_alloc_pinned(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  return p;
}
int fg_host_free_pinned(void* p) {
  FG_CUDA(cudaFreeHost(p));
  return FG_OK;
}
int fg_memcpy(fg_ctx* c, void* dst, const void* src, size_t bytes) {
  ENTER(c);
  FG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int64_t fg_kernel_launches(fg_ctx* c) { return c ? c->launches : -1; }

int64_t fg_debug_tensor(fg_ctx* c, const char* name, float* dst, int64_t max_elems) {
  if (!c || !name) return -1;
  cudaSetDevice(c->device);
  struct Ent { const char* n; const float* p; int64_t per; int B; };
  const int gb = c->G_B, db = c->D_B;
  const Ent ents[] = {
      {"G.z0", c->G_z0, 8192, gb}, {"G.h0", c->G_h0, 8192, gb}, {"G.z1", c->G_z1, 65536, gb}, {"G.h1", c->G_h1, 65536, gb},
      {"G.z2", c->G_z2, 131072, gb}, {"G.h2", c->G_h2, 131072, gb}, {"G.z3", c->G_z3, 1024 * c->C, gb},
      {"G.y", c->G_y, 1024 * c->C, gb}, {"G.dz2", c->G_dz2, 131072, gb}, {"G.dz1", c->G_dz1, 65536, gb},
      {"G.dz0", c->G_dz0, 8192, gb}, {"D.z1", c->D_z[0], 65536, db}, {"D.z2", c->D_z[1], 32768, db},
      {"D.z3", c->D_z[2], 16384, db}, {"D.z4", c->D_z[3], 8192, db}, {"D.p4", c->D_p[3], 2048, db},
      {"D.logit", c->D_logit, 1, db}, {"D.out", c->D_out, 1, db}, {"D.dx", c->D_dx, 1024 * c->C, db},
      {"D.masks", c->D_masks, kMaskPerSample, db}, {"G.bn_mean1", c->bn_mean1, 256, 1}, {"G.bn_istd1", c->bn_istd1, 256, 1},
      {"G.bn_mean2", c->bn_mean2, 128, 1}, {"G.bn_istd2", c->bn_istd2, 128, 1},
      {"D.zl1", c->D_zl1, 512, db}, {"D.zl2", c->D_zl2, 512, db},
      {"Dstep.z1", c->keep_D[0], 65536, c->keep_B}, {"Dstep.z2", c->keep_D[1], 32768, c->keep_B},
      {"Dstep.z3", c->keep_D[2], 16384, c->keep_B}, {"Dstep.z4", c->keep_D[3], 8192, c->keep_B},
      {"Dstep.zl1", c->keep_D[4], 512, c->keep_B}, {"Dstep.zl2", c->keep_D[5], 512, c->keep_B},
      {"Dstep.logit", c->keep_D[6], 1, c->keep_B}, {"Dstep.out", c->keep_D[7], 1, c->keep_B}};
  for (const Ent& e : ents)
    if (!strcmp(e.n, name)) {
      const int64_t n = e.per * e.B;
      if (!e.p) {
        fg_set_error("fg_debug_tensor: '%s' has not been produced (option \"debug_keep\" + fg_train_step)", name);
        return -1;
      }
      if (dst) {
        if (n > max_elems) return -2;
        if (to_user(c, dst, e.p, n) != FG_OK) return -3;
      }
      return n;
    }
  fg_set_error("fg_debug_tensor: unknown tensor '%s'", name);
  return -1;
}

int fg_bench_tf32_peak(fg_ctx* c, int iters, double* tflops) {
  ENTER(c);
  FG_REQUIRE(tflops && iters > 0, "fg_bench_tf32_peak: bad arguments");
  return tc_tf32_peak(c, iters, 5, tflops);
}

int fg_event_record(fg_ctx* c, int slot) {
  ENTER(c);
  FG_REQUIRE(slot >= 0 && slot < 16, "fg_event_record: slot out of range");
  if (!c->events[slot]) FG_CUDA(cudaEventCreate(&c->events[slot]));
  FG_CUDA(cudaEventRecord(c->events[slot], c->stream));
  return FG_OK;
}
int fg_event_elapsed_ms(fg_ctx* c, int a, int b, double* ms) {
  ENTER(c);
  FG_REQUIRE(a >= 0 && a < 16 && b >= 0 && b < 16 && ms && c->events[a] && c->events[b], "fg_event_elapsed_ms: bad slots");
  FG_CUDA(cudaEventSynchronize(c->events[b]));
  float f = 0;
  FG_CUDA(cudaEventElapsedTime(&f, c->events[a], c->events[b]));
  *ms = f;
  return FG_OK;
}
int fg_timing_enable(fg_ctx* c, int on) {
  ENTER(c);
  FG_CUDA(cudaStreamSynchronize(c->stream));
  c->timing = on != 0;
  for (auto& kv : c->timers) {
    for (auto& pr : kv.second.pending) {
      cudaEventDestroy(pr.first);
      cudaEventDestroy(pr.second);
    }
    kv.second = TimerRec();
  }
  return FG_OK;
}
int fg_timing_get(fg_ctx* c, const char* name, double* ms_total, int64_t* launches) {
  ENTER(c);
  FG_CUDA(cudaStreamSynchronize(c->stream));
  double tot = 0;
  int64_t cnt = 0;
  const size_t len = strlen(name);
  for (auto& kv : c->timers) {
    // prefix match ("G.C2" sums fwd+dgrad+wgrad); "*" matches everything
    if (strcmp(name, "*") != 0 && kv.first.compare(0, len, name) != 0) continue;
    TimerRec& r = kv.second;
    for (auto& pr : r.pending) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) {
        r.ms += ms;
        r.launches++;
      }
      cudaEventDestroy(pr.first);
      cudaEventDestroy(pr.second);
    }
    r.pending.clear();
    tot += r.ms;
    cnt += r.launches;
  }
  if (ms_total) *ms_total = tot;
  if (launches) *launches = cnt;
  return FG_OK;
}

}  // extern "C"
