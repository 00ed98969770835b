// C ABI of libfg_b200.so (include/fg_b200.h).  Thin: argument checking, host/device pointer
// classification, NCHW<->NHWC at the boundary, then nets.cu / kernels.
#include <cstdarg>
#include <cstdlib>
#include <cstring>

#include "convl.h"
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

bool fg_is_dev(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
int fg_to_dev(fg_ctx* c, const float* p, size_t n, float* staging, const float** out) {
  if (fg_is_dev(p)) {
    *out = p;
    return FG_OK;
  }
  FG_CUDA(cudaMemcpyAsync(staging, p, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  *out = staging;
  return FG_OK;
}
int fg_to_user(fg_ctx* c, float* dst, const float* src_dev, size_t n) {
  if (dst == src_dev) return FG_OK;
  const bool dev = fg_is_dev(dst);
  FG_CUDA(cudaMemcpyAsync(dst, src_dev, n * sizeof(float), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                          c->stream));
  if (!dev) FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int64_t debug_tensor_copy(fg_ctx* c, const char* what, const DebugTensor* ents, size_t n_ents, const char* name, float* dst,
                          int64_t max_elems) {
  for (size_t i = 0; i < n_ents; ++i) {
    const DebugTensor& e = ents[i];
    if (strcmp(e.name, name)) continue;
    const int64_t n = e.per * e.B;
    if (!e.p) {
      fg_set_error("%s: '%s' has not been produced (Dstep.*: option \"debug_keep\" + a train step)", what, name);
      return -1;
    }
    if (dst) {
      if (n > max_elems) return -2;
      if (fg_to_user(c, dst, e.p, n) != FG_OK) return -3;
    }
    return n;
  }
  fg_set_error("%s: unknown tensor '%s'", what, name);
  return -1;
}

namespace {
// d_iters D iterations + g_iters G iterations of the loop body on inputs stacked per iteration, for the entry `what`
int train_step_iters(fg_ctx* c, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                     const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                     fg_step_stats* stats) {
  ENTER(c);
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h && real && noise_D && noise_G));
  const size_t nd = d_iters, ng = g_iters, Bh = B / 2, M = c->maxB, img = (size_t)c->C * 1024;
  IterStage& s = c->iter_stage;
  const float *r, *zd, *zg, *md, *mg;
  FG_TRY(s.in(c, c->allocs, 0, real, nd * Bh * img, nd * M / 2 * img, &r));
  FG_TRY(s.in(c, c->allocs, 1, noise_D, nd * Bh * kNoiseDim, nd * M / 2 * kNoiseDim, &zd));
  FG_TRY(s.in(c, c->allocs, 2, noise_G, ng * B * kNoiseDim, ng * M * kNoiseDim, &zg));
  FG_TRY(s.in(c, c->allocs, 3, masks_D, nd * B * kMaskPerSample, nd * M * kMaskPerSample, &md));
  FG_TRY(s.in(c, c->allocs, 4, masks_G, ng * B * kMaskPerSample, ng * M * kMaskPerSample, &mg));
  NetStep st(c, h, B, r, zd, zg);
  return pair_train_step(st, d_iters, g_iters, md, mg, seed, {r, zd, zg, md, mg, nullptr}, nullptr, stats);
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
    c->net.G_packed = c->net.D_packed = false;
    return FG_OK;
  }
  if (!strcmp(key, "params_dirty")) {
    c->net.G_packed = c->net.D_packed = false;
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
    c->net.G_packed = c->net.D_packed = false;
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
  if (!strcmp(key, "bwd_merge")) {  // see fg_ctx::bwd_merge
    FG_REQUIRE(v >= 0 && v <= 2, "bwd_merge must be 0 (two launches), 1 (merged where it is faster) or 2 (merged where possible)");
    c->bwd_merge = (int)v;
    return FG_OK;
  }
  if (!strcmp(key, "bwd_merge_ctas")) {
    FG_REQUIRE(v >= 0, "bwd_merge_ctas must be >= 0 (0: one CTA per SM)");
    c->bwd_merge_ctas = v > (1 << 20) ? (1 << 20) : (int)v;
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
  if (!strcmp(key, "bwd_merge")) return c->bwd_merge;
  if (!strcmp(key, "bwd_merge_ctas")) return c->bwd_merge_ctas;
  if (!strcmp(key, "optimizer_D")) return c->opt_D;
  if (!strcmp(key, "optimizer_G")) return c->opt_G;
  if (!strcmp(key, "last_conv_kind")) return c->last_conv_kind;
  if (!strcmp(key, "last_conv_tile_m")) return c->last_conv_tile_m;
  if (!strcmp(key, "last_conv_tile_n")) return c->last_conv_tile_n;
  if (!strcmp(key, "last_conv_format")) return c->last_conv_format;
  if (!strcmp(key, "last_conv_splits")) return c->last_conv_splits;
  return -1;
}

int64_t fg_param_count(int net, int channels) {
  if (channels != 1 && channels != 3) return -1;
  return net == FG_NET_G ? make_g_layout(channels, 32).total : net == FG_NET_D ? make_d_layout(channels).total : -1;
}
int fg_set_params(fg_ctx* c, int net, const float* src) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_set_params(c, c->net, net, src);
}
int fg_get_params(fg_ctx* c, int net, float* dst) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_get_params(c, c->net, net, dst);
}
int fg_get_grads(fg_ctx* c, int net, float* dst) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_get_grads(c, c->net, net, dst);
}
int fg_zero_grads(fg_ctx* c, int net) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_zero_grads(c, c->net, net);
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
  NetPair& np = c->net;
  const bool d = net == FG_NET_D;
  (d ? np.PD : np.PG) = params_dev ? params_dev : (d ? c->ownPD : c->ownPG);
  float* own_g = d ? c->ownGD : c->ownGG;
  const int64_t n = d ? np.nD : np.nG;
  (d ? np.gD : np.gG) = grads_dev ? grads_dev : own_g;
  (d ? np.tailD : np.tailG) = grads_dev ? c->tail_sep + (d ? kGradTail : 0) : own_g + n;
  np.G_packed = np.D_packed = false;
  return FG_OK;
}
float* fg_params_ptr(fg_ctx* c, int net) { return !c ? nullptr : net == FG_NET_D ? c->net.PD : net == FG_NET_G ? c->net.PG : nullptr; }
float* fg_grads_ptr(fg_ctx* c, int net) { return !c ? nullptr : net == FG_NET_D ? c->net.gD : net == FG_NET_G ? c->net.gG : nullptr; }

int fg_set_adam_state(fg_ctx* c, int net, const float* m, const float* v, int t) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_set_adam_state(c, c->net, net, m, v, t);
}
int fg_get_adam_state(fg_ctx* c, int net, float* m, float* v, int* t) {
  ENTER(c);
  FG_REQUIRE(net == FG_NET_G || net == FG_NET_D, "net must be FG_NET_G or FG_NET_D");
  return pair_get_adam_state(c, c->net, net, m, v, t);
}
int fg_set_bn_state(fg_ctx* c, const float* src) {
  ENTER(c);
  return pair_set_bn_state(c, c->net, src);
}
int fg_get_bn_state(fg_ctx* c, float* dst) {
  ENTER(c);
  return pair_get_bn_state(c, c->net, dst);
}

// ---- L-net ------------------------------------------------------------------------------------------
int fg_G_forward(fg_ctx* c, const float* noise, int B, int training, float* images_out) {
  ENTER(c);
  FG_REQUIRE(noise && B >= 1 && B <= c->maxB, "fg_G_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  c->net.G_packed = false;  // parameters may have been edited through fg_params_ptr()
  const float* nd;
  FG_TRY(fg_to_dev(c, noise, (size_t)B * kNoiseDim, c->in_noiseG, &nd));
  FG_TRY(gen_forward(c->env, c->G, c->net, nd, B, training != 0));
  if (images_out) {
    FG_TRY(k_nhwc_to_nchw(c, c->G.y, c->io_dev, B, c->C, 1024));
    FG_TRY(fg_to_user(c, images_out, c->io_dev, (size_t)B * c->C * 1024));
  }
  return FG_OK;
}
int fg_G_backward(fg_ctx* c, const float* d_images, float* d_noise) {
  ENTER(c);
  FG_REQUIRE(d_images, "fg_G_backward: d_images is null");
  const int B = c->G.B;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_images, (size_t)B * c->C * 1024, c->io_dev, &dd));
  FG_TRY(k_nchw_to_nhwc(c, dd, c->io_dev2, B, c->C, 1024));
  float* dn = nullptr;
  if (d_noise) dn = fg_is_dev(d_noise) ? d_noise : c->in_noiseD;
  FG_TRY(gen_backward(c->env, c->G, c->net, c->io_dev2, dn));
  if (d_noise && dn != d_noise) FG_TRY(fg_to_user(c, d_noise, dn, (size_t)B * kNoiseDim));
  return FG_OK;
}
int fg_D_forward(fg_ctx* c, const float* images, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(c);
  FG_REQUIRE(images && B >= 1 && B <= c->maxB, "fg_D_forward: bad arguments (B=%d, max %d)", B, c->maxB);
  c->net.D_packed = false;
  fg_hyper h;
  fg_hyper_default(&h);
  const float* xd;
  FG_TRY(fg_to_dev(c, images, (size_t)B * c->C * 1024, c->io_dev, &xd));
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
  if (out) FG_TRY(fg_to_user(c, out, c->D_out, B));
  return FG_OK;
}
int fg_D_backward(fg_ctx* c, const float* d_out, int want_wgrad, float* d_images) {
  ENTER(c);
  FG_REQUIRE(d_out, "fg_D_backward: d_out is null");
  const int B = c->D_B;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_out, B, c->D_targets, &dd));
  FG_TRY(k_sigmoid_grad_mul(c, dd, c->D_out, c->D_dlogit, B));
  FG_TRY(net_D_backward(c, c->D_dlogit, want_wgrad != 0, d_images != nullptr));
  if (d_images) {
    FG_TRY(k_nhwc_to_nchw(c, c->D_dx, c->io_dev, B, c->C, 1024));
    FG_TRY(fg_to_user(c, d_images, c->io_dev, (size_t)B * c->C * 1024));
  }
  return FG_OK;
}
int fg_bce_forward(fg_ctx* c, const float* x, const float* t, int n, float* loss_out) {
  ENTER(c);
  FG_REQUIRE(x && t && loss_out && n > 0 && n <= c->maxB, "fg_bce_forward: bad arguments");
  const float *xd, *td;
  FG_TRY(fg_to_dev(c, x, n, c->io_dev, &xd));
  FG_TRY(fg_to_dev(c, t, n, c->io_dev2, &td));
  FG_TRY(k_bce_fwd(c, xd, td, n, c->D_targets));
  return fg_to_user(c, loss_out, c->D_targets, 1);
}
int fg_bce_backward(fg_ctx* c, const float* x, const float* t, int n, float* dx) {
  ENTER(c);
  FG_REQUIRE(x && t && dx && n > 0 && n <= c->maxB, "fg_bce_backward: bad arguments");
  const float *xd, *td;
  FG_TRY(fg_to_dev(c, x, n, c->io_dev, &xd));
  FG_TRY(fg_to_dev(c, t, n, c->io_dev2, &td));
  FG_TRY(k_bce_bwd(c, xd, td, n, c->D_targets));
  return fg_to_user(c, dx, c->D_targets, n);
}
int fg_optim_step(fg_ctx* c, int net, const fg_hyper* h, float grad_scale) {
  ENTER(c);
  FG_REQUIRE(h && (net == FG_NET_G || net == FG_NET_D), "fg_optim_step: bad arguments");
  // no accuracy information at this level: no gate, and the fused steps' accuracy history is not touched
  FG_TRY(k_optim_prep(c, c->net.dstats, net, h));
  return pair_optim(c, c->net, net, h, grad_scale);
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
  return train_step_iters(c, "fg_train_step", h, B, 1, 1, real, noise_D, noise_G, masks_D, masks_G, seed, stats);
}
int fg_train_step_iters(fg_ctx* c, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                        const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                        fg_step_stats* stats) {
  return train_step_iters(c, "fg_train_step_iters", h, B, d_iters, g_iters, real, noise_D, noise_G, masks_D, masks_G, seed,
                          stats);
}

int fg_sample(fg_ctx* c, const float* noise, int N, int chunk, float* images_out) {
  ENTER(c);
  FG_REQUIRE(noise && images_out && N >= 1 && chunk >= 1 && chunk <= c->maxB, "fg_sample: bad arguments (chunk %d, max %d)",
             chunk, c->maxB);
  const bool out_dev = fg_is_dev(images_out);
  const size_t img = (size_t)c->C * 1024;
  c->net.G_packed = false;
  for (int s = 0; s < N; s += chunk) {
    const int b = std::min(chunk, N - s);
    const float* nd;
    FG_TRY(fg_to_dev(c, noise + (size_t)s * kNoiseDim, (size_t)b * kNoiseDim, c->in_noiseG, &nd));
    // sample.lua never calls :evaluate() => BatchNorm uses the statistics of each chunk (SURVEY 3.4)
    FG_TRY(gen_forward(c->env, c->G, c->net, nd, b, true));
    float* dst = images_out + (size_t)s * img;
    if (out_dev) {
      FG_TRY(k_nhwc_to_nchw(c, c->G.y, dst, b, c->C, 1024));
    } else {
      FG_TRY(k_nhwc_to_nchw(c, c->G.y, c->io_dev, b, c->C, 1024));
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
  const int db = c->D_B;
  std::vector<DebugTensor> ents = {
      {"D.z1", c->D_z[0], 65536, db}, {"D.z2", c->D_z[1], 32768, db}, {"D.z3", c->D_z[2], 16384, db},
      {"D.z4", c->D_z[3], 8192, db}, {"D.p4", c->D_p[3], 2048, db}, {"D.logit", c->D_logit, 1, db},
      {"D.out", c->D_out, 1, db}, {"D.dx", c->D_dx, 1024 * c->C, db}, {"D.masks", c->D_masks, kMaskPerSample, db},
      {"D.zl1", c->D_zl1, 512, db}, {"D.zl2", c->D_zl2, 512, db}};
  pair_keep_rows(c->net, ents);
  gen_debug_rows(c->G, ents);
  return debug_tensor_copy(c, "fg_debug_tensor", ents.data(), ents.size(), name, dst, max_elems);
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
