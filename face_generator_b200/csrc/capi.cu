// C ABI of libfg_b200.so (include/fg_b200.h): the context (fg_ctx: its stream, options and shared workspaces), the
// last error, host/device pointer classification, events and timers.  The entry points of each net sit next to its code
// (nets.cu, nets_s16.cu, nets_c2f.cu, ...).
#include <algorithm>
#include <cstdarg>
#include <cstdlib>
#include <cstring>

#include "fg_internal.h"
#include "k_conv_tc.h"
#include "ups_gan.h"

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
      fg_set_error("%s: '%s' has not been produced (Dstep.* / Dbwd.*: option \"debug_keep\" + a train step / D backward)", what, name);
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
// the workspaces every net on the context shares
int ctx_alloc(fg_ctx* c) {
  const size_t B = c->maxB, C = c->C;
  auto dalloc = [c](auto** p, size_t n) { return fg_dalloc(c, c->allocs, reinterpret_cast<float**>(p), n); };
  FG_TRY(dalloc(&c->lop_sx, 2));
  FG_TRY(dalloc(&c->lop_sy, 2));
  FG_TRY(dalloc(&c->seed_dev, 2 * kMaxIters));  // one stream root per iteration (k_seed_roots)
  c->splitk_ws_elems = (size_t)c->sm_count * 4 * 128 * 128;  // >= splits x output of every split-K weight gradient
  FG_TRY(dalloc(&c->splitk_ws, c->splitk_ws_elems));
  c->red_ws_elems = (size_t)4 << 20;  // >= blocks x partials of every ordered reduction (checked at each launch)
  FG_TRY(dalloc(&c->red_ws, 2 * c->red_ws_elems));
  FG_TRY(dalloc(&c->red_ws_opt, 2 * kOptRedRows));
  FG_TRY(dalloc(&c->red_ticket, 2));  // zeroed; every ordered reduction resets its ticket
  FG_TRY(dalloc(&c->bwd_claim, 1));
  FG_TRY(dalloc(&c->small_ws, (size_t)kSmallMaxParts * 9 * 4 * 128));
  FG_TRY(dalloc(&c->bn_acc, 4 * 256 * 2));  // doubles
  FG_TRY(dalloc(&c->bn_slice_acc, 32 * 4 * 256 * 2 + 64));  // doubles + tickets (zero-initialised)
  FG_TRY(dalloc(&c->bn_parts, B * 3072));  // G.C2: 8 tiles/image x 3 x 128 ch; G.C1: 2 tiles/image x 3 x 256 ch
  fg_ctx::Workspaces& s = c->side_ws;  // the same for a generator forward on side_stream
  FG_TRY(dalloc(&s.red_ws, 2 * c->red_ws_elems));
  FG_TRY(dalloc(&s.red_ticket, 2));
  FG_TRY(dalloc(&s.bn_acc, 4 * 256 * 2));
  FG_TRY(dalloc(&s.bn_slice_acc, 32 * 4 * 256 * 2 + 64));
  FG_TRY(dalloc(&s.bn_parts, B * 3072));
  fg_ctx::WgradWorkspaces& w = c->wgrad_ws;  // and for the weight gradients on wgrad_stream
  FG_TRY(dalloc(&w.splitk_ws, c->splitk_ws_elems));
  FG_TRY(dalloc(&w.red_ws, 2 * c->red_ws_elems));
  FG_TRY(dalloc(&w.red_ticket, 2));
  FG_TRY(dalloc(&w.small_ws, (size_t)kSmallMaxParts * 9 * 4 * 128));
  c->io_dev_elems = std::max<size_t>(B * 1024 * C, B * kMaskPerSample);
  return dalloc(&c->io_dev, c->io_dev_elems);
}
void ctx_free(fg_ctx* c) {
  for (void* p : c->allocs) cudaFree(p);
  c->allocs.clear();
  for (int i = 0; i < 8; ++i)
    if (c->scratch[i]) cudaFree(c->scratch[i]);
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
  return fg_create_disc(out, device, max_batch, channels, FG_DISC_D32B);
}

int64_t fg_disc_param_count(int disc, int channels) {
  if (channels != 1 && channels != 3) return -1;
  if (disc == FG_DISC_D32B) return fg_param_count(FG_NET_D, channels);
  return dbr_param_count(disc, channels);
}
int fg_disc_mask_per_sample(int disc) {
  if (disc == FG_DISC_D32B) return kMaskPerSample;
  return dbr_mask_per_sample(disc);
}
int fg_disc_side(int disc) {
  if (disc == FG_DISC_D32B) return 32;
  return dbr_side(disc);
}

int fg_create_disc(fg_ctx** out, int device, int max_batch, int channels, int disc) {
  if (!out) { fg_set_error("fg_create: out is null"); return FG_ERR_INVALID; }
  *out = nullptr;
  if (disc == FG_DISC_DEFAULT) disc = FG_DISC_D32B;
  FG_REQUIRE(fg_disc_side(disc), "fg_create_disc: unknown discriminator %d", disc);
  if (fg_disc_side(disc) != 32) {
    fg_set_error("fg_create_disc: discriminator %d is a 16x16 net; the 32x32 nets take FG_DISC_D32B or FG_DISC_D32", disc);
    return FG_ERR_UNSUPPORTED;
  }
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
  int r = ctx_alloc(c);
  if (r == FG_OK) r = net32_alloc(c, disc);
  if (r == FG_OK) r = tc_init(c);
  if (r != FG_OK) {
    net32_free(c);
    ctx_free(c);
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
  for (cudaStream_t s : {c->comm_stream, c->side_stream, c->wgrad_stream})
    if (s) {
      cudaStreamSynchronize(s);
      cudaStreamDestroy(s);
    }
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  for (cudaEvent_t e : {c->ev_wfork, c->ev_wjoin})
    if (e) cudaEventDestroy(e);
  tc_destroy(c);
  net32_free(c);
  jpeg_enc_scratch_free(c->jpeg_enc);
  ctx_free(c);
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
    return FG_OK;
  }
  if (!strcmp(key, "params_dirty")) {
    NetPair& p = net32_pair(c);
    p.G_pack = p.D_pack = -1;
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
  if (!strcmp(key, "bwd_streams")) {  // see fg_ctx::bwd_streams
    FG_REQUIRE(v == 0 || v == 1, "bwd_streams must be 0 (one stream) or 1 (weight gradients on a stream of their own)");
    c->bwd_streams = (int)v;
    return FG_OK;
  }
  if (!strcmp(key, "bwd_merge_ctas")) {
    FG_REQUIRE(v >= 0, "bwd_merge_ctas must be >= 0 (0: one CTA per SM)");
    c->bwd_merge_ctas = v > (1 << 20) ? (1 << 20) : (int)v;
    return FG_OK;
  }
  if (!strcmp(key, "jpeg_route")) {  // tests only: 0 (default) by file size, 1 one CTA per file, 2 many CTAs per file
    FG_REQUIRE(v >= 0 && v <= 2, "jpeg_route must be 0 (by file size), 1 (one CTA per file) or 2 (many CTAs per file)");
    c->jpeg_route = (int)v;
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
  if (!strcmp(key, "jpeg_route")) return c->jpeg_route;
  if (!strcmp(key, "channels")) return c->C;
  if (!strcmp(key, "sm_count")) return c->sm_count;
  if (!strcmp(key, "bn_epilogue")) return c->bn_epilogue;
  if (!strcmp(key, "edge_impl")) return c->edge_impl;
  if (!strcmp(key, "mma_f16")) return c->mma_f16;
  if (!strcmp(key, "dp_overlap")) return c->dp_overlap;
  if (!strcmp(key, "use_graph")) return c->use_graph;
  if (!strcmp(key, "bwd_merge")) return c->bwd_merge;
  if (!strcmp(key, "bwd_merge_ctas")) return c->bwd_merge_ctas;
  if (!strcmp(key, "bwd_streams")) return c->bwd_streams;
  if (!strcmp(key, "optimizer_D")) return c->opt_D;
  if (!strcmp(key, "optimizer_G")) return c->opt_G;
  if (!strcmp(key, "last_conv_kind")) return c->last_conv_kind;
  if (!strcmp(key, "last_conv_tile_m")) return c->last_conv_tile_m;
  if (!strcmp(key, "last_conv_tile_n")) return c->last_conv_tile_n;
  if (!strcmp(key, "last_conv_format")) return c->last_conv_format;
  if (!strcmp(key, "last_conv_splits")) return c->last_conv_splits;
  if (!strcmp(key, "step_graph_launches")) return c->graph_launches;
  return -1;
}

int fg_adam_step(fg_ctx* c, float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                 float eps, int t, float l1_grad, float l2, float clampv, float grad_scale) {
  ENTER(c);
  FG_REQUIRE(p && g && m && v && n > 0 && t >= 1, "fg_adam_step: bad arguments");
  const double step = (double)lr * sqrt(1.0 - pow((double)beta2, t)) / (1.0 - pow((double)beta1, t));
  return k_adam(c, p, g, m, v, n, beta1, beta2, eps, l1_grad, l2, clampv, grad_scale, nullptr, nullptr, (float)step,
                nullptr);
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
