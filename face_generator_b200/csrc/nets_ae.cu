// The autoencoder of train_autoencoder.lua and the batch step that trains it:
//   MODEL_AE = View(I) Linear(I, 512) ReLU Linear(512, d) Tanh Dropout(0.5) Linear(d, 256) ReLU Linear(256, I) Sigmoid
//              View(1, S, S)                      I = S^2 (grayscale), d = --noiseDim          train_autoencoder.lua:80-92
//   step = fevalAE (nn.AbsCriterion against the inputs, L1 / L2 penalty gradients) + optim.adam with an empty config,
//          no gradient clamp                                                                                  :178-209
// An image [1][S][S] already is its View(I) row, so every tensor here is [B][features] and nothing is transposed.
// The four Linear layers are ConvL layers (convl.h) and the optimizer is k_optim_update; this file adds the
// elementwise layers, each one pass over its tensor that also reduces the FP16 max|output| its consumer scales by.
//
// nn.AbsCriterion's gradient is +1/n where y >= t (a tie counts as positive) and -1/n elsewhere -- the THNN rule, as
// recalled (third-party code, not part of the reference tree).  nn.ReLU passes the gradient where z > 0.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "convl.h"
#include "fg_internal.h"
#include "k_f16split.cuh"
#include "k_ordered.cuh"
#include "k_stream.cuh"

namespace {
constexpr int kH1 = 512, kH3 = 256;
constexpr uint64_t kKindMask = 0;  // the random stream (step seed, kind) of the dropout keep flags

__global__ void ae_relu_fwd_kernel(const float* __restrict__ z, float* __restrict__ h, int64_t n, unsigned* __restrict__ amax) {
  float am = 0.f;
  GRID_STRIDE(i, n) {
    const float o = fmaxf(z[i], 0.f);
    h[i] = o;
    am = fmaxf(am, finite_abs(o));
  }
  amax_commit(amax, am);
}
// dz = dh [z > 0]
__global__ void ae_relu_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ z, float* __restrict__ dz, int64_t n,
                                   unsigned* __restrict__ amax) {
  float am = 0.f;
  GRID_STRIDE(i, n) {
    const float o = z[i] > 0.f ? dh[i] : 0.f;
    dz[i] = o;
    am = fmaxf(am, finite_abs(o));
  }
  amax_commit(amax, am);
}
// code = tanh(z); h = code * keep * scale (h may be null).  The keep flags are the given ones (masks_in), or drawn with
// probability 1 - p on the stream (*seed_dev, kKindMask), or all 1 (both null: evaluation, scale 1); flags_out (may be
// null) receives the flags used.
__global__ void ae_tanh_dropout_fwd_kernel(const float* __restrict__ z, const float* __restrict__ masks_in,
                                           const uint64_t* __restrict__ seed_dev, float p, float scale,
                                           float* __restrict__ code, float* __restrict__ h, float* __restrict__ flags_out,
                                           int64_t n, unsigned* __restrict__ amax) {
  const uint64_t root = seed_dev ? *seed_dev : 0;
  float am = 0.f;
  GRID_STRIDE(i, n) {
    const float cv = tanhf(z[i]);
    float keep = 1.f;
    if (masks_in) keep = masks_in[i];
    else if (seed_dev) keep = (float)(stream_bits(root, kKindMask, i) >> 40) * (1.0f / 16777216.0f) >= p ? 1.f : 0.f;
    code[i] = cv;
    if (flags_out) flags_out[i] = keep;
    const float o = cv * keep * scale;
    if (h) h[i] = o;
    am = fmaxf(am, finite_abs(o));
  }
  amax_commit(amax, am);
}
// dz = dh * keep * scale * (1 - code^2); masks null: keep * scale = 1
__global__ void ae_tanh_dropout_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ masks, float scale,
                                           const float* __restrict__ code, float* __restrict__ dz, int64_t n,
                                           unsigned* __restrict__ amax) {
  float am = 0.f;
  GRID_STRIDE(i, n) {
    const float cv = code[i];
    float d = dh[i];
    if (masks) d *= masks[i] * scale;
    const float o = d * (1.f - cv * cv);
    dz[i] = o;
    am = fmaxf(am, finite_abs(o));
  }
  amax_commit(amax, am);
}
// nn.AbsCriterion (size-averaged) against targets t, after nn.Sigmoid when SIGMOID (z: logits, y: its output) or on z
// itself: *loss = mean |y - t|, summed in block order; dz = the criterion's gradient, through Sigmoid.backward as the
// reference composes it, (+-1/n) (1 - y) y, so that a sigmoid saturated to exactly 0 or 1 passes exactly 0.
// y, dz and loss may each be null.
template <bool SIGMOID>
__global__ void __launch_bounds__(256) ae_abs_kernel(const float* __restrict__ z, const float* __restrict__ t,
                                                     float* __restrict__ y, float* __restrict__ dz, int64_t n,
                                                     double* __restrict__ ws, unsigned* __restrict__ ticket,
                                                     float* __restrict__ loss, unsigned* __restrict__ amax) {
  const float invN = 1.0f / (float)n;
  double s = 0;
  float am = 0.f;
  GRID_STRIDE(i, n) {
    const float yy = SIGMOID ? 1.0f / (1.0f + expf(-z[i])) : z[i];
    const float e = yy - t[i];
    if (SIGMOID && y) y[i] = yy;
    s += (double)fabsf(e);
    float g = e >= 0.f ? invN : -invN;
    if (SIGMOID) g = g * (1.0f - yy) * yy;
    if (dz) dz[i] = g;
    am = fmaxf(am, finite_abs(g));
  }
  amax_commit(amax, am);
  if (!loss) return;
  s = block_sum256(s);
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
  if (ordered_last_block(ticket)) {
    if (threadIdx.x == 0) *loss = (float)(ordered_sum(ws, gridDim.x, 1, 0) / (double)n);
    ordered_release(ticket);
  }
}

struct AeStats {  // device; mirrored to fg_ae_stats
  float loss;
  int t;
  float step;  // the Adam step size of the update that follows (k_adam_prep)
};
}  // namespace

int k_relu_fwd(fg_ctx* c, const float* z, float* h, int64_t n) {
  ae_relu_fwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(z, h, n, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_relu_bwd(fg_ctx* c, const float* dh, const float* z, float* dz, int64_t n) {
  ae_relu_bwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(dh, z, dz, n, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_tanh_dropout_fwd(fg_ctx* c, const float* z, const float* masks_in, const uint64_t* seed_dev, float p, float* code, float* h,
                       float* flags_out, int64_t n) {
  const float scale = masks_in || seed_dev ? 1.0f / (1.0f - p) : 1.f;
  ae_tanh_dropout_fwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(z, masks_in, seed_dev, p, scale, code, h, flags_out, n,
                                                                      take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_tanh_dropout_bwd(fg_ctx* c, const float* dh, const float* masks, float p, const float* code, float* dz, int64_t n) {
  ae_tanh_dropout_bwd_kernel<<<grid_for(n, 256), 256, 0, c->stream>>>(dh, masks, 1.0f / (1.0f - p), code, dz, n, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}
int k_abs_criterion(fg_ctx* c, bool sigmoid, const float* z, const float* t, float* y, float* dz, int64_t n, float* loss) {
  const int grid = grid_for(n, 256, c->sm_count * 4);
  FG_TRY(red_check(c, grid, 1));
  if (sigmoid) ae_abs_kernel<true><<<grid, 256, 0, c->stream>>>(z, t, y, dz, n, c->red_ws, c->red_ticket, loss, take_amax(c));
  else ae_abs_kernel<false><<<grid, 256, 0, c->stream>>>(z, t, y, dz, n, c->red_ws, c->red_ticket, loss, take_amax(c));
  LAUNCH_CHECK(c);
  return FG_OK;
}

struct fg_ae {
  fg_ctx* c = nullptr;
  int S = 32, I = 1024, d = 256, maxB = 0;
  NetPair net;  // the G half only: parameters, gradients, Adam moments and the step graphs
  ConvL L[4];
  ScalePairs pairs;  // x and dY of the four layers, and the env's shared dY pair
  AeStats* dstats = nullptr;
  AeStats* hstats = nullptr;  // pinned mirror
  // activations and gradients of the last forward / backward, [B][features]
  const float* x = nullptr;  // the input rows: xbuf, or the caller's device images during a train step
  float *xbuf = nullptr, *z1 = nullptr, *h1 = nullptr, *z2 = nullptr, *code = nullptr, *h2 = nullptr, *z3 = nullptr,
        *h3 = nullptr, *z4 = nullptr, *y = nullptr, *masks = nullptr;
  float *dz4 = nullptr, *dz3 = nullptr, *dz2 = nullptr, *dz1 = nullptr, *dh = nullptr;
  float *in_img = nullptr, *in_masks = nullptr;  // staging of host inputs
  int B = 0, grad_B = 0;
  bool train = true, valid = false;
  float p_drop = 0.5f;  // Dropout probability of the last training forward
  std::vector<void*> allocs;
  ConvLEnv env;
};

namespace {
// the Linear packs take any width; a multiple of 8 keeps every row of every operand 32-byte aligned, and a multiple of 64
// puts Linear(512, d) and Linear(d, 256) on the tensor cores (otherwise those two run on the fp32 FFMA kernels)
bool ae_shape_ok(int size, int d) { return (size == 16 || size == 32) && d >= 8 && d <= 1024 && d % 8 == 0; }

// getParameters() order: [L1W L1b L2W L2b L3W L3b L4W L4b], weights [out][in]
int64_t make_ae_layout(ConvL* L, int I, int d) {
  static const char* tf[4] = {"ae.L1.fwd", "ae.L2.fwd", "ae.L3.fwd", "ae.L4.fwd"};
  static const char* td[4] = {"ae.L1.dgrad", "ae.L2.dgrad", "ae.L3.dgrad", "ae.L4.dgrad"};
  static const char* tw[4] = {"ae.L1.wgrad", "ae.L2.wgrad", "ae.L3.wgrad", "ae.L4.wgrad"};
  const int ci[4] = {I, kH1, d, kH3}, co[4] = {kH1, d, kH3, I};
  int64_t o = 0;
  for (int i = 0; i < 4; ++i) {
    L[i].Cin = ci[i]; L[i].Cout = co[i]; L[i].k = 1; L[i].H = 1;
    L[i].w_off = o; o += (int64_t)co[i] * ci[i];
    L[i].b_off = o; o += co[i];
    L[i].tf = tf[i]; L[i].td = td[i]; L[i].tw = tw[i];
  }
  L[0].need_dgrad = false;  // nothing in front of the input
  return o;
}

int dalloc(fg_ae* n, float** p, size_t elems) { return fg_dalloc(n->c, n->allocs, p, elems); }

int ae_alloc(fg_ae* n) {
  fg_ctx* c = n->c;
  const size_t B = n->maxB, I = n->I, d = n->d;
  n->env.c = c;
  n->env.maxB = n->maxB;
  n->env.allocs = &n->allocs;
  const int64_t np = make_ae_layout(n->L, n->I, n->d);
  NetPair& p = n->net;
  p.nG = np;
  FG_TRY(dalloc(n, &p.PG, np));
  FG_TRY(dalloc(n, &p.gG, np + kGradTail));
  p.tailG = p.gG + np;
  FG_TRY(dalloc(n, &p.mG, np));
  FG_TRY(dalloc(n, &p.vG, np));
  float* tmp = nullptr;
  FG_TRY(dalloc(n, &tmp, (sizeof(AeStats) + 3) / 4));
  n->dstats = (AeStats*)tmp;
  FG_CUDA(cudaMallocHost((void**)&n->hstats, sizeof(AeStats)));
  memset(n->hstats, 0, sizeof(AeStats));
  FG_TRY(n->pairs.alloc(c, n->allocs, 9));
  FG_TRY(n->pairs.take(&n->env.dy.s));
  for (ConvL& L : n->L) {
    FG_TRY(n->pairs.take(&L.x.s));
    FG_TRY(n->pairs.take(&L.sdy));
    FG_TRY(convl_alloc(n->env, L));
  }
  for (auto [q, per] : {std::pair<float**, size_t>{&n->xbuf, I}, {&n->z1, kH1}, {&n->h1, kH1}, {&n->z2, d}, {&n->code, d},
                        {&n->h2, d}, {&n->z3, kH3}, {&n->h3, kH3}, {&n->z4, I}, {&n->y, I}, {&n->masks, d}, {&n->dz4, I},
                        {&n->dz3, kH3}, {&n->dz2, d}, {&n->dz1, kH1}, {&n->dh, std::max<size_t>(kH1, d)}, {&n->in_img, I},
                        {&n->in_masks, d}})
    FG_TRY(dalloc(n, q, B * per));
  // the widest dY split (L4's output or Linear(512, d)'s) and the largest packed weight gradient
  const size_t wide = std::max<size_t>(std::max<size_t>(I, d), kH1);
  FG_TRY(dalloc(n, &n->env.dy.hi, B * wide));
  FG_TRY(dalloc(n, &n->env.dy.lo, B * wide));
  FG_TRY(dalloc(n, &n->env.ws, (size_t)kH1 * std::max(I, d)));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int ae_pack(fg_ae* n) {
  if (n->net.G_pack == pack_key(n->c)) return FG_OK;
  for (ConvL& L : n->L) FG_TRY(convl_pack(n->c, L, n->net.PG));
  n->net.G_pack = pack_key(n->c);
  return FG_OK;
}

// x (device rows [B][I]) -> z4 (logits).  training: Dropout with the given keep flags (device [B][d]) or, when null,
// flags drawn from c->seed_dev; evaluation: identity
int ae_forward(fg_ae* n, const float* x, int B, bool training, const float* masks, float p) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  const float* P = n->net.PG;
  FG_TRY(ae_pack(n));
  n->x = x;
  n->B = B;
  n->train = training;
  n->p_drop = p;
  FG_TRY(n->pairs.reset(c));
  FG_TRY(convl_fwd(e, n->L[0], x, P, n->z1, B));
  {
    AmaxInto am(c, n->L[1].x);
    FG_TRY(k_relu_fwd(c, n->z1, n->h1, (int64_t)B * kH1));
  }
  FG_TRY(convl_fwd(e, n->L[1], n->h1, P, n->z2, B));
  {
    AmaxInto am(c, n->L[2].x);
    FG_TRY(k_tanh_dropout_fwd(c, n->z2, training ? masks : nullptr, training && !masks ? c->seed_dev : nullptr, p, n->code, n->h2,
                              training ? n->masks : nullptr, (int64_t)B * n->d));
  }
  FG_TRY(convl_fwd(e, n->L[2], n->h2, P, n->z3, B));
  {
    AmaxInto am(c, n->L[3].x);
    FG_TRY(k_relu_fwd(c, n->z3, n->h3, (int64_t)B * kH3));
  }
  FG_TRY(convl_fwd(e, n->L[3], n->h3, P, n->z4, B));
  n->valid = true;
  return FG_OK;
}
// from dz4 (gradient at the logits) of the last forward: += the parameter gradients.  dz4's producer ran under
// AmaxInto(L[3].sdy, &env.dy.amax_ready) after the last pairs.reset.
int ae_backward(fg_ae* n) {
  fg_ctx* c = n->c;
  ConvLEnv& e = n->env;
  float* G = n->net.gG;
  const int B = n->B;
  n->grad_B = B;
  FG_TRY(convl_bwd(e, n->L[3], n->h3, n->dz4, G, n->dh, B));
  {
    AmaxInto am(c, n->L[2].sdy, &e.dy.amax_ready);
    FG_TRY(k_relu_bwd(c, n->dh, n->z3, n->dz3, (int64_t)B * kH3));
  }
  FG_TRY(convl_bwd(e, n->L[2], n->h2, n->dz3, G, n->dh, B));
  {
    AmaxInto am(c, n->L[1].sdy, &e.dy.amax_ready);
    FG_TRY(k_tanh_dropout_bwd(c, n->dh, n->train ? n->masks : nullptr, n->p_drop, n->code, n->dz2, (int64_t)B * n->d));
  }
  FG_TRY(convl_bwd(e, n->L[1], n->h1, n->dz2, G, n->dh, B));
  {
    AmaxInto am(c, n->L[0].sdy, &e.dy.amax_ready);
    FG_TRY(k_relu_bwd(c, n->dh, n->z1, n->dz1, (int64_t)B * kH1));
  }
  return convl_bwd(e, n->L[0], n->x, n->dz1, G, nullptr, B);
}

// the per-batch body of train_autoencoder.lua:178-209 on device inputs (images [B][I], masks [B][d] or null: drawn)
int train_step(fg_ae* n, const fg_ae_hyper* h, int B, const float* img, const float* masks) {
  fg_ctx* c = n->c;
  NetPair& p = n->net;
  FG_TRY(pair_zero_grads(c, p, FG_NET_G));
  FG_TRY(ae_forward(n, img, B, true, masks, h->p_drop));
  {
    AmaxInto am(c, n->L[3].sdy, &n->env.dy.amax_ready);
    FG_TRY(k_abs_criterion(c, true, n->z4, img, n->y, n->dz4, (int64_t)B * n->I, &n->dstats->loss));
  }
  FG_TRY(ae_backward(n));
  FG_TRY(k_adam_prep(c, &n->dstats->t, &n->dstats->step, h->lr, h->beta1, h->beta2));
  FG_TRY(k_optim_update(c, FG_OPT_ADAM, p.PG, p.gG, p.mG, p.vG, p.nG, h->beta1, h->beta2, h->eps, 0.f, h->L1, h->L2, 0.f, 1.0f,
                        &n->dstats->step, nullptr, &n->dstats->t));
  p.G_pack = -1;
  FG_CUDA(cudaMemcpyAsync(n->hstats, n->dstats, sizeof(AeStats), cudaMemcpyDeviceToHost, c->stream));
  return FG_OK;
}

int run_train_step(fg_ae* n, const fg_ae_hyper* h, int B, const float* img_dev, const float* masks_dev, uint64_t seed,
                   fg_ae_stats* stats) {
  fg_ctx* c = n->c;
  FG_TRY(net_graph_run(c, n->net, B, h, sizeof(*h), {img_dev, masks_dev}, seed,
                       [&]() { return train_step(n, h, B, img_dev, masks_dev); }));
  // a replayed step does not run the host side of its body: set what it would have set.  The optimizer has moved the
  // parameters away from the activations, so fg_ae_backward needs a new forward.
  n->x = img_dev;
  n->B = n->grad_B = B;
  n->train = true;
  n->p_drop = h->p_drop;
  n->valid = false;
  if (stats) {
    FG_CUDA(cudaStreamSynchronize(c->stream));
    stats->loss = n->hstats->loss;
    stats->t = n->hstats->t;
  }
  return FG_OK;
}
int step_args_ok(const fg_ae* n, const fg_ae_hyper* h, int B, const char* what) {
  FG_REQUIRE(h, "%s: null hyper-parameters", what);
  FG_REQUIRE(B >= 1 && B <= n->maxB, "%s: batch %d out of range [1,%d]", what, B, n->maxB);
  FG_REQUIRE(h->p_drop >= 0.f && h->p_drop < 1.f, "%s: p_drop %g outside [0,1)", what, h->p_drop);
  return FG_OK;
}
}  // namespace

#define ENTER(n)                                \
  do {                                          \
    if (!(n) || !(n)->c) {                      \
      fg_set_error("null fg_ae");               \
      return FG_ERR_INVALID;                    \
    }                                           \
    FG_CUDA(cudaSetDevice((n)->c->device));     \
  } while (0)

extern "C" {

void fg_ae_hyper_default(fg_ae_hyper* h) {
  if (!h) return;
  h->lr = 1e-3f;
  h->beta1 = 0.9f;
  h->beta2 = 0.999f;
  h->eps = 1e-8f;
  h->L1 = 0.f;
  h->L2 = 0.f;
  h->p_drop = 0.5f;
}

int64_t fg_ae_param_count(int size, int noise_dim) {
  if (!ae_shape_ok(size, noise_dim)) return -1;
  ConvL L[4];
  return make_ae_layout(L, size * size, noise_dim);
}

int fg_ae_create(fg_ctx* ctx, int size, int noise_dim, fg_ae** out) {
  if (!ctx || !out) {
    fg_set_error("fg_ae_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  if (ctx->C != 1) {
    fg_set_error("fg_ae_create: the autoencoder is grayscale (train_autoencoder.lua); this context has %d channels", ctx->C);
    return FG_ERR_UNSUPPORTED;
  }
  if (ctx->world > 1) {
    fg_set_error("fg_ae_create: the autoencoder runs on one GPU; this context is data parallel (%d ranks)", ctx->world);
    return FG_ERR_UNSUPPORTED;
  }
  if (size != 16 && size != 32) {
    fg_set_error("fg_ae_create: image size %d; the autoencoder supports 16 and 32", size);
    return FG_ERR_UNSUPPORTED;
  }
  if (!ae_shape_ok(size, noise_dim)) {
    fg_set_error("fg_ae_create: noise_dim %d; the code width must be a multiple of 8 in [8, 1024]", noise_dim);
    return FG_ERR_UNSUPPORTED;
  }
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_ae* n = new fg_ae();
  n->c = ctx;
  n->S = size;
  n->I = size * size;
  n->d = noise_dim;
  n->maxB = ctx->maxB;
  const int r = ae_alloc(n);
  if (r != FG_OK) {
    fg_ae_destroy(n);
    return r;
  }
  *out = n;
  return FG_OK;
}
int fg_ae_destroy(fg_ae* n) {
  if (!n) return FG_OK;
  if (n->c) {
    cudaSetDevice(n->c->device);
    cudaStreamSynchronize(n->c->stream);
  }
  pair_free(n->net);
  if (n->hstats) cudaFreeHost(n->hstats);
  for (void* p : n->allocs) cudaFree(p);
  delete n;
  return FG_OK;
}

int fg_ae_set_params(fg_ae* n, const float* src) {
  ENTER(n);
  FG_REQUIRE(src, "fg_ae_set_params: null source");
  return pair_set_params(n->c, n->net, FG_NET_G, src);
}
int fg_ae_get_params(fg_ae* n, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst, "fg_ae_get_params: null destination");
  return pair_get_params(n->c, n->net, FG_NET_G, dst);
}
int fg_ae_get_grads(fg_ae* n, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst, "fg_ae_get_grads: null destination");
  return pair_get_grads(n->c, n->net, FG_NET_G, dst);
}
int fg_ae_zero_grads(fg_ae* n) {
  ENTER(n);
  return pair_zero_grads(n->c, n->net, FG_NET_G);
}
int fg_ae_set_adam_state(fg_ae* n, const float* m, const float* v, int t) {
  ENTER(n);
  fg_ctx* c = n->c;
  const size_t bytes = n->net.nG * sizeof(float);
  if (m) FG_CUDA(cudaMemcpyAsync(n->net.mG, m, bytes, cudaMemcpyDefault, c->stream));
  if (v) FG_CUDA(cudaMemcpyAsync(n->net.vG, v, bytes, cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemcpyAsync(&n->dstats->t, &t, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int fg_ae_get_adam_state(fg_ae* n, float* m, float* v, int* t) {
  ENTER(n);
  fg_ctx* c = n->c;
  if (m) FG_TRY(fg_to_user(c, m, n->net.mG, n->net.nG));
  if (v) FG_TRY(fg_to_user(c, v, n->net.vG, n->net.nG));
  if (t) {
    FG_CUDA(cudaMemcpyAsync(t, &n->dstats->t, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  return FG_OK;
}

int fg_ae_forward(fg_ae* n, const float* x, int B, int training, const float* masks, uint64_t seed, float* code_out, float* out) {
  ENTER(n);
  FG_REQUIRE(x, "fg_ae_forward: null input");
  FG_REQUIRE(B >= 1 && B <= n->maxB, "fg_ae_forward: batch %d out of range [1,%d]", B, n->maxB);
  fg_ctx* c = n->c;
  const size_t im = (size_t)B * n->I;
  fg_ae_hyper h;
  fg_ae_hyper_default(&h);
  // the rows are kept for fg_ae_backward's weight gradient, whatever the caller does with its buffer
  FG_CUDA(cudaMemcpyAsync(n->xbuf, x, im * sizeof(float), cudaMemcpyDefault, c->stream));
  const float* md = nullptr;
  if (training && masks) FG_TRY(fg_to_dev(c, masks, (size_t)B * n->d, n->in_masks, &md));
  if (training && !masks) FG_TRY(k_set_u64(c, c->seed_dev, seed));
  FG_TRY(ae_forward(n, n->xbuf, B, training != 0, md, h.p_drop));
  FG_TRY(k_sigmoid_fwd(c, n->z4, n->y, (int64_t)im));
  if (code_out) FG_TRY(fg_to_user(c, code_out, n->code, (size_t)B * n->d));
  if (out) FG_TRY(fg_to_user(c, out, n->y, im));
  return FG_OK;
}
int fg_ae_backward(fg_ae* n, const float* dout) {
  ENTER(n);
  FG_REQUIRE(dout, "fg_ae_backward: null gradient");
  fg_ctx* c = n->c;
  if (!n->valid) {
    fg_set_error("fg_ae_backward: no forward to differentiate (a train step leaves none)");
    return FG_ERR_STATE;
  }
  const size_t im = (size_t)n->B * n->I;
  const float* dd;
  FG_TRY(fg_to_dev(c, dout, im, n->in_img, &dd));
  FG_TRY(n->pairs.reset(c));
  {
    AmaxInto am(c, n->L[3].sdy, &n->env.dy.amax_ready);
    FG_TRY(k_sigmoid_bwd(c, dd, n->y, n->dz4, (int64_t)im));
  }
  return ae_backward(n);
}

int fg_ae_train_step(fg_ae* n, const fg_ae_hyper* h, int B, const float* images, const float* masks, uint64_t seed,
                     fg_ae_stats* stats) {
  ENTER(n);
  FG_REQUIRE(images, "fg_ae_train_step: null images");
  FG_TRY(step_args_ok(n, h, B, "fg_ae_train_step"));
  fg_ctx* c = n->c;
  const float *id, *md = nullptr;
  FG_TRY(fg_to_dev(c, images, (size_t)B * n->I, n->in_img, &id));
  if (masks) FG_TRY(fg_to_dev(c, masks, (size_t)B * n->d, n->in_masks, &md));
  return run_train_step(n, h, B, id, md, seed, stats);
}

// the batch idx[0..B) of the dataset at S x S (fg_dataset_gather_sized into device memory: no synchronisation), then the step
int fg_ae_train_step_dataset(fg_ae* n, fg_dataset* d, const fg_ae_hyper* h, const int32_t* idx, int B, uint64_t seed,
                             fg_ae_stats* stats) {
  ENTER(n);
  FG_TRY(dataset_check_feed(d, n->c, "fg_ae_train_step_dataset"));
  FG_REQUIRE(idx, "fg_ae_train_step_dataset: null indices");
  FG_TRY(step_args_ok(n, h, B, "fg_ae_train_step_dataset"));
  FG_TRY(fg_dataset_gather_sized(d, idx, B, n->S, n->in_img));
  return run_train_step(n, h, B, n->in_img, nullptr, seed, stats);
}

// MODEL_AE:forward(images) for N images in chunks of at most `chunk`; chunk k of a training-mode call draws its keep
// flags from seed + k (train_autoencoder.lua:137-145 never calls evaluate(), so its plotted samples are training = 1)
int fg_ae_reconstruct(fg_ae* n, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* out) {
  ENTER(n);
  FG_REQUIRE(images && out && N >= 1 && chunk >= 1 && chunk <= n->maxB, "fg_ae_reconstruct: bad arguments (chunk %d, max %d)",
             chunk, n->maxB);
  fg_ctx* c = n->c;
  fg_ae_hyper h;
  fg_ae_hyper_default(&h);
  const bool out_dev = fg_is_dev(out);
  uint64_t k = 0;
  for (int64_t s = 0; s < N; s += chunk, ++k) {
    const int b = (int)std::min<int64_t>(chunk, N - s);
    const size_t im = (size_t)b * n->I;
    const float* xd;
    FG_TRY(fg_to_dev(c, images + (size_t)s * n->I, im, n->in_img, &xd));
    if (training) FG_TRY(k_set_u64(c, c->seed_dev, seed + k));
    FG_TRY(ae_forward(n, xd, b, training != 0, nullptr, h.p_drop));
    float* dst = out_dev ? out + (size_t)s * n->I : n->y;
    FG_TRY(k_sigmoid_fwd(c, n->z4, dst, (int64_t)im));
    if (!out_dev) {
      FG_CUDA(cudaMemcpyAsync(out + (size_t)s * n->I, n->y, im * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
      FG_CUDA(cudaStreamSynchronize(c->stream));  // y and in_img are reused by the next chunk
    }
  }
  n->valid = false;  // the rows of the last chunk are the caller's
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

int64_t fg_ae_debug_tensor(fg_ae* n, const char* name, float* dst, int64_t max_elems) {
  if (!n || !n->c || !name) {
    fg_set_error("fg_ae_debug_tensor: null argument");
    return -1;
  }
  cudaSetDevice(n->c->device);
  const int B = n->B, gb = n->grad_B;
  const int64_t I = n->I, d = n->d;
  const DebugTensor ents[] = {{"x", n->x, I, B}, {"z1", n->z1, kH1, B}, {"h1", n->h1, kH1, B}, {"z2", n->z2, d, B},
                              {"code", n->code, d, B}, {"h2", n->h2, d, B}, {"z3", n->z3, kH3, B}, {"h3", n->h3, kH3, B},
                              {"z4", n->z4, I, B}, {"y", n->y, I, B}, {"masks", B && n->train ? n->masks : nullptr, d, B},
                              {"dz4", gb ? n->dz4 : nullptr, I, gb}, {"dz3", gb ? n->dz3 : nullptr, kH3, gb},
                              {"dz2", gb ? n->dz2 : nullptr, d, gb}, {"dz1", gb ? n->dz1 : nullptr, kH1, gb},
                              {"loss", &n->dstats->loss, 1, 1}};
  return debug_tensor_copy(n->c, "fg_ae_debug_tensor", ents, sizeof(ents) / sizeof(ents[0]), name, dst, max_elems);
}

}  // extern "C"
