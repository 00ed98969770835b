// The trainable state of a G/D pair (NetPair, fg_internal.h) and what every train step does with it: allocation,
// zeroing and all-reducing the gradients, the accuracy gate and optimizer, the data-parallel broadcast, the statistics
// mirror, the C ABI's set / get bodies, the CUDA-graph replay of the step and the adversarial.lua loop body itself.
// Shared by the trainer of the 32x32 and --scale 16 nets (ups_gan.cu) and the coarse-to-fine nets (nets_c2f.cu).
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "convl.h"
#include "fg_internal.h"

namespace {
struct Half {  // one net of the pair
  float *P, *g, *tail, *m, *v;
  int64_t n;
};
Half half(const NetPair& p, int net) {
  if (net == FG_NET_D) return Half{p.PD, p.gD, p.tailD, p.mD, p.vD, p.nD};
  return Half{p.PG, p.gG, p.tailG, p.mG, p.vG, p.nG};
}
int* step_count(DeviceStats* s, int net) { return net == FG_NET_D ? &s->t_D : &s->t_G; }
}  // namespace

int fg_dalloc(fg_ctx* c, std::vector<void*>& allocs, float** p, size_t n) {
  void* q = nullptr;
  FG_CUDA(cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(float)));
  FG_CUDA(cudaMemsetAsync(q, 0, std::max<size_t>(n, 1) * sizeof(float), c->stream));
  allocs.push_back(q);
  *p = (float*)q;
  return FG_OK;
}

void ctx_swap_side(fg_ctx* c) {
  fg_ctx::Workspaces& s = c->side_ws;
  std::swap(c->stream, c->side_stream);
  std::swap(c->red_ws, s.red_ws);
  std::swap(c->red_ticket, s.red_ticket);
  std::swap(c->bn_acc, s.bn_acc);
  std::swap(c->bn_slice_acc, s.bn_slice_acc);
  std::swap(c->bn_parts, s.bn_parts);
}

int pair_alloc(fg_ctx* c, std::vector<void*>& allocs, NetPair& p, int64_t nG, int64_t nD, bool bn) {
  p.nG = nG;
  p.nD = nD;
  FG_TRY(fg_dalloc(c, allocs, &p.PG, nG));
  FG_TRY(fg_dalloc(c, allocs, &p.PD, nD));
  FG_TRY(fg_dalloc(c, allocs, &p.gG, nG + kGradTail));
  FG_TRY(fg_dalloc(c, allocs, &p.gD, nD + kGradTail));
  p.tailG = p.gG + nG;
  p.tailD = p.gD + nD;
  FG_TRY(fg_dalloc(c, allocs, &p.mG, nG));
  FG_TRY(fg_dalloc(c, allocs, &p.vG, nG));
  FG_TRY(fg_dalloc(c, allocs, &p.mD, nD));
  FG_TRY(fg_dalloc(c, allocs, &p.vD, nD));
  if (bn) {
    FG_TRY(fg_dalloc(c, allocs, &p.bnG, kBnState));
    float init[kBnState];
    for (int i = 0; i < kBnState; ++i) init[i] = (i >= 256 && i < 512) || i >= 640 ? 1.f : 0.f;
    FG_CUDA(cudaMemcpyAsync(p.bnG, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  float* tmp = nullptr;
  FG_TRY(fg_dalloc(c, allocs, &tmp, (sizeof(DeviceStats) + 3) / 4));
  p.dstats = (DeviceStats*)tmp;
  FG_TRY(fg_dalloc(c, allocs, &p.acc_hist, kAccHistMax));
  FG_CUDA(cudaMallocHost((void**)&p.hstats, sizeof(DeviceStats)));
  memset(p.hstats, 0, sizeof(DeviceStats));
  return FG_OK;
}

void pair_clear_graphs(NetPair& p) {
  for (auto& g : p.graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  p.graphs.clear();
}
void pair_free(NetPair& p) {
  pair_clear_graphs(p);
  if (p.hstats) cudaFreeHost(p.hstats);
  p.hstats = nullptr;
  for (NetPair::Keep& k : p.keep) {
    if (k.copy) cudaFree(k.copy);
    k.copy = nullptr;
  }
}

int pair_zero_grads(fg_ctx* c, NetPair& p, int net) {
  const Half h = half(p, net);
  if (h.tail == h.g + h.n) {
    FG_CUDA(cudaMemsetAsync(h.g, 0, sizeof(float) * (h.n + kGradTail), c->stream));
  } else {  // caller-owned gradient buffer (fg_bind_params): the tail lives in the library
    FG_CUDA(cudaMemsetAsync(h.g, 0, sizeof(float) * h.n, c->stream));
    FG_CUDA(cudaMemsetAsync(h.tail, 0, sizeof(float) * kGradTail, c->stream));
  }
  return FG_OK;
}
int pair_allreduce_grads(fg_ctx* c, NetPair& p, int net) {
  if (c->world <= 1) return FG_OK;
  const Half h = half(p, net);
  if (h.tail == h.g + h.n) return net_allreduce(c, h.g, h.n + kGradTail);
  FG_TRY(net_group(true));
  FG_TRY(net_allreduce(c, h.g, h.n));
  FG_TRY(net_allreduce(c, h.tail, kGradTail));
  return net_group(false);
}

int pair_gate(fg_ctx* c, NetPair& p, int net, const fg_hyper* h, int B, float world, bool accumulate) {
  return k_gate_and_prep(c, p.dstats, p.acc_hist, net, h, half(p, net).tail, B, world, accumulate);
}

int IterStage::reserve(fg_ctx* c, std::vector<void*>& allocs, int k, size_t n) {
  if (cap[k] >= n) return FG_OK;
  if (p[k]) {
    FG_CUDA(cudaStreamSynchronize(c->stream));  // an earlier step may still read the old buffer
    allocs.erase(std::find(allocs.begin(), allocs.end(), (void*)p[k]));
    cudaFree(p[k]);
    p[k] = nullptr;
    cap[k] = 0;
  }
  FG_TRY(fg_dalloc(c, allocs, &p[k], n));
  cap[k] = n;
  return FG_OK;
}

int IterStage::in(fg_ctx* c, std::vector<void*>& allocs, int k, const float* q, size_t n, size_t cap_n, const float** out) {
  *out = q;
  if (!q || fg_is_dev(q)) return FG_OK;
  FG_TRY(reserve(c, allocs, k, std::max(n, cap_n)));
  return fg_to_dev(c, q, n, p[k], out);
}

int step_check(fg_ctx* c, const char* what, int B, int nd, int ng, bool inputs, const fg_dataset* d, bool fed) {
  if (nd < 1 || nd > kMaxIters || ng < 1 || ng > kMaxIters) {
    fg_set_error("%s: %d D and %d G iterations; each count must lie in [1, %d]", what, nd, ng, kMaxIters);
    return FG_ERR_UNSUPPORTED;
  }
  if (fed) FG_TRY(dataset_check_feed(d, c, what));
  FG_REQUIRE(inputs, "%s: null input", what);
  FG_REQUIRE(B >= 4 && B % 2 == 0 && B <= c->maxB, "%s: batch %d must be even, >= 4 and <= max_batch %d", what, B, c->maxB);
  return FG_OK;
}

namespace {
__global__ void adam_prep_kernel(int* t_dev, float* step_dev, float lr, float beta1, float beta2) {
  const int t = *t_dev + 1;
  *t_dev = t;
  *step_dev = (float)((double)lr * sqrt(1.0 - pow((double)beta2, (double)t)) / (1.0 - pow((double)beta1, (double)t)));
}
}  // namespace
int k_adam_prep(fg_ctx* c, int* t_dev, float* step_dev, float lr, float beta1, float beta2) {
  adam_prep_kernel<<<1, 1, 0, c->stream>>>(t_dev, step_dev, lr, beta1, beta2);
  LAUNCH_CHECK(c);
  return FG_OK;
}

// penalty -> clamp -> interruptable optimizer on the flat vectors (adversarial.lua:219-231, interruptable_optimizers.lua)
int pair_optim(fg_ctx* c, NetPair& p, int net, const fg_hyper* h, float grad_scale) {
  const bool isD = net == FG_NET_D;
  const Half x = half(p, net);
  DeviceStats* s = p.dstats;
  const float l1 = isD ? h->D_L1 : h->G_L1, l2 = isD ? h->D_L2 : h->G_L2;
  const bool pen = l1 != 0.f || l2 != 0.f;
  // G quirk: the L1 gradient term is multiplied by G_L2 (adversarial.lua:223, adversarial_c2f.lua:108)
  const float l1_grad = !pen ? 0.f : (isD ? l1 : l2);
  if (pen) FG_TRY(k_penalty_loss(c, x.P, x.n, l1, l2, isD ? &s->loss_D : &s->loss_G));
  ScopedTimer tm(c, p.optim_timer[isD]);
  FG_TRY(k_optim_update(c, isD ? c->opt_D : c->opt_G, x.P, x.g, x.m, x.v, x.n, h->beta1, h->beta2, h->eps,
                        isD ? c->sgd_mom_D : c->sgd_mom_G, l1_grad, pen ? l2 : 0.f, isD ? h->D_clamp : h->G_clamp, grad_scale,
                        isD ? &s->step_D : &s->step_G, isD ? &s->do_train_D : &s->do_train_G, step_count(s, net)));
  (isD ? p.D_pack : p.G_pack) = -1;
  return FG_OK;
}

// everything a replica's next step depends on: parameters, optimizer moments, BN running statistics AND the device-side
// step counters / accuracy history (the Adam bias correction uses t: a rank that resumed from a checkpoint at t > 0
// while the others start at 0 would otherwise take a different step size and diverge)
int pair_broadcast(fg_ctx* c, NetPair& p) {
  if (c->world <= 1) return FG_OK;
  FG_TRY(net_group(true));
  const size_t bG = p.nG * sizeof(float), bD = p.nD * sizeof(float);
  FG_TRY(net_broadcast(c, p.PG, bG));
  FG_TRY(net_broadcast(c, p.PD, bD));
  FG_TRY(net_broadcast(c, p.mG, bG));
  FG_TRY(net_broadcast(c, p.vG, bG));
  FG_TRY(net_broadcast(c, p.mD, bD));
  FG_TRY(net_broadcast(c, p.vD, bD));
  if (p.bnG) FG_TRY(net_broadcast(c, p.bnG, kBnState * sizeof(float)));
  FG_TRY(net_broadcast(c, p.dstats, sizeof(DeviceStats)));
  FG_TRY(net_broadcast(c, p.acc_hist, kAccHistMax * sizeof(float)));
  FG_TRY(net_group(false));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  p.G_pack = p.D_pack = -1;
  return FG_OK;
}

int pair_step_stats(fg_ctx* c, const NetPair& p, fg_step_stats* stats) {
  if (!stats) return FG_OK;
  FG_CUDA(cudaStreamSynchronize(c->stream));
  const DeviceStats& s = *p.hstats;
  stats->loss_D = s.loss_D;
  stats->loss_G = s.loss_G;
  for (int i = 0; i < 4; ++i) stats->conf[i] = s.conf[i];
  stats->trained_D = s.trained_D;
  stats->t_D = s.t_D;
  stats->t_G = s.t_G;
  stats->acc_D = s.acc_D;
  return FG_OK;
}

// ---- bodies of the set / get entry points (host or device pointers; a set synchronises) ------------------------------
int pair_set_params(fg_ctx* c, NetPair& p, int net, const float* src) {
  const Half h = half(p, net);
  FG_CUDA(cudaMemcpyAsync(h.P, src, h.n * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  (net == FG_NET_D ? p.D_pack : p.G_pack) = -1;
  return FG_OK;
}
int pair_get_params(fg_ctx* c, const NetPair& p, int net, float* dst) {
  const Half h = half(p, net);
  return fg_to_user(c, dst, h.P, h.n);
}
int pair_get_grads(fg_ctx* c, const NetPair& p, int net, float* dst) {
  const Half h = half(p, net);
  return fg_to_user(c, dst, h.g, h.n);
}
int pair_set_adam_state(fg_ctx* c, NetPair& p, int net, const float* m, const float* v, int t) {
  const Half h = half(p, net);
  if (m) FG_CUDA(cudaMemcpyAsync(h.m, m, h.n * sizeof(float), cudaMemcpyDefault, c->stream));
  if (v) FG_CUDA(cudaMemcpyAsync(h.v, v, h.n * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaMemcpyAsync(step_count(p.dstats, net), &t, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int pair_get_adam_state(fg_ctx* c, const NetPair& p, int net, float* m, float* v, int* t) {
  const Half h = half(p, net);
  if (m) FG_TRY(fg_to_user(c, m, h.m, h.n));
  if (v) FG_TRY(fg_to_user(c, v, h.v, h.n));
  if (t) {
    FG_CUDA(cudaMemcpyAsync(t, step_count(p.dstats, net), sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
  }
  return FG_OK;
}
int pair_set_bn_state(fg_ctx* c, NetPair& p, const float* src) {
  FG_CUDA(cudaMemcpyAsync(p.bnG, src, kBnState * sizeof(float), cudaMemcpyDefault, c->stream));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}
int pair_get_bn_state(fg_ctx* c, const NetPair& p, float* dst) { return fg_to_user(c, dst, p.bnG, kBnState); }

// ---------------------------------------------------------------------------------------------------
// CUDA-graph replay of the step.  A step is ~200 launches of mostly short kernels; replaying a captured graph removes
// the launch gaps (measured 4.19 -> 3.87 ms at batch 256).  A graph bakes in every kernel argument, so it is keyed on all
// of them: batch, hyper-parameters, input pointers, stream, communicator, option epoch (which every option, stream and
// bound-buffer change bumps) and what the weight packs depend on.  The first step with a new key runs eagerly (it also
// performs the lazy allocations), the second is captured, later ones are replayed.
// ---------------------------------------------------------------------------------------------------
namespace {
template <class T>
void key_add(std::vector<uint8_t>& k, const T& v) {
  const uint8_t* q = reinterpret_cast<const uint8_t*>(&v);
  k.insert(k.end(), q, q + sizeof(T));
}
}  // namespace

// The packs are marked stale before the capture and after every replay: the captured sequence has to contain the pack
// kernels whatever the flags said at capture time, and a replayed optimizer step invalidates them again.
int net_graph_run(fg_ctx* c, NetPair& p, int B, const void* hyper, size_t hyper_bytes, std::initializer_list<const void*> inputs,
                  uint64_t seed, const std::function<int()>& body, int nd, int ng) {
  FG_TRY(k_set_u64(c, c->seed_dev, seed));
  static const bool env_off = getenv("FG_GRAPH") && atoi(getenv("FG_GRAPH")) == 0;
  if (!c->use_graph || env_off || c->timing || c->debug_keep) return body();
  std::vector<uint8_t> key;
  key_add(key, c->graph_epoch);
  key_add(key, B);
  key_add(key, nd);
  key_add(key, ng);
  key_add(key, pack_key(c));
  const uint8_t* hb = static_cast<const uint8_t*>(hyper);
  key.insert(key.end(), hb, hb + hyper_bytes);
  for (const void* q : inputs) key_add(key, q);
  key_add(key, (const void*)c->stream);
  key_add(key, c->nccl_comm);
  std::vector<StepGraph>& cache = p.graphs;
  StepGraph* e = nullptr;
  for (auto& g : cache)
    if (g.key == key) e = &g;
  if (!e) {
    if (cache.size() >= 8) {  // oldest out
      if (cache.front().exec) cudaGraphExecDestroy(cache.front().exec);
      cache.erase(cache.begin());
    }
    cache.emplace_back();
    cache.back().key = key;
    return body();  // eager: warms every lazy allocation
  }
  if (e->failed) return body();
  if (!e->exec) {
    p.G_pack = p.D_pack = -1;
    const int64_t l0 = c->launches;
    FG_CUDA(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed));
    const int r = body();
    cudaGraph_t g = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(c->stream, &g);
    cudaGraphExec_t ex = nullptr;
    if (r == FG_OK && ce == cudaSuccess && g && cudaGraphInstantiate(&ex, g, 0) == cudaSuccess) {
      e->exec = ex;
      e->launches = c->launches - l0;
      c->launches = l0;
    } else {
      cudaGetLastError();
      e->failed = true;
    }
    if (g) cudaGraphDestroy(g);
    FG_TRY(r);
    if (e->failed) {  // nothing ran during the failed capture
      FG_TRY(k_set_u64(c, c->seed_dev, seed));
      return body();
    }
  }
  FG_CUDA(cudaGraphLaunch(e->exec, c->stream));
  c->launches += e->launches;
  c->graph_launches++;
  p.G_pack = p.D_pack = -1;
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------------
// The adversarial.lua loop body (:240-288; adversarial_c2f.lua:121-187) on the nets of one trainer: nd D iterations,
// then ng G iterations.  The dropout masks of iteration j are drawn from the stream root c->seed_dev[j] (k_seed_roots;
// [0] is the step seed).
// ---------------------------------------------------------------------------------------------------
namespace {
int keep_dstep(fg_ctx* c, NetPair& p, int B) {
  for (NetPair::Keep& k : p.keep) {
    if (!k.copy) FG_CUDA(cudaMalloc((void**)&k.copy, sizeof(float) * c->maxB * k.per));
    FG_CUDA(cudaMemcpyAsync(k.copy, k.src, sizeof(float) * B * k.per, cudaMemcpyDeviceToDevice, c->stream));
  }
  p.keep_B = B;
  return FG_OK;
}

// a second stream *s of c's and the fork / join events, made on first use
int fork_init(fg_ctx* c, cudaStream_t* s) {
  if (!*s) FG_CUDA(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
  if (!c->ev_fork) FG_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  if (!c->ev_join) FG_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  return FG_OK;
}

int step_body(StepNets& s, int nd, int ng, const float* masksD, const float* masksG, const std::function<int()>* feed) {
  fg_ctx* c = s.c;
  NetPair& p = *s.pair;
  const fg_hyper* h = s.h;
  const int B = s.B, Bh = B / 2;
  const size_t mask = (size_t)B * s.mask;
  const float world = (float)c->world;
  fg_hyper hg = *h;  // the gate's: without the accuracy gate D trains at any accuracy
  if (!s.gate) hg.D_maxAcc = 1e30f;
  if (nd > 1 || ng > 1) FG_TRY(k_seed_roots(c, c->seed_dev, std::max(nd, ng)));
  if (feed) FG_TRY((*feed)());
  // With one GPU the first G iteration's gradient zeroing and generator forward run on side_stream, next to the last D
  // iteration's D forward, backward and update, whose small launches leave most SMs idle.  They read G's parameters and
  // weight packs (changed only by G's optimizer), their inputs and G's BatchNorm running statistics, and the D
  // iterations write none of these once their own generator forwards (a generator of their own: StepNets::g_side) have
  // updated the running statistics.  So the side stream forks right after the last of those forwards and joins before
  // the G iteration's D forward; started earlier, it would only compete with them for the SMs.  Its persistent
  // convolutions run on half the SMs (a one-wave launch on all of them would hold every SM until it ends and stall the
  // D chain behind it; measured on an H100 SXM at 700 W, batch 256: 6.83 -> 6.61 ms per step, the same within noise
  // for 50 to 74 reserved SMs, less gain at 16, a loss at 82 and 90).  Timing runs stay serial (per-launch timers on one stream would
  // misattribute the overlap), and so do debug_keep runs.
  const bool side = s.g_side() && c->world == 1 && !c->timing && !c->debug_keep;
  auto fork_g = [&]() -> int {
    FG_TRY(fork_init(c, &c->side_stream));
    FG_CUDA(cudaEventRecord(c->ev_fork, c->stream));
    FG_CUDA(cudaStreamWaitEvent(c->side_stream, c->ev_fork, 0));
    ctx_swap_side(c);
    c->reserve_sms = c->sm_count / 2;
    int r = pair_zero_grads(c, p, FG_NET_G);
    if (r == FG_OK) r = s.g_forward(0, false);
    c->reserve_sms = 0;
    if (r == FG_OK && cudaEventRecord(c->ev_join, c->stream) != cudaSuccess) r = FG_ERR_CUDA;
    ctx_swap_side(c);
    return r;
  };
  // with dp_overlap, D's gradient all-reduce, gate and optimizer run on the communication stream while the next G
  // forward (it depends on G's parameters only: the fakes of the next D iteration or the first G iteration's samples)
  // proceeds on the compute stream; D is joined right after it.  The replicas stay bit-identical: the same reductions
  // in the same order, only on another stream.
  const bool overlap = s.overlap && c->world > 1 && c->dp_overlap && !c->timing;
  bool forked = false;
  auto g_forward = [&](int j, bool d_iter) -> int {
    // while the collective is in flight the persistent convolution kernels leave a few SMs to it (FG_DP_RESERVE_SMS)
    static const int reserve = getenv("FG_DP_RESERVE_SMS") ? atoi(getenv("FG_DP_RESERVE_SMS")) : 0;
    c->reserve_sms = forked ? reserve : 0;
    const int r = s.g_forward(j, d_iter);
    c->reserve_sms = 0;
    FG_TRY(r);
    if (forked) FG_CUDA(cudaStreamWaitEvent(c->stream, c->ev_join, 0));
    forked = false;
    return FG_OK;
  };
  auto masks = [&](const float* given, int j, int kind) -> int {
    if (given)
      FG_CUDA(cudaMemcpyAsync(s.masks, given + j * mask, sizeof(float) * mask, cudaMemcpyDeviceToDevice, c->stream));
    else
      FG_TRY(s.draw_masks(kind, c->seed_dev + j));
    return FG_OK;
  };
  for (int j = 0; j < nd; ++j) {
    // ---- D iteration j (adversarial.lua:240-268) ----
    FG_TRY(g_forward(j, true));  // createImages
    if (side && j == nd - 1) FG_TRY(fork_g());
    FG_TRY(s.d_input(j));
    FG_TRY(masks(masksD, j, 1));
    FG_TRY(pair_zero_grads(c, p, FG_NET_D));
    FG_TRY(s.d_forward(false));
    FG_TRY(k_sigmoid_bce(c, s.logit, s.out, s.dlogit, &p.dstats->loss_D, p.tailD, B, Bh));
    if (c->debug_keep) FG_TRY(keep_dstep(c, p, B));
    FG_TRY(s.d_backward(true, false));
    const bool acc = j > 0;  // conf / trained_D add up over the step's D iterations
    if (overlap) {
      FG_TRY(fork_init(c, &c->comm_stream));
      FG_CUDA(cudaEventRecord(c->ev_fork, c->stream));
      FG_CUDA(cudaStreamWaitEvent(c->comm_stream, c->ev_fork, 0));
      cudaStream_t compute = c->stream;
      c->stream = c->comm_stream;
      int r = pair_allreduce_grads(c, p, FG_NET_D);
      if (r == FG_OK) r = pair_gate(c, p, FG_NET_D, &hg, B, world, acc);
      if (r == FG_OK) r = pair_optim(c, p, FG_NET_D, h, 1.0f / world);
      if (r == FG_OK && cudaEventRecord(c->ev_join, c->comm_stream) != cudaSuccess) r = FG_ERR_CUDA;
      c->stream = compute;
      FG_TRY(r);
      forked = true;
    } else {
      FG_TRY(pair_allreduce_grads(c, p, FG_NET_D));
      FG_TRY(pair_gate(c, p, FG_NET_D, &hg, B, world, acc));
      FG_TRY(pair_optim(c, p, FG_NET_D, h, 1.0f / world));
    }
  }
  if (side) FG_CUDA(cudaStreamWaitEvent(c->stream, c->ev_join, 0));
  for (int j = 0; j < ng; ++j) {
    // ---- G iteration j (adversarial.lua:275-288) ----
    if (!side || j > 0) {
      FG_TRY(pair_zero_grads(c, p, FG_NET_G));
      FG_TRY(g_forward(j, false));
    }
    FG_TRY(masks(masksG, j, 2));
    FG_TRY(s.d_forward(true));
    FG_TRY(k_sigmoid_bce(c, s.logit, s.out, s.dlogit, &p.dstats->loss_G, p.tailG, B, B));
    FG_TRY(s.d_backward(false, true));  // D's weight grads are discarded by the reference (:209 vs :92)
    FG_TRY(s.g_backward());
    FG_TRY(pair_allreduce_grads(c, p, FG_NET_G));
    FG_TRY(pair_gate(c, p, FG_NET_G, &hg, B, world));
    FG_TRY(pair_optim(c, p, FG_NET_G, h, 1.0f / world));
  }
  FG_CUDA(cudaMemcpyAsync(p.hstats, p.dstats, sizeof(DeviceStats), cudaMemcpyDeviceToHost, c->stream));
  return FG_OK;
}
}  // namespace

int pair_train_step(StepNets& s, int nd, int ng, const float* masksD, const float* masksG, uint64_t seed,
                    std::initializer_list<const void*> inputs, const std::function<int()>* feed, fg_step_stats* stats) {
  FG_TRY(net_graph_run(
      s.c, *s.pair, s.B, s.h, sizeof(*s.h), inputs, seed, [&]() { return step_body(s, nd, ng, masksD, masksG, feed); }, nd, ng));
  return pair_step_stats(s.c, *s.pair, stats);
}

void pair_keep_rows(const NetPair& p, std::vector<DebugTensor>& ents) {
  for (const NetPair::Keep& k : p.keep) ents.push_back({k.name, k.copy, k.per, p.keep_B});
}
