// UpsGan (ups_gan.h): the 32x32 and --scale 16 trainers of train.lua, an UpsGen generator (gen.cu) and a discriminator
// (GanD) in the adversarial.lua loop body (adversarial.lua:54-300; the loop itself is pair_train_step in netpair.cu), and
// the bodies of their C entry points.
#include "ups_gan.h"

#include <algorithm>

namespace {
// the nets in the loop body: real [B/2][C][S][S], noiseD [B/2][100] and noiseG [B][100] per iteration
struct GanStep final : StepNets {
  UpsGan& n;
  GanD& D;
  const float *real, *noiseD, *noiseG;
  GanStep(UpsGan& n, const fg_hyper* h, int B, const float* real, const float* noiseD, const float* noiseG)
      : StepNets(n.c, n.net, h, B, n.D->logit, n.D->out, n.D->dlogit, n.D->masks, n.d.mask, true, n.d.overlap), n(n),
        D(*n.D), real(real), noiseD(noiseD), noiseG(noiseG) {}
  bool g_side() const override { return true; }
  int g_forward(int j, bool d_iter) override {
    const int rows = d_iter ? B / 2 : B;
    return gen_forward(d_iter ? n.env_f : n.env, d_iter ? n.F : n.G, n.net,
                       (d_iter ? noiseD : noiseG) + (size_t)j * rows * kNoiseDim, rows, true);
  }
  int d_input(int j) override {
    const int Bh = B / 2, HW = n.G.S * n.G.S;
    const size_t img = (size_t)c->C * HW;
    FG_TRY(k_nchw_to_nhwc(c, real + (size_t)j * Bh * img, D.x, Bh, c->C, HW));
    FG_CUDA(cudaMemcpyAsync(D.x + Bh * img, n.F.y, sizeof(float) * Bh * img, cudaMemcpyDeviceToDevice, c->stream));
    return FG_OK;
  }
  int draw_masks(int kind, const uint64_t* root) override { return D.draw_masks(B, kind, h, root); }
  int d_forward(bool on_g) override { return D.forward(on_g ? n.G.y : D.x, B, true, h); }
  int d_backward(bool want_wgrad, bool want_dx) override { return D.backward(want_wgrad, want_dx); }
  int g_backward() override { return gen_backward(n.env, n.G, n.net, D.dx, nullptr); }
};
}  // namespace

int gan_alloc(UpsGan& n, fg_ctx* c, const GanDesc& d, std::unique_ptr<GanD> D, float* io) {
  n.c = c;
  n.d = d;
  n.D = std::move(D);
  n.D->n = &n;
  ConvLEnv& e = n.env;
  e.c = c;
  e.maxB = c->maxB;
  e.allocs = &n.allocs;
  FG_TRY(pair_alloc(c, n.allocs, n.net, make_g_layout(c->C, d.g.side).total, n.D->layout(c->C), true));
  // G's share of the scratch: the split of its largest dY (G.C2's [maxB][S][S][128]) and its largest weight gradient
  // (the collapsed 5x5 packs, or G.L1 padded to K = l1_kpad on the tensor cores: (S/4)^2 * 128 rows x (kpad + 100))
  const size_t S = d.g.side;
  n.g_dy = (size_t)c->maxB * S * S * 128;
  n.g_ws = std::max<size_t>(36 * 256 * 128, d.g.l1_kpad ? S * S / 16 * 128 * (d.g.l1_kpad + kNoiseDim) : 0);
  FG_TRY(n.D->alloc());
  FG_TRY(gen_alloc(e, n.G, d.g));
  // the layer scratch of the weight gradients on the wgrad stream (option bwd_streams): G.C3's and those of the 32x32
  // D's tensor-core layers, the largest D.C4's 9 x 512 x 256
  FG_TRY(convl_dalloc(e, &e.ws_w, std::max<size_t>(n.g_ws, 9 * 512 * 256)));
  n.env_f.c = c;
  n.env_f.maxB = c->maxB / 2;
  n.env_f.allocs = &n.allocs;
  FG_TRY(gen_alloc_fwd(n.env_f, n.F, n.G));
  const size_t B = c->maxB, img = B * d.g.side * d.g.side * c->C;
  n.img[0] = io;
  if (!io) FG_TRY(convl_dalloc(e, &n.img[0], img));
  FG_TRY(convl_dalloc(e, &n.img[1], img));
  FG_TRY(convl_dalloc(e, &n.z[0], B * kNoiseDim));
  FG_TRY(convl_dalloc(e, &n.z[1], B * kNoiseDim));
  FG_CUDA(cudaStreamSynchronize(c->stream));
  return FG_OK;
}

void gan_free(UpsGan& n) {
  pair_free(n.net);
  n.D.reset();
  for (void* p : n.allocs) cudaFree(p);
  n.allocs.clear();
}

int gan_pack_D(UpsGan& n, const std::vector<ConvL*>& layers) {
  if (n.net.D_pack == pack_key(n.c)) return FG_OK;
  for (ConvL* L : layers) FG_TRY(convl_pack(n.c, *L, n.net.PD));
  n.net.D_pack = pack_key(n.c);
  return FG_OK;
}

int gan_train_step_iters(UpsGan& n, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                         const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                         fg_step_stats* stats) {
  fg_ctx* c = n.c;
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h && real && noise_D && noise_G));
  const size_t nd = d_iters, ng = g_iters, Bh = B / 2, M = c->maxB, mask = n.d.mask;
  const size_t img = (size_t)c->C * n.G.S * n.G.S;
  IterStage& s = n.iter_stage;
  const float *r, *zd, *zg, *md, *mg;
  FG_TRY(s.in(c, n.allocs, 0, real, nd * Bh * img, nd * M / 2 * img, &r));
  FG_TRY(s.in(c, n.allocs, 1, noise_D, nd * Bh * kNoiseDim, nd * M / 2 * kNoiseDim, &zd));
  FG_TRY(s.in(c, n.allocs, 2, noise_G, ng * B * kNoiseDim, ng * M * kNoiseDim, &zg));
  FG_TRY(s.in(c, n.allocs, 3, masks_D, nd * B * mask, nd * M * mask, &md));
  FG_TRY(s.in(c, n.allocs, 4, masks_G, ng * B * mask, ng * M * mask, &mg));
  GanStep st(n, h, B, r, zd, zg);
  return pair_train_step(st, d_iters, g_iters, md, mg, seed, {r, zd, zg, md, mg, nullptr}, nullptr, stats);
}

int gan_train_step_dataset_iters(UpsGan& n, fg_dataset* d, const char* what, const fg_hyper* h, int B, int d_iters,
                                 int g_iters, uint64_t seed, fg_step_stats* stats) {
  fg_ctx* c = n.c;
  FG_TRY(step_check(c, what, B, d_iters, g_iters, h, d, true));
  const int Bh = B / 2, S = n.G.S;
  const size_t M = c->maxB, img = (size_t)c->C * S * S;
  IterStage& s = n.iter_stage;
  FG_TRY(s.reserve(c, n.allocs, 0, d_iters * M / 2 * img));
  FG_TRY(s.reserve(c, n.allocs, 1, d_iters * M / 2 * kNoiseDim));
  FG_TRY(s.reserve(c, n.allocs, 2, g_iters * M * kNoiseDim));
  float *real = s.p[0], *zd = s.p[1], *zg = s.p[2];
  const std::function<int()> feed = [&]() -> int {
    for (int j = 0; j < d_iters; ++j) {
      FG_TRY(dataset_draw_gather(d, 0, Bh, S, real + (size_t)j * Bh * img, c->seed_dev + j, 4));
      FG_TRY(noise_uniform_dev(c, 1, (int64_t)Bh * kNoiseDim, zd + (size_t)j * Bh * kNoiseDim, c->seed_dev + j, 4));
    }
    for (int j = 0; j < g_iters; ++j)
      FG_TRY(noise_uniform_dev(c, 2, (int64_t)B * kNoiseDim, zg + (size_t)j * B * kNoiseDim, c->seed_dev + j, 4));
    return FG_OK;
  };
  GanStep st(n, h, B, real, zd, zg);
  return pair_train_step(st, d_iters, g_iters, nullptr, nullptr, seed, {real, zd, zg, nullptr, nullptr, d}, &feed, stats);
}

int gan_G_forward(UpsGan& n, const float* noise, int B, bool training, float* images_out) {
  fg_ctx* c = n.c;
  const int HW = n.G.S * n.G.S;
  const float* nd;
  FG_TRY(fg_to_dev(c, noise, (size_t)B * kNoiseDim, n.z[0], &nd));
  FG_TRY(gen_forward(n.env, n.G, n.net, nd, B, training));
  if (images_out) {
    FG_TRY(k_nhwc_to_nchw(c, n.G.y, n.img[0], B, c->C, HW));
    FG_TRY(fg_to_user(c, images_out, n.img[0], (size_t)B * c->C * HW));
  }
  return FG_OK;
}

int gan_G_backward(UpsGan& n, const float* d_images, float* d_noise) {
  fg_ctx* c = n.c;
  const int B = n.G.B, HW = n.G.S * n.G.S;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_images, (size_t)B * c->C * HW, n.img[0], &dd));
  FG_TRY(k_nchw_to_nhwc(c, dd, n.img[1], B, c->C, HW));
  float* dn = nullptr;
  if (d_noise) dn = fg_is_dev(d_noise) ? d_noise : n.z[1];
  FG_TRY(gen_backward(n.env, n.G, n.net, n.img[1], dn));
  if (d_noise && dn != d_noise) FG_TRY(fg_to_user(c, d_noise, dn, (size_t)B * kNoiseDim));
  return FG_OK;
}

int gan_D_forward(UpsGan& n, const float* images, int B, bool training, const float* masks, uint64_t seed, float* out) {
  fg_ctx* c = n.c;
  GanD& D = *n.D;
  const int HW = n.G.S * n.G.S;
  fg_hyper h;
  fg_hyper_default(&h);
  const float* xd;
  FG_TRY(fg_to_dev(c, images, (size_t)B * c->C * HW, n.img[0], &xd));
  FG_TRY(k_nchw_to_nhwc(c, xd, D.x, B, c->C, HW));
  if (training) {
    if (masks) {
      FG_CUDA(cudaMemcpyAsync(D.masks, masks, sizeof(float) * B * n.d.mask, cudaMemcpyDefault, c->stream));
    } else {
      FG_TRY(D.draw_masks(B, seed, &h, nullptr));
    }
  }
  FG_TRY(D.forward(D.x, B, training, &h));
  FG_TRY(k_sigmoid_fwd(c, D.logit, D.out, B));
  if (out) FG_TRY(fg_to_user(c, out, D.out, B));
  return FG_OK;
}

int gan_D_backward(UpsGan& n, const float* d_out, bool want_wgrad, float* d_images) {
  fg_ctx* c = n.c;
  GanD& D = *n.D;
  const int B = D.B, HW = n.G.S * n.G.S;
  const float* dd;
  FG_TRY(fg_to_dev(c, d_out, B, n.z[0], &dd));
  FG_TRY(k_sigmoid_grad_mul(c, dd, D.out, D.dlogit, B));
  FG_TRY(D.backward(want_wgrad, d_images != nullptr));
  if (d_images) {
    FG_TRY(k_nhwc_to_nchw(c, D.dx, n.img[0], B, c->C, HW));
    FG_TRY(fg_to_user(c, d_images, n.img[0], (size_t)B * c->C * HW));
  }
  return FG_OK;
}

int64_t gan_debug_tensor(UpsGan& n, const char* what, const char* name, float* dst, int64_t max_elems) {
  cudaSetDevice(n.c->device);
  std::vector<DebugTensor> ents;
  n.D->debug_rows(ents);
  pair_keep_rows(n.net, ents);
  gen_debug_rows(n.G, ents);
  return debug_tensor_copy(n.c, what, ents.data(), ents.size(), name, dst, max_elems);
}
