// The `--scale 16` nets of train.lua (models.create_G / create_D pick them when dimensions[2] == 16, models.lua:87-104)
// and the adversarial.lua loop body on them:
//   G16 = models.lua:27-51   create_G_decoder_upsampling16: Linear(100, 128*4*4) View(128,4,4) PReLU | Up2 conv(128->256,5)
//         BN PReLU | Up2 conv(256->128,5) BN PReLU | conv(128->C,3) Sigmoid  -- the 32x32 generator with every size halved
//   D   = create_D16_d (models.lua:279-316, the default), create_D16, create_D16_b or create_D16_c: the branched
//         discriminators of nets_dbr.cu
//   loop = adversarial.lua:83-288 (the same fevalD / fevalG_on_D / accuracy gate / interruptable optimizers as the 32x32 nets)
// Trainer: the 32x32 nets' trainer type at side 16 (UpsGan, ups_gan.cu); G16 is the 32x32 nets' generator type at side
// 16 (UpsGen, gen.cu).  This file holds the C entry points.
#include <algorithm>

#include "fg_internal.h"
#include "ups_gan.h"

constexpr int kSide = 16;

struct fg_s16 : UpsGan {};

#define ENTER(n)                                         \
  do {                                                   \
    if (!(n) || !(n)->c) {                               \
      fg_set_error("null fg_s16");                       \
      return FG_ERR_INVALID;                             \
    }                                                    \
    FG_CUDA(cudaSetDevice((n)->c->device));              \
  } while (0)

extern "C" {

int fg_s16_create(fg_ctx* ctx, fg_s16** out) { return fg_s16_create_disc(ctx, FG_DISC_D16_D, out); }

int fg_s16_create_disc(fg_ctx* ctx, int disc, fg_s16** out) {
  if (!ctx || !out) {
    fg_set_error("fg_s16_create: null argument");
    return FG_ERR_INVALID;
  }
  *out = nullptr;
  if (disc == FG_DISC_DEFAULT) disc = FG_DISC_D16_D;
  FG_REQUIRE(fg_disc_side(disc), "fg_s16_create_disc: unknown discriminator %d", disc);
  if (fg_disc_side(disc) != kSide) {
    fg_set_error("fg_s16_create_disc: discriminator %d is a 32x32 net; the --scale 16 nets take FG_DISC_D16_D, "
                 "FG_DISC_D16, FG_DISC_D16_B or FG_DISC_D16_C", disc);
    return FG_ERR_UNSUPPORTED;
  }
  FG_CUDA(cudaSetDevice(ctx->device));
  fg_s16* n = new fg_s16();
  n->disc = disc;
  // G.L1 keeps K = 100 (on the FFMA kernels): padding it would change its bits.  Two backward launches per 5x5 layer.
  const GanDesc k16{{kSide, "s16.", 0, false}, dbr_mask_per_sample(disc), false};
  const int r = gan_alloc(*n, ctx, k16, dbr_make(disc), nullptr);
  if (r != FG_OK) {
    fg_s16_destroy(n);
    return r;
  }
  *out = n;
  return FG_OK;
}
int fg_s16_destroy(fg_s16* n) {
  if (!n) return FG_OK;
  if (n->c) {
    cudaSetDevice(n->c->device);
    cudaStreamSynchronize(n->c->stream);
  }
  gan_free(*n);
  delete n;
  return FG_OK;
}
int64_t fg_s16_param_count(int net, int channels) {
  if (net != FG_NET_D) return make_g_layout(channels, kSide).total;
  return dbr_param_count(FG_DISC_D16_D, channels);
}
int fg_s16_mask_per_sample(void) { return dbr_mask_per_sample(FG_DISC_D16_D); }
int fg_s16_get_disc(fg_s16* n) {
  ENTER(n);
  return n->disc;
}

int fg_s16_set_params(fg_s16* n, int net, const float* src) {
  ENTER(n);
  FG_REQUIRE(src && (net == FG_NET_G || net == FG_NET_D), "fg_s16_set_params: bad arguments");
  return pair_set_params(n->c, n->net, net, src);
}
int fg_s16_get_params(fg_s16* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_s16_get_params: bad arguments");
  return pair_get_params(n->c, n->net, net, dst);
}
int fg_s16_get_grads(fg_s16* n, int net, float* dst) {
  ENTER(n);
  FG_REQUIRE(dst && (net == FG_NET_G || net == FG_NET_D), "fg_s16_get_grads: bad arguments");
  return pair_get_grads(n->c, n->net, net, dst);
}
int fg_s16_zero_grads(fg_s16* n, int net) {
  ENTER(n);
  return pair_zero_grads(n->c, n->net, net);
}
float* fg_s16_params_ptr(fg_s16* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->net.PD : n->net.PG); }
float* fg_s16_grads_ptr(fg_s16* n, int net) { return !n ? nullptr : (net == FG_NET_D ? n->net.gD : n->net.gG); }

int fg_s16_set_adam_state(fg_s16* n, int net, const float* m, const float* v, int t) {
  ENTER(n);
  return pair_set_adam_state(n->c, n->net, net, m, v, t);
}
int fg_s16_get_adam_state(fg_s16* n, int net, float* m, float* v, int* t) {
  ENTER(n);
  return pair_get_adam_state(n->c, n->net, net, m, v, t);
}
// running_mean / running_var of G's two nn.SpatialBatchNormalization layers: [mean1 256][var1 256][mean2 128][var2 128]
int fg_s16_set_bn_state(fg_s16* n, const float* src768) {
  ENTER(n);
  FG_REQUIRE(src768, "fg_s16_set_bn_state: null source");
  return pair_set_bn_state(n->c, n->net, src768);
}
int fg_s16_get_bn_state(fg_s16* n, float* dst768) {
  ENTER(n);
  FG_REQUIRE(dst768, "fg_s16_get_bn_state: null destination");
  return pair_get_bn_state(n->c, n->net, dst768);
}

// noise [B][100] -> images [B][C][16][16] (NCHW; host or device pointers).  training != 0: batch statistics + running
// stat update (nn_utils.lua:52 createImages leaves G in training mode); 0: evaluate() with the running statistics.
int fg_s16_G_forward(fg_s16* n, const float* noise, int B, int training, float* img_out) {
  ENTER(n);
  FG_REQUIRE(noise && B >= 1 && B <= n->c->maxB, "fg_s16_G_forward: bad arguments (batch %d, max %d)", B, n->c->maxB);
  return gan_G_forward(*n, noise, B, training != 0, img_out);
}
int fg_s16_G_backward(fg_s16* n, const float* d_img, float* d_noise) {
  ENTER(n);
  FG_REQUIRE(d_img, "fg_s16_G_backward: null gradient");
  return gan_G_backward(*n, d_img, d_noise);
}
int fg_s16_D_forward(fg_s16* n, const float* img, int B, int training, const float* masks, uint64_t seed, float* out) {
  ENTER(n);
  FG_REQUIRE(img && B >= 1 && B <= n->c->maxB, "fg_s16_D_forward: bad arguments (batch %d, max %d)", B, n->c->maxB);
  return gan_D_forward(*n, img, B, training != 0, masks, seed, out);
}
// fg_D_score on D16_d: predictions for N 16x16 images in chunks of `chunk`, dropout masks of chunk s drawn from
// seed + s when training (sample.lua --scale 16 never calls evaluate())
int fg_s16_D_score(fg_s16* n, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out) {
  ENTER(n);
  FG_REQUIRE(images && preds_out && N >= 1 && chunk >= 1 && chunk <= n->c->maxB, "fg_s16_D_score: bad arguments (chunk %d, max %d)",
             chunk, n->c->maxB);
  const size_t img = (size_t)n->c->C * 256;
  for (int64_t s = 0; s < N; s += chunk) {
    const int b = (int)std::min<int64_t>(chunk, N - s);
    FG_TRY(fg_s16_D_forward(n, images + (size_t)s * img, b, training, nullptr, seed + (uint64_t)s, preds_out + s));
  }
  return FG_OK;
}
int fg_s16_D_backward(fg_s16* n, const float* d_out, int want_wgrad, float* d_img) {
  ENTER(n);
  FG_REQUIRE(d_out, "fg_s16_D_backward: null gradient");
  return gan_D_backward(*n, d_out, want_wgrad != 0, d_img);
}

// data parallel: rank 0's parameters, optimizer moments, step counters and BatchNorm running statistics to every rank
int fg_s16_dp_broadcast_params(fg_s16* n) {
  ENTER(n);
  return pair_broadcast(n->c, n->net);
}

int fg_s16_train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                      const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_iters(*n, "fg_s16_train_step", h, B, 1, 1, real, noise_D, noise_G, masks_D, masks_G, seed, stats);
}

// train.lua --scale 16 fed on the device: real = gather at 16x16 of draw(4*seed, B/2), noise_D = uniform(4*seed+1),
// noise_G = uniform(4*seed+2), dropout masks from `seed` (the streams of fg_train_step_dataset)
int fg_s16_train_step_dataset(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_dataset_iters(*n, d, "fg_s16_train_step_dataset", h, B, 1, 1, seed, stats);
}

// d_iters D iterations + g_iters G iterations on inputs stacked per iteration (fg_train_step_iters at 16x16)
int fg_s16_train_step_iters(fg_s16* n, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                            const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G,
                            uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_iters(*n, "fg_s16_train_step_iters", h, B, d_iters, g_iters, real, noise_D, noise_G, masks_D,
                              masks_G, seed, stats);
}

// fg_s16_train_step_iters fed on the device: the streams of fg_train_step_dataset_iters, the real halves at 16x16
int fg_s16_train_step_dataset_iters(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters,
                                    uint64_t seed, fg_step_stats* stats) {
  ENTER(n);
  return gan_train_step_dataset_iters(*n, d, "fg_s16_train_step_dataset_iters", h, B, d_iters, g_iters, seed, stats);
}

int64_t fg_s16_debug_tensor(fg_s16* n, const char* name, float* dst, int64_t max_elems) {
  if (!n || !n->c || !name) {
    fg_set_error("fg_s16_debug_tensor: null argument");
    return -1;
  }
  return gan_debug_tensor(*n, "fg_s16_debug_tensor", name, dst, max_elems);
}

}  // extern "C"
