// UpsGan (ups_gan.cu): the trainer of an UpsGen generator and a discriminator, which the 32x32 nets (nets.cu) and the
// --scale 16 nets (nets_s16.cu) both are.  What differs between the sizes is data (GanDesc) and one object, the
// discriminator (GanD); the trainer code never asks which size it serves.
#pragma once
#include <memory>
#include <vector>

#include "convl.h"

struct UpsGan;

// The discriminator of an UpsGan (n): its layers, activations and keep flags, on n's allocation list.  Input x and its
// gradient dx NHWC [B][S][S][C]; logit, sigmoid out and dlogit [B]; GanDesc::mask keep flags per sample.
struct GanD {
  UpsGan* n = nullptr;
  float *x = nullptr, *logit = nullptr, *out = nullptr, *dlogit = nullptr, *masks = nullptr, *dx = nullptr;
  int B = 0;  // batch of the last forward
  virtual ~GanD() = default;
  virtual int64_t layout(int C) = 0;  // the flat parameter layout (getParameters() order): the parameter count
  // its layers and buffers, the layer scratch both nets share (n->env) and the pair's "Dstep.*" table
  virtual int alloc() = 0;
  // keep flags already in masks when training
  virtual int forward(const float* x, int B, bool training, const fg_hyper* h) = 0;
  virtual int backward(bool want_wgrad, bool want_dx) = 0;  // from dlogit; want_dx: the input gradient into dx
  // keep flags of B samples from stream `seed` (root, may be null: the step's stream root on the device)
  virtual int draw_masks(int B, uint64_t seed, const fg_hyper* h, const uint64_t* root) = 0;
  virtual void debug_rows(std::vector<DebugTensor>& rows) const = 0;  // "D.*" of fg_*debug_tensor
};

// What differs between the sizes, as data
struct GanDesc {
  GenDesc g;      // g.side is the side of every image both nets see
  int64_t mask;   // D's keep flags per sample
  bool overlap;   // StepNets::overlap: option dp_overlap may run D's update next to the following G forward
};

// The branched discriminators of models.lua (nets_dbr.cu): create_D32 at side 32, create_D16_d and create_D16 / _b / _c
// at side 16.  disc is FG_DISC_*; every function refuses (side 0, count / width -1, null D) a value that is not one of
// those five.  dbr_param_count takes any channel count C.
int dbr_side(int disc);
int64_t dbr_param_count(int disc, int C);
int dbr_mask_per_sample(int disc);
std::unique_ptr<GanD> dbr_make(int disc);

struct UpsGan {
  fg_ctx* c = nullptr;
  int disc = 0;  // FG_DISC_* of D
  GanDesc d{};
  NetPair net;
  UpsGen G;
  // the generator of the D iterations' fakes: forward only, on G's weight packs, at maxB / 2 (gen_alloc_fwd).  Everything
  // read from G after a step (its outputs, the "G.*" debug rows) is the G iteration's, and the first G iteration's
  // forward may run next to the last D iteration (step_body).  env_f: its allocation context
  UpsGen F;
  ConvLEnv env_f;
  std::unique_ptr<GanD> D;
  // staging at the C ABI: NCHW images from / to the caller and their NHWC conversion; noise rows (or D's output
  // gradient) from the caller and the noise gradient to it
  float *img[2] = {nullptr, nullptr}, *z[2] = {nullptr, nullptr};
  IterStage iter_stage;  // the inputs of the host-fed and device-fed train steps, stacked per iteration
  std::vector<void*> allocs;
  // the scratch G's and D's layers share: env.dy is the split of the current dY, env.ws the packed weight-gradient
  // workspace (largest layer of either net).  D allocates both; g_dy / g_ws (floats) are G's needs, set by gan_alloc
  // before D's alloc()
  ConvLEnv env;
  size_t g_dy = 0, g_ws = 0;
};

// n's pair, D, G and staging on ctx c.  io: a buffer of at least maxB * side^2 * C floats to borrow as img[0], or null
// for one of n's own
int gan_alloc(UpsGan& n, fg_ctx* c, const GanDesc& d, std::unique_ptr<GanD> D, float* io);
void gan_free(UpsGan& n);  // the pair's graphs and mirror, D, and every buffer on n.allocs
int gan_pack_D(UpsGan& n, const std::vector<ConvL*>& layers);  // D's layers, unless net.D_pack is the current pack_key()
// d_iters D iterations + g_iters G iterations of the loop body (pair_train_step) on inputs stacked per iteration:
// real [B/2][C][S][S], noise_D [B/2][100] and noise_G [B][100], masks_D / masks_G [B][mask] (may be null), for entry `what`
int gan_train_step_iters(UpsGan& n, const char* what, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                         const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                         fg_step_stats* stats);
// the same fed on the device: the inputs of D iteration j are gather(draw(4*r_j)) at side S and uniform(4*r_j+1), those
// of G iteration j uniform(4*r_j+2), r_j the stream root of iteration j (fg_b200.h; r_0 = seed).  The draws run inside
// the step (one graph launch per call once captured), each reading its root from c->seed_dev.
int gan_train_step_dataset_iters(UpsGan& n, fg_dataset* d, const char* what, const fg_hyper* h, int B, int d_iters,
                                 int g_iters, uint64_t seed, fg_step_stats* stats);
// the bodies of fg_*G_forward / G_backward / D_forward / D_backward: NCHW images, host or device pointers
int gan_G_forward(UpsGan& n, const float* noise, int B, bool training, float* images_out);
int gan_G_backward(UpsGan& n, const float* d_images, float* d_noise);
int gan_D_forward(UpsGan& n, const float* images, int B, bool training, const float* masks, uint64_t seed, float* out);
int gan_D_backward(UpsGan& n, const float* d_out, bool want_wgrad, float* d_images);
int64_t gan_debug_tensor(UpsGan& n, const char* what, const char* name, float* dst, int64_t max_elems);
