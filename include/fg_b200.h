/* fg_b200.h -- C ABI of the H100-native GAN train-step hot path of aleju/face-generator.
 *
 * The reference (Lua/Torch7) has NO native FFI for this path: its "plugin surface" is Torch7's
 * Lua-level nn.Module protocol plus train.lua's globals (SURVEY.md section 8b).  This header is
 * therefore the ABI a LuaJIT `ffi.cdef` binds (see INTEGRATION.md and
 * face_generator_b200/lua/fg_ffi.lua); each entry cites the reference interface it replaces.
 *
 * Conventions
 *   - extern "C", plain C types only.  Every call returns 0 (FG_OK) or a negative FG_ERR_*;
 *     nothing throws or exits.  fg_last_error() returns a description of the last failure.
 *   - Tensors at the boundary are dense fp32 in the REFERENCE layouts: images NCHW
 *     [B][C][32][32], noise [B][100], flat parameter vectors in getParameters() order with conv
 *     weights [Cout][Cin][kH][kW] and Linear weights [out][in].  (Internally everything is NHWC.)
 *   - Data pointers may be HOST or DEVICE pointers (classified with cudaPointerGetAttributes);
 *     host buffers are staged through pinned memory on the context's stream -- this is the
 *     replacement of the reference's nn.Copy host<->device hops (utils/nn_utils.lua:355-362).
 *   - One fg_ctx per GPU, no concurrent calls on one ctx (Lua is single-threaded).
 *   - There is NO CPU fallback: every entry needs a CUDA device of compute capability 10.x.
 */
#ifndef FG_B200_H
#define FG_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct fg_ctx fg_ctx;

enum {
  FG_OK = 0,
  FG_ERR_INVALID = -1,      /* bad argument (odd batch, batch > max_batch, NULL, ...) */
  FG_ERR_CUDA = -2,         /* CUDA runtime / driver error (sticky on the ctx)        */
  FG_ERR_NCCL = -3,         /* NCCL error                                             */
  FG_ERR_UNSUPPORTED = -4,  /* valid request the library does not implement           */
  FG_ERR_STATE = -5         /* call order violated (backward without forward, ...)    */
};
enum { FG_NET_G = 0, FG_NET_D = 1 };

/* Which implementation the big convolutions use (fg_set_option "conv_impl"). */
enum {
  FG_CONV_SIMT = 0,         /* fp32 FFMA implicit GEMM (first correct path, any shape)          */
  FG_CONV_TC_DENSE = 1,     /* wgmma 3xTF32 implicit GEMM, dense 5x5 taps on the low-res input   */
  FG_CONV_TC_COLLAPSED = 2  /* wgmma 3-term split, upsample folded into four 3x3 phase convs    */
};

/* OPT.D_optmethod / OPT.G_optmethod (train.lua:38-39; adversarial.lua:259-285):
 * fg_set_option(ctx, "optimizer_D" | "optimizer_G", FG_OPT_*).  With FG_OPT_ADAGRAD / FG_OPT_SGD
 * fg_hyper.lr_D / lr_G carry OPTSTATE.adagrad.*.learningRate (default 1e-3) resp.
 * OPTSTATE.sgd.*.learningRate (--D_SGD_lr / --G_SGD_lr, default 0.02); SGD momentum (= dampening,
 * interruptable_optimizers.lua:104-105) via fg_set_option_f(ctx, "sgd_momentum_D" | "_G", m).
 * State reuse: Adagrad's paramVariance lives in the Adam `v` buffer, SGD's momentum buffer in `m`,
 * state.evalCounter in `t`.                                                                        */
enum { FG_OPT_ADAM = 0, FG_OPT_ADAGRAD = 1, FG_OPT_SGD = 2 };

/* Hyper-parameters of one adversarial.lua loop body; defaults = train.lua:16-50 +
 * interruptable_optimizers.lua:53-57. */
typedef struct fg_hyper {
  float lr_D, lr_G;         /* Adam learning rates (--D_adam_lr/--G_adam_lr; -1 there => 1e-3)   */
  float beta1, beta2, eps;  /* 0.9, 0.999, 1e-8                                                   */
  float D_L1, D_L2;         /* 0, 1e-4   (adversarial.lua:103-109)                                */
  float G_L1, G_L2;         /* 0, 0      (adversarial.lua:218-224; L1 grad term uses G_L2, :223)  */
  float D_clamp, G_clamp;   /* 1, 5      (adversarial.lua:121-123, :226-228); 0 = off             */
  float D_maxAcc;           /* 1.01: D is only stepped while mean accuracy < this (:156-178)      */
  int32_t accs_interval;    /* length of the accuracy history (train.lua:207)                     */
  float p_spatial, p_drop;  /* 0.2, 0.5  SpatialDropout / Dropout probabilities (models.lua)      */
} fg_hyper;

typedef struct fg_step_stats {
  float loss_D, loss_G;     /* f returned by fevalD / fevalG_on_D (incl. penalty terms)           */
  int32_t conf[4];          /* D-step confusion: [pred1&real, pred0&real, pred1&fake, pred0&fake] */
  int32_t trained_D;        /* 0 when the accuracy gate skipped D's Adam step                     */
  int32_t t_D, t_G;         /* Adam step counters after this iteration                            */
  float acc_D;              /* D's accuracy on this batch (confusionBatchD.totalValid)            */
} fg_step_stats;

const char* fg_version(void);
const char* fg_last_error(void);
void fg_hyper_default(fg_hyper* h);

/* ---- context ------------------------------------------------------------------------------- */
/* channels = IMG_DIMENSIONS[1] (1 or 3, train.lua:92-93); max_batch = largest OPT.batchSize.    */
int fg_create(fg_ctx** out, int device, int max_batch, int channels);
int fg_destroy(fg_ctx* ctx);
int fg_set_stream(fg_ctx* ctx, void* cuda_stream);      /* cutorch's current stream; NULL = own  */
int fg_sync(fg_ctx* ctx);
/* keys: "conv_impl" (FG_CONV_*), "optimizer_D" / "optimizer_G" (FG_OPT_*), "debug_keep" (tests: keep the D
 * step's pre-activations of fg_train_step as "Dstep.*" debug tensors), "edge_impl" / "bn_epilogue"
 * (0 selects the round-1 kernels for the 3-channel convolutions / a separate BatchNorm statistics
 * pass: cross-checks), "params_dirty" (re-pack weights
 * after writing through fg_params_ptr); unknown keys return FG_ERR_INVALID                        */
int fg_set_option(fg_ctx* ctx, const char* key, int64_t value);
int64_t fg_get_option(fg_ctx* ctx, const char* key);
int fg_set_option_f(fg_ctx* ctx, const char* key, double value);    /* "sgd_momentum_D", "sgd_momentum_G"     */

/* ---- parameters: replaces MODEL:getParameters() (train.lua:151-152) -------------------------- */
int64_t fg_param_count(int net, int channels);
int fg_set_params(fg_ctx* ctx, int net, const float* src);
int fg_get_params(fg_ctx* ctx, int net, float* dst);
int fg_get_grads(fg_ctx* ctx, int net, float* dst);
int fg_zero_grads(fg_ctx* ctx, int net);                 /* GRAD_PARAMETERS_x:zero()              */
float* fg_params_ptr(fg_ctx* ctx, int net);              /* device pointers for Torch aliasing    */
float* fg_grads_ptr(fg_ctx* ctx, int net);
/* Borrow caller-owned DEVICE buffers (fg_param_count floats each, 16-byte aligned) as the flat
 * parameter / gradient vectors of `net`.  train.lua:151-152 `MODEL:getParameters()` re-points every
 * module's weight / gradWeight into ONE new flat storage; a b200.Fused module then passes
 * weight:data() / gradWeight:data() here, so that the tensors the reference's loop mutates
 * (GRAD_PARAMETERS:zero() / :add() / :clamp(), the optimizer's in-place update of PARAMETERS,
 * adversarial.lua:92-123, interruptable_optimizers.lua:78-90) ARE the buffers the kernels read and
 * write.  The buffers are used as they are (nothing is copied).  NULL restores the library's own
 * buffer for that vector.  Packed weights are rebuilt on the next forward.                        */
int fg_bind_params(fg_ctx* ctx, int net, float* params_dev, float* grads_dev);
/* OPTSTATE.adam.{D,G}.{m,v,t} (interruptable_optimizers.lua:69-75); any pointer may be NULL     */
int fg_set_adam_state(fg_ctx* ctx, int net, const float* m, const float* v, int t);
int fg_get_adam_state(fg_ctx* ctx, int net, float* m, float* v, int* t);
/* G's BatchNorm running statistics [rm1(256) rv1(256) rm2(128) rv2(128)]                          */
int fg_set_bn_state(fg_ctx* ctx, const float* src768);
int fg_get_bn_state(fg_ctx* ctx, float* dst768);

/* ---- L-net: MODEL_G / MODEL_D :forward / :backward ------------------------------------------- */
/* models.lua:57-81.  noise [B][100] -> images [B][C][32][32] (may be NULL to keep on device).   */
int fg_G_forward(fg_ctx* ctx, const float* noise, int B, int training, float* images_out);
/* d_images [B][C][32][32]; accumulates into G's grad buffer; d_noise may be NULL.               */
int fg_G_backward(fg_ctx* ctx, const float* d_images, float* d_noise);
/* models.lua:382-416.  masks: [B][1984] keep flags (0/1) per sample =
 * [64|128|256|512] SpatialDropout + [512|512] Dropout; NULL => drawn in-kernel from `seed`.
 * training=0 => evaluate() semantics.  out [B] sigmoid outputs (may be NULL).                   */
int fg_D_forward(fg_ctx* ctx, const float* images, int B, int training, const float* masks, uint64_t seed,
                 float* out);
/* d_out [B]; want_wgrad=0 skips D's weight gradients (the G step discards them,
 * adversarial.lua:209 vs :92); d_images [B][C][32][32] may be NULL.                             */
int fg_D_backward(fg_ctx* ctx, const float* d_out, int want_wgrad, float* d_images);
/* nn.BCECriterion forward/backward (train.lua:148); x,t length n.                               */
int fg_bce_forward(fg_ctx* ctx, const float* x, const float* t, int n, float* loss_out);
int fg_bce_backward(fg_ctx* ctx, const float* x, const float* t, int n, float* dx);
/* penalty + clamp + interruptableAdam (or the optimizer chosen with "optimizer_D"/"optimizer_G")
 * on the ctx's own buffers (adversarial.lua:103-123, interruptable_optimizers.lua:7-167).
 * grad_scale multiplies the gradient first (1/N for DP).                                         */
int fg_optim_step(fg_ctx* ctx, int net, const fg_hyper* h, float grad_scale);

/* ---- L-op: raw-pointer optimizer for b200.Adam (DEVICE pointers) ----------------------------- */
int fg_adam_step(fg_ctx* ctx, float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1,
                 float beta2, float eps, int t, float l1_grad, float l2, float clampv, float grad_scale);

/* ---- L-op: single layers at the nn.Module boundary (NCHW, DEVICE or HOST pointers) ----------- */
/* cudnn.SpatialConvolution / nn.SpatialConvolution, stride 1, pad (k-1)/2 (models.lua:64,69,73,385-400)
 * and layers/cudnnSpatialConvolutionUpsample.lua with factor=1 (identical math).                 */
int fg_conv2d_forward(fg_ctx* ctx, const float* x, const float* w, const float* b, float* y, int N, int Cin, int H,
                      int W, int Cout, int k);
int fg_conv2d_backward_data(fg_ctx* ctx, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W,
                            int Cout, int k);
/* accumulates (dw += , db +=) like accGradParameters; db may be NULL                             */
int fg_conv2d_backward_filter(fg_ctx* ctx, const float* x, const float* dy, float* dw, float* db, int N, int Cin,
                              int H, int W, int Cout, int k);
/* layers/cudnnSpatialConvolutionUpsample.lua with any factor (:4-16 constructor, :18-30 updateOutput, :32-58 backward):
 * a "same" convolution to nOutputPlane*factor*factor planes whose output [N][nOutputPlane*f*f][H][W] is RE-VIEWED (not
 * permuted) as [N][nOutputPlane][H*f][W*f] -- the same contiguous bytes, so y / dy here are that buffer under either
 * shape.  w is [nOutputPlane*f*f][Cin][k][k], b [nOutputPlane*f*f].  factor = 1 is fg_conv2d_*.                      */
int fg_scu_forward(fg_ctx* ctx, const float* x, const float* w, const float* b, float* y, int N, int Cin, int H, int W,
                   int nOutputPlane, int k, int factor);
int fg_scu_backward_data(fg_ctx* ctx, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W,
                         int nOutputPlane, int k, int factor);
int fg_scu_backward_filter(fg_ctx* ctx, const float* x, const float* dy, float* dw, float* db, int N, int Cin, int H,
                           int W, int nOutputPlane, int k, int factor);
/* nn.Linear (models.lua:59,406-412)                                                              */
int fg_linear_forward(fg_ctx* ctx, const float* x, const float* w, const float* b, float* y, int N, int in, int out);
int fg_linear_backward(fg_ctx* ctx, const float* x, const float* w, const float* dy, float* dx, float* dw, float* db,
                       int N, int in, int out);
/* nn.SpatialBatchNormalization training mode (models.lua:65,70); save_mean/save_istd [C]         */
int fg_bn_forward_train(fg_ctx* ctx, const float* x, const float* gamma, const float* beta, float* y,
                        float* save_mean, float* save_istd, float* run_mean, float* run_var, int N, int C, int HW);
int fg_bn_backward(fg_ctx* ctx, const float* x, const float* gamma, const float* save_mean, const float* save_istd,
                   const float* dy, float* dx, float* dgamma, float* dbeta, int N, int C, int HW);
/* nn.PReLU with one shared slope (models.lua:61,...)                                             */
int fg_prelu_forward(fg_ctx* ctx, const float* x, const float* slope, float* y, int64_t n);
int fg_prelu_backward(fg_ctx* ctx, const float* x, const float* slope, const float* dy, float* dx, float* dslope,
                      int64_t n);
/* nn.SpatialUpSamplingNearest(2) (models.lua:63,68): x [N][C][H][W] -> y [N][C][2H][2W];
 * backward sums each 2x2 block of dy.                                                            */
int fg_upsample2_forward(fg_ctx* ctx, const float* x, float* y, int N, int C, int H, int W);
int fg_upsample2_backward(fg_ctx* ctx, const float* dy, float* dx, int N, int C, int H, int W);
/* nn.SpatialAveragePooling(2,2,2,2) (models.lua:388,...): x [N][C][H][W] -> y [N][C][H/2][W/2]   */
int fg_avgpool2_forward(fg_ctx* ctx, const float* x, float* y, int N, int C, int H, int W);
int fg_avgpool2_backward(fg_ctx* ctx, const float* dy, float* dx, int N, int C, int H, int W);
/* nn.SpatialMaxPooling(2,2) (models_c2f.lua:251,256): first strict maximum in row-major window
 * order wins (THNN); the backward recomputes the arg-max from x.                                 */
int fg_maxpool2_forward(fg_ctx* ctx, const float* x, float* y, int N, int C, int H, int W);
int fg_maxpool2_backward(fg_ctx* ctx, const float* x, const float* dy, float* dx, int N, int C, int H, int W);
/* nn.Dropout (spatial=0: one keep flag per element, y = x*mask/(1-p), models.lua:408,411) and
 * nn.SpatialDropout (spatial=1: one flag per (n,c) plane, NO rescale, models.lua:387,...).
 * mask holds 0/1 keep flags (n elements resp. N*C); mask == NULL means evaluate(): Dropout is the
 * identity, SpatialDropout multiplies by (1-p).  The backward is the same map applied to dy.     */
int fg_dropout_forward(fg_ctx* ctx, const float* x, const float* mask, float p, int spatial, float* y, int N, int C,
                       int HW);
int fg_dropout_backward(fg_ctx* ctx, const float* dy, const float* mask, float p, int spatial, float* dx, int N,
                        int C, int HW);
/* draws keep flags (1 with probability 1-p) for the two layers above into a DEVICE buffer        */
int fg_dropout_mask(fg_ctx* ctx, float* mask_dev, int64_t n, float p, uint64_t seed);
/* nn.Sigmoid (models.lua:74,413)                                                                 */
int fg_sigmoid_forward(fg_ctx* ctx, const float* x, float* y, int64_t n);
int fg_sigmoid_backward(fg_ctx* ctx, const float* y, const float* dy, float* dx, int64_t n);

/* ---- L-step: the adversarial.lua:54-300 loop body -------------------------------------------- */
/* real [B/2][C][32][32] in [0,1]; noise_D [B/2][100], noise_G [B][100] ~ U(-1,1)
 * (utils/nn_utils.lua:35-39); masks_D / masks_G [B][1984] or NULL (then drawn from seed).
 * Runs 1 D iteration + 1 G iteration incl. both Adam updates.  stats may be NULL (fully
 * asynchronous); otherwise the call synchronises the stream and fills it.                        */
int fg_train_step(fg_ctx* ctx, const fg_hyper* h, int B, const float* real, const float* noise_D,
                  const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                  fg_step_stats* stats);
/* sample.lua:80 / nn_utils.lua:45-69: G forward over N noise vectors in chunks (train-mode BN). */
int fg_sample(fg_ctx* ctx, const float* noise, int N, int chunk, float* images_out);

/* ---- coarse-to-fine GAN (train_c2f.lua; BASELINE configs[3]) --------------------------------- */
/* G = models_c2f.lua:113-145 create_G_d, D = models_c2f.lua:237-278 create_D_c, both at 32x32 on
 * the ctx's channel count; cudnn.SpatialConvolutionUpsample with factor 1
 * (layers/cudnnSpatialConvolutionUpsample.lua) is a "same" convolution.  The object borrows the
 * ctx (stream, device, DP communicator, "conv_impl"); destroy it before the ctx.  Flat parameter
 * vectors follow getParameters() order: G [c1W c1b a1 ... c4W c4b a4 c5W c5b], D [c1W c1b a1 ...
 * c4W c4b a4 L1W L1b a5 L2W L2b].                                                                 */
typedef struct fg_c2f fg_c2f;
int fg_c2f_create(fg_ctx* ctx, fg_c2f** out);
int fg_c2f_destroy(fg_c2f* n);
int64_t fg_c2f_param_count(int net, int channels);        /* 1 101 319 / 8 797 382 for colour      */
int fg_c2f_mask_per_sample(void);                         /* 16896 = [256][8][8] + [512] nn.Dropout */
int fg_c2f_set_params(fg_c2f* n, int net, const float* src);
int fg_c2f_get_params(fg_c2f* n, int net, float* dst);
int fg_c2f_get_grads(fg_c2f* n, int net, float* dst);
int fg_c2f_zero_grads(fg_c2f* n, int net);
float* fg_c2f_params_ptr(fg_c2f* n, int net);
float* fg_c2f_grads_ptr(fg_c2f* n, int net);
int fg_c2f_set_adam_state(fg_c2f* n, int net, const float* m, const float* v, int t);
int fg_c2f_get_adam_state(fg_c2f* n, int net, float* m, float* v, int* t);
/* MODEL_G:forward({noise, cond}): noise [B][1][32][32], cond (coarse image) [B][C][32][32]
 * -> generated diff [B][C][32][32] (may be NULL).  backward accumulates into G's grad buffer.    */
int fg_c2f_G_forward(fg_c2f* n, const float* noise, const float* cond, int B, float* diff_out);
int fg_c2f_G_backward(fg_c2f* n, const float* d_diff);
/* MODEL_D:forward({diff, cond}) -> [B] sigmoid outputs; masks [B][16896] nn.Dropout keep flags
 * or NULL (drawn from seed); training=0 => evaluate().  d_diff = MODEL_D.gradInput[1].           */
int fg_c2f_D_forward(fg_c2f* n, const float* diff, const float* cond, int B, int training, const float* masks,
                     uint64_t seed, float* out);
int fg_c2f_D_backward(fg_c2f* n, const float* d_out, int want_wgrad, float* d_diff);
/* one adversarial_c2f.lua:121-187 loop body (1 D iteration + 1 G iteration, optim.adam for both):
 * real_diff [B/2][C][32][32] (fine - coarse of the real half), cond_D [B][C][32][32] (rows < B/2
 * go with the real half, the rest feed G), noise_D [B/2][1][32][32], cond_G / noise_G [B] redrawn
 * for the G step, masks_* [B][16896] or NULL.  h->D_maxAcc / accs_interval are ignored (the c2f
 * loop has no accuracy gate).                                                                     */
int fg_c2f_train_step(fg_c2f* n, const fg_hyper* h, int B, const float* real_diff, const float* cond_D,
                      const float* noise_D, const float* cond_G, const float* noise_G, const float* masks_D,
                      const float* masks_G, uint64_t seed, fg_step_stats* stats);

/* ---- the --scale 16 nets (train.lua --scale 16; models.lua:87-104 pick them for 16x16 images) ---- */
/* G = models.lua:27-51 create_G_decoder_upsampling16 (the 32x32 generator with every spatial size halved),
 * D = models.lua:279-316 create_D16_d (conv branch with two stride-2 convolutions + dense branch, ConcatTable ->
 * JoinTable -> Linear(1152,1) -> Sigmoid), loop = adversarial.lua:83-288 incl. the accuracy gate and the
 * interruptable optimizers.  Same object model as fg_c2f (borrows the ctx; destroy it before the ctx).  Flat
 * parameter vectors in getParameters() order: G [L1W L1b a1 C1W C1b g1 be1 a2 C2W C2b g2 be2 a3 C3W C3b],
 * D [c1W c1b a1 .. c4W c4b a4 F1W F1b af E1W E1b ae1 E2W E2b ae2 JW Jb].                                  */
typedef struct fg_s16 fg_s16;
int fg_s16_create(fg_ctx* ctx, fg_s16** out);
int fg_s16_destroy(fg_s16* n);
int64_t fg_s16_param_count(int net, int channels);
int fg_s16_mask_per_sample(void);                         /* 1152 = 1024 SpatialDropout planes + 128 Dropout */
int fg_s16_set_params(fg_s16* n, int net, const float* src);
int fg_s16_get_params(fg_s16* n, int net, float* dst);
int fg_s16_get_grads(fg_s16* n, int net, float* dst);
int fg_s16_zero_grads(fg_s16* n, int net);
float* fg_s16_params_ptr(fg_s16* n, int net);
float* fg_s16_grads_ptr(fg_s16* n, int net);
int fg_s16_set_adam_state(fg_s16* n, int net, const float* m, const float* v, int t);
int fg_s16_get_adam_state(fg_s16* n, int net, float* m, float* v, int* t);
int fg_s16_set_bn_state(fg_s16* n, const float* src768);  /* [mean1 256][var1 256][mean2 128][var2 128]   */
int fg_s16_get_bn_state(fg_s16* n, float* dst768);
/* noise [B][100] -> images [B][C][16][16] (may be NULL); training=0 => evaluate() (running statistics).
 * backward accumulates into G's grad buffer; d_noise [B][100] may be NULL.                                */
int fg_s16_G_forward(fg_s16* n, const float* noise, int B, int training, float* img_out);
int fg_s16_G_backward(fg_s16* n, const float* d_img, float* d_noise);
/* images [B][C][16][16] -> [B] sigmoid outputs; masks [B][1152] keep flags or NULL (drawn from seed).     */
int fg_s16_D_forward(fg_s16* n, const float* img, int B, int training, const float* masks, uint64_t seed, float* out);
int fg_s16_D_backward(fg_s16* n, const float* d_out, int want_wgrad, float* d_img);
/* fg_train_step on the 16x16 nets: real [B/2][C][16][16], noise_D [B/2][100], noise_G [B][100],
 * masks_* [B][1152] or NULL.                                                                              */
int fg_s16_train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                      const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats);

/* ---- device-resident dataset and on-GPU batch assembly ---------------------------------------- */
/* Replaces dataset.lua:80-117 (image.load(path, nbChannels, "float") + image.scale(img, 32, 32)) and
 * the per-sample batch loop of adversarial.lua:244-249 for the train step's input side: the DECODED
 * images stay on the GPU as uint8 [N][Cs][Hs][Ws] (planar, 0..255; dataset.originalScale = 64) and
 * one kernel produces the normalised, re-scaled fp32 batch.  Cs = 3 with a 1-channel ctx applies
 * image.rgb2y.  Scaling follows image.scale's default mode (area average when shrinking, linear
 * interpolation when enlarging).                                                                  */
typedef struct fg_dataset fg_dataset;
int fg_dataset_create(fg_ctx* ctx, int64_t N, int Cs, int Hs, int Ws, fg_dataset** out);
int fg_dataset_destroy(fg_dataset* d);
int64_t fg_dataset_size(fg_dataset* d);
int fg_dataset_upload(fg_dataset* d, int64_t first, int64_t count, const uint8_t* images);
/* out [B][C][32][32] (host or device) for B 0-based indices (host or device int32)              */
int fg_dataset_gather(fg_dataset* d, const int32_t* idx, int B, float* out);
/* the counter-based streams fg_train_step_dataset draws from: B indices in [0,N) / n floats in
 * [-1,1) (NN_UTILS.createNoiseInputs, utils/nn_utils.lua:35-39); outputs host or device           */
int fg_dataset_draw(fg_dataset* d, uint64_t seed, int B, int32_t* idx_out);
int fg_noise_uniform(fg_ctx* ctx, uint64_t seed, int64_t n, float* out);
/* fg_train_step with every input produced on the device: real = gather(draw(4*seed, B/2)),
 * noise_D = uniform(4*seed+1), noise_G = uniform(4*seed+2), dropout masks from `seed`             */
int fg_train_step_dataset(fg_ctx* ctx, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats);

/* ---- scoring helpers of the sampler / the c2f trainer ------------------------------------------ */
/* device part of NN_UTILS.sortImagesByPrediction (utils/nn_utils.lua:90-98; sample.lua:84-85):
 * D's prediction for N images [N][C][32][32], `chunk` (= OPT.batchSize) at a time.  training=1 is
 * what sample.lua does (it never calls evaluate(): dropout live, masks from seed), 0 = evaluate(). */
int fg_D_score(fg_ctx* ctx, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out);
/* brute-force nearest neighbour by torch.dist (2-norm): for each of Q queries [Q][D] the index of
 * the closest of N candidates [N][D] and the distance (D <= 3072); ties -> lowest index            */
int fg_nearest(fg_ctx* ctx, const float* queries, int Q, const float* cands, int64_t N, int D, int32_t* idx_out,
               float* dist_out);
/* findClosestNeighboursOf (sample.lua:141-159) against the device-resident training set            */
int fg_dataset_nearest(fg_dataset* d, const float* queries, int Q, int32_t* idx_out, float* dist_out);
/* one sample of adversarial_c2f.lua:305-325 approxParzen: min_k || G({noise_k, coarse}) + coarse - fine ||,
 * noise [K][1][32][32], coarse / fine [C][32][32]                                                   */
int fg_c2f_parzen_dist(fg_c2f* n, const float* noise, const float* coarse, const float* fine, int K, float* dist_out);

/* ---- Torch7 checkpoint files (host only, no GPU needed) --------------------------------------- */
/* Reads the binary torch.save format of the reference's checkpoints -- torch.save(filename,
 * {D=MODEL_D, G=MODEL_G, opt=OPT, epoch=EPOCH}) at adversarial.lua:328 / adversarial_c2f.lua:216,
 * read back by sample.lua:251-258 and train.lua:104-124 -- and writes files stock torch.load
 * reads.  `path` arguments are dotted keys from the root table ("G", "opt.batchSize", "epoch",
 * "G.modules.2"); numeric segments index array parts.  CudaTensor/CudaStorage are read as float. */
typedef struct fg_t7 fg_t7;
int fg_t7_open(const char* path, fg_t7** out);
int fg_t7_close(fg_t7* f);
/* 0 nil, 1 number, 2 string, 3 table, 4 torch object (nn module ...), 5 boolean, 6 function,
 * 16 tensor, 17 storage; -1 when the path does not exist                                         */
int fg_t7_kind(fg_t7* f, const char* path);
int fg_t7_number(fg_t7* f, const char* path, double* out);
/* string value, or the class name of a torch object ("nn.Sequential"); returns its length or -1  */
int64_t fg_t7_string(fg_t7* f, const char* path, char* dst, int64_t cap);
/* tensor as row-major floats (strides/offset honoured); dst may be NULL (count only); dims8 may
 * be NULL or receives up to 8 sizes (0-terminated).  Returns the element count or -1.            */
int64_t fg_t7_tensor(fg_t7* f, const char* path, float* dst, int64_t cap, int64_t* dims8);
/* flat parameter vector of the nn module tree at `path` in MODEL:getParameters() order
 * (train.lua:151-152: module order, weight then bias; containers incl. the nn.Copy wrappers of
 * NN_UTILS.activateCuda are walked through) -- ready for fg_set_params / fg_c2f_set_params.      */
int64_t fg_t7_net_params(fg_t7* f, const char* path, float* dst, int64_t cap);
/* BatchNorm running statistics per BN layer in module order: running_mean[C], running_var[C]
 * (a 2015-era running_std is converted) -- for G this is the fg_set_bn_state layout.             */
int64_t fg_t7_net_bn_state(fg_t7* f, const char* path, float* dst, int64_t cap);
/* class-name skeleton, e.g. "nn.Sequential{nn.Copy,nn.Sequential{nn.Linear,...},nn.Copy}"       */
int64_t fg_t7_net_describe(fg_t7* f, const char* path, char* dst, int64_t cap);
/* writer: ONE root table {key = torch.FloatTensor | number | string}.  Used to export flat
 * parameter / Adam-state vectors (the reference drops its optimizer state, train.lua:122); a
 * Torch host restores them with PARAMETERS_G:copy(file.G) after MODELS.create_G().               */
typedef struct fg_t7_writer fg_t7_writer;
int fg_t7_writer_open(const char* path, fg_t7_writer** out);
int fg_t7_writer_add_tensor(fg_t7_writer* w, const char* key, const float* data, const int64_t* dims, int ndim);
int fg_t7_writer_add_number(fg_t7_writer* w, const char* key, double v);
int fg_t7_writer_add_string(fg_t7_writer* w, const char* key, const char* s);
int fg_t7_writer_close(fg_t7_writer* w);                  /* writes the file and frees the writer   */

/* ---- data parallel: one process per GPU, NCCL over NVLink (new functionality, SURVEY 8e) ----- */
int fg_dp_unique_id(void* out128);                        /* ncclGetUniqueId, 128 bytes           */
int fg_dp_init(fg_ctx* ctx, const void* id128, int nranks, int rank);
/* rank 0's G/D parameters, optimizer moments, BN running statistics, step counters (t_D, t_G) and
 * the D-accuracy history to all ranks -- call after loading a checkpoint on rank 0               */
int fg_dp_broadcast_params(fg_ctx* ctx);
int fg_c2f_dp_broadcast_params(fg_c2f* n);                /* same for the coarse-to-fine nets      */
int fg_s16_dp_broadcast_params(fg_s16* n);                /* same for the --scale 16 nets          */
int fg_dp_world(fg_ctx* ctx);                             /* nranks (1 when DP is off)            */

/* ---- plain device-memory helpers for FFI hosts without a CUDA binding ------------------------ */
void* fg_dev_alloc(size_t bytes);
int fg_dev_free(void* p);
void* fg_host_alloc_pinned(size_t bytes);
int fg_host_free_pinned(void* p);
int fg_memcpy(fg_ctx* ctx, void* dst, const void* src, size_t bytes);   /* any direction, on ctx stream */

/* ---- introspection used by tests / bench ------------------------------------------------------ */
int64_t fg_kernel_launches(fg_ctx* ctx);                  /* kernels launched by this ctx so far   */
/* copy an internal activation (NHWC) to dst: names "G.z0","G.h0","G.z1","G.h1","G.z2","G.h2","G.z3" */
int64_t fg_debug_tensor(fg_ctx* ctx, const char* name, float* dst, int64_t max_elems);
/* timing of the dominant kernel family inside the last fg_train_step (CUDA events on the ctx
 * stream): returns ms in out[0..n) for the names in fg_timing_names(); 0 when not enabled.       */
/* whole-step timing on the ctx stream: record CUDA event `slot` (0..15), elapsed ms between two. */
int fg_event_record(fg_ctx* ctx, int slot);
int fg_event_elapsed_ms(fg_ctx* ctx, int slot_a, int slot_b, double* ms);
int fg_timing_enable(fg_ctx* ctx, int on);
/* tensor-pipe probe for the roofline: TFLOP/s of back-to-back tf32 wgmmas (two warpgroups of M=64,N=256,K=8 per
 * SM, operands resident in shared memory) on all SMs, best of 5 event-timed launches of `iters` x 4 MMAs per SM */
int fg_bench_tf32_peak(fg_ctx* ctx, int iters, double* tflops);
int fg_timing_get(fg_ctx* ctx, const char* name, double* ms_total, int64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* FG_B200_H */
