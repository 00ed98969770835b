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
 * after writing through fg_params_ptr), "bwd_streams" (1, the default: the weight gradients of the 32x32 D
 * and of G.C3 and G.C1 run on a second stream beside the data-gradient chain of the backward, same bits; 0: one
 * stream); unknown keys return FG_ERR_INVALID
 *
 * Read-only keys of fg_get_option: which kernel the last fg_conv2d_* / fg_scu_* / fg_linear_* call launched
 * (a call launches one: forward, data gradient or weight gradient; fg_linear_backward with both dx and dw
 * records the weight gradient).  All 0 after a call that launched none (a refused one).
 *   "last_conv_kind"     FG_KERNEL_*
 *   "last_conv_tile_m"   TAPCONV: 128 (pixels)  WGRAD_TC: 128 (Cout)  EDGE_REDUCE: NS (outputs)
 *                        EDGE_EXPAND: CS (inputs)  SIMT / SIMT_FLATK / WGRAD_SIMT: TM (rows per thread)
 *   "last_conv_tile_n"   TAPCONV / WGRAD_TC: BN  EDGE_REDUCE: VEC (channels per lane)
 *                        EDGE_EXPAND: N (outputs)  SIMT / SIMT_FLATK / WGRAD_SIMT: TN (columns per thread)
 *   "last_conv_format"   0 fp32 FFMA, 1 3xTF32 tensor cores, 2 3xFP16 tensor cores
 *   "last_conv_splits"   K splits of a weight gradient (1: unsplit, written straight to its output);
 *                        1 for every other kernel
 * and how many train steps on this context, of any of its nets, ran as a launch of a captured CUDA graph:
 *   "step_graph_launches"                                                                             */
enum {
  FG_KERNEL_NONE = 0,
  FG_KERNEL_TAPCONV = 1,      /* wgmma forward / data gradient (tapconv_tc_kernel)                   */
  FG_KERNEL_WGRAD_TC = 2,     /* wgmma weight gradient (wgrad_tc_kernel)                             */
  FG_KERNEL_EDGE_REDUCE = 3,  /* 3x3, W = 32, 64 / 128 -> 1 / 3 channels (conv_reduce_kernel)         */
  FG_KERNEL_EDGE_EXPAND = 4,  /* 3x3, W = 32, 1 / 3 / 4 -> 64 / 128 channels (conv_expand_kernel)     */
  FG_KERNEL_SIMT = 5,         /* FFMA implicit GEMM (conv_simt_kernel)                               */
  FG_KERNEL_SIMT_FLATK = 6,   /* FFMA, taps x channels flattened for Cin < 16 (conv_simt_flatk_kernel) */
  FG_KERNEL_WGRAD_SIMT = 7    /* FFMA weight gradient (wgrad_simt_kernel)                            */
};
int fg_set_option(fg_ctx* ctx, const char* key, int64_t value);
int64_t fg_get_option(fg_ctx* ctx, const char* key);
int fg_set_option_f(fg_ctx* ctx, const char* key, double value);    /* "sgd_momentum_D", "sgd_momentum_G"     */

/* ---- discriminators: the D of the 32x32 nets (fg_create_disc) and of the --scale 16 nets (fg_s16_create_disc) ----
 * models.lua defines six; create_D picks FG_DISC_D32B at 32x32 and FG_DISC_D16_D at 16x16 (the nets' defaults,
 * which fg_create / fg_s16_create build).  The other four are the three-branch nets (3x3 conv branch, 5x5 conv branch,
 * dense branch -> JoinTable(2) -> Linear -> PReLU -> Dropout -> Linear(1) -> Sigmoid) the author trained against
 * before them.  All p = 0.5 dropouts; keep flags per sample in module order.  A D of the other side is refused with
 * FG_ERR_UNSUPPORTED before anything is allocated.                                                            */
enum {
  FG_DISC_DEFAULT = 0,  /* the size's own: D32B at 32x32, D16_D at 16x16                             */
  FG_DISC_D32B = 1,     /* models.lua:382-416 create_D32b  (32x32)                                    */
  FG_DISC_D16_D = 2,    /* models.lua:279-316 create_D16_d (16x16)                                    */
  FG_DISC_D32 = 3,      /* models.lua:322-376 create_D32   (32x32)                                    */
  FG_DISC_D16 = 4,      /* models.lua:110-159 create_D16   (16x16)                                    */
  FG_DISC_D16_B = 5,    /* models.lua:161-216 create_D16_b (16x16)                                    */
  FG_DISC_D16_C = 6     /* models.lua:218-277 create_D16_c (16x16)                                    */
};
/* fg_create with discriminator `disc` (FG_DISC_DEFAULT / D32B / D32)                                    */
int fg_create_disc(fg_ctx** out, int device, int max_batch, int channels, int disc);
int fg_get_disc(fg_ctx* ctx);                      /* FG_DISC_* of the 32x32 D (never DEFAULT); < 0 on error */
/* D's getParameters() length for 1 or 3 channels and its keep flags per sample; -1 for an unknown disc
 * (or FG_DISC_DEFAULT, which names no net by itself) or channel count                                    */
int64_t fg_disc_param_count(int disc, int channels);
int fg_disc_mask_per_sample(int disc);
int fg_disc_side(int disc);                        /* 32 or 16; 0 for an unknown disc                       */

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
 * [64|128|256|512] SpatialDropout + [512|512] Dropout (another D: [B][fg_disc_mask_per_sample(D)], module order);
 * NULL => drawn in-kernel from `seed`.
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
 * grad_scale multiplies the gradient first (1/N for DP).  The step is never gated: it advances t
 * of `net` and steps it, and leaves D's accuracy history, conf, acc_D and trained_D as the last
 * fused step left them (a module-level step has no batch accuracy; adversarial.lua's gate only
 * sees the fused steps' accuracies).  The clamp is fminf(fmaxf(g, -c), c): a NaN gradient element
 * becomes -c under a clamp (Torch's CPU clamp keeps the NaN) and stays NaN without one.          */
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
/* G = models_c2f.lua:113-145 create_G_d, D = models_c2f.lua:237-278 create_D_c (or another pair of
 * models_c2f.lua's nets, fg_c2f_create_nets), both at the fine size S = train_c2f.lua --fineSize (16, 32
 * or 64; fg_c2f_create: 32) on the ctx's channel count.
 * Every image, noise and mask buffer below is at the net's S: images [B][C][S][S], noise
 * [B][1][S][S], masks [B][fg_c2f_disc_mask_per_sample(D, S)].  cudnn.SpatialConvolutionUpsample with
 * factor 1 (layers/cudnnSpatialConvolutionUpsample.lua) is a "same" convolution.  The object borrows the
 * ctx (stream, device, DP communicator, "conv_impl"); destroy it before the ctx.  Flat parameter
 * vectors follow getParameters() order: G [c1W c1b a1 ... c4W c4b a4 c5W c5b], D [c1W c1b a1 ...
 * c4W c4b a4 L1W L1b a5 L2W L2b] (create_G_d / create_D_c; the other nets the same per layer).       */
typedef struct fg_c2f fg_c2f;
int fg_c2f_create(fg_ctx* ctx, fg_c2f** out);            /* fg_c2f_create_sized(ctx, 32, out)      */
/* fg_c2f_create_nets(ctx, fine_size, FG_C2F_G_DEFAULT, FG_C2F_D_DEFAULT, out); any fine size other
 * than 16, 32, 64 -> FG_ERR_UNSUPPORTED before anything is allocated                               */
int fg_c2f_create_sized(fg_ctx* ctx, int fine_size, fg_c2f** out);
int fg_c2f_fine_size(fg_c2f* n);
int fg_c2f_destroy(fg_c2f* n);
int64_t fg_c2f_param_count(int net, int channels);        /* 1 101 319 / 8 797 382 for colour      */
int fg_c2f_mask_per_sample(void);                         /* 16896 = [256][8][8] + [512] nn.Dropout */
/* at fine size S: G unchanged, D's Linear 256*(S/4)^2 -> 512 (colour D: 2 505 926 at 16, 33 963 206
 * at 64); keep flags [256][S/4][S/4] + [512] (4608 / 16896 / 66048); -1 for an unsupported size.
 * These four always describe the default pair, create_G_d / create_D_c.                            */
int64_t fg_c2f_param_count_sized(int net, int channels, int fine_size);
int fg_c2f_mask_per_sample_sized(int fine_size);
/* models_c2f.lua's generators and discriminators; create_G / create_D pick create_G_d / create_D_c     */
enum {
  FG_C2F_G_DEFAULT = 0, /* create_G_d                                                               */
  FG_C2F_G_D = 1,       /* models_c2f.lua:113-145 create_G_d (64,3) (64,3) (128,5) (256,5) (C,7)    */
  FG_C2F_G_A = 2,       /* models_c2f.lua:16-45   create_G_a (64,3) (128,7) (C,5)                   */
  FG_C2F_G_B = 3,       /* models_c2f.lua:47-78   create_G_b (64,3) (64,3) (256,5) (C,7)            */
  FG_C2F_G_C = 4        /* models_c2f.lua:80-111  create_G_c (64,3) (128,3) (256,5) (C,7)           */
};
enum {
  FG_C2F_D_DEFAULT = 0, /* create_D_c                                                               */
  FG_C2F_D_C = 1,       /* models_c2f.lua:237-278 create_D_c 64, 64 pool, 128, 256 pool             */
  FG_C2F_D_A = 2,       /* models_c2f.lua:156-192 create_D_a 64, 64 pool                            */
  FG_C2F_D_B = 3        /* models_c2f.lua:194-235 create_D_b 64, 64 pool, 128, 128 pool             */
};
/* the c2f nets with generator `gen` (FG_C2F_G_*) and discriminator `disc` (FG_C2F_D_*); an unknown net
 * or fine size -> FG_ERR_UNSUPPORTED before anything is allocated.  Every fg_c2f_* entry point then
 * follows that pair: parameter vectors fg_c2f_gen_param_count / fg_c2f_disc_param_count long, keep
 * flags fg_c2f_disc_mask_per_sample wide.                                                           */
int fg_c2f_create_nets(fg_ctx* ctx, int fine_size, int gen, int disc, fg_c2f** out);
int fg_c2f_get_gen(fg_c2f* n);                   /* FG_C2F_G_* of G (never DEFAULT); < 0 on error       */
int fg_c2f_get_disc(fg_c2f* n);                  /* FG_C2F_D_* of D (never DEFAULT); < 0 on error       */
/* getParameters() lengths and D's keep flags per sample (the pooled map View flattens, in NCHW order,
 * then [512]); no GPU needed; -1 for an unknown net, a channel count < 1 or an unsupported fine size  */
int64_t fg_c2f_gen_param_count(int gen, int channels);
int64_t fg_c2f_disc_param_count(int disc, int channels, int fine_size);
int fg_c2f_disc_mask_per_sample(int disc, int fine_size);
int fg_c2f_set_params(fg_c2f* n, int net, const float* src);
int fg_c2f_get_params(fg_c2f* n, int net, float* dst);
int fg_c2f_get_grads(fg_c2f* n, int net, float* dst);
int fg_c2f_zero_grads(fg_c2f* n, int net);
float* fg_c2f_params_ptr(fg_c2f* n, int net);
float* fg_c2f_grads_ptr(fg_c2f* n, int net);
int fg_c2f_set_adam_state(fg_c2f* n, int net, const float* m, const float* v, int t);
int fg_c2f_get_adam_state(fg_c2f* n, int net, float* m, float* v, int* t);
/* MODEL_G:forward({noise, cond}): noise [B][1][S][S], cond (coarse image) [B][C][S][S]
 * -> generated diff [B][C][S][S] (may be NULL).  backward accumulates into G's grad buffer.    */
int fg_c2f_G_forward(fg_c2f* n, const float* noise, const float* cond, int B, float* diff_out);
int fg_c2f_G_backward(fg_c2f* n, const float* d_diff);
/* MODEL_D:forward({diff, cond}) -> [B] sigmoid outputs; masks [B][mask_per_sample] keep flags
 * or NULL (drawn from seed); training=0 => evaluate().  d_diff = MODEL_D.gradInput[1].           */
int fg_c2f_D_forward(fg_c2f* n, const float* diff, const float* cond, int B, int training, const float* masks,
                     uint64_t seed, float* out);
int fg_c2f_D_backward(fg_c2f* n, const float* d_out, int want_wgrad, float* d_diff);
/* one adversarial_c2f.lua:121-187 loop body (1 D iteration + 1 G iteration, optim.adam for both):
 * real_diff [B/2][C][S][S] (fine - coarse of the real half), cond_D [B][C][S][S] (rows < B/2
 * go with the real half, the rest feed G), noise_D [B/2][1][S][S], cond_G / noise_G [B] redrawn
 * for the G step, masks_* [B][mask_per_sample] or NULL.  h->D_maxAcc / accs_interval are ignored (the c2f
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
/* fg_s16_create with discriminator `disc` (FG_DISC_DEFAULT / D16_D / D16 / D16_B / D16_C); masks and D's parameter
 * vector of every fg_s16_* entry point then follow that D (fg_disc_param_count / fg_disc_mask_per_sample)      */
int fg_s16_create_disc(fg_ctx* ctx, int disc, fg_s16** out);
int fg_s16_get_disc(fg_s16* n);                  /* FG_DISC_* of D (never DEFAULT); < 0 on error           */
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
/* images [B][C][16][16] -> [B] sigmoid outputs; masks [B][fg_disc_mask_per_sample(D)] keep flags (1152 for
 * create_D16_d) or NULL (drawn from seed).                                                                */
int fg_s16_D_forward(fg_s16* n, const float* img, int B, int training, const float* masks, uint64_t seed, float* out);
int fg_s16_D_backward(fg_s16* n, const float* d_out, int want_wgrad, float* d_img);
/* fg_train_step on the 16x16 nets: real [B/2][C][16][16], noise_D [B/2][100], noise_G [B][100],
 * masks_* [B][fg_disc_mask_per_sample(D)] (1152 for create_D16_d) or NULL.                                 */
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
/* the inverse of fg_dataset_upload: rows [first, first+count) into out (host or device), [count][Cs][Hs][Ws]  */
int fg_dataset_download(fg_dataset* d, int64_t first, int64_t count, uint8_t* out);
/* JPEG files straight into the cache (dataset.lua loadImagesFromDirs' image.load(path, Cs, 'byte')).
 * Supported: baseline / extended sequential Huffman (SOF0, SOF1), 8-bit, one scan holding every
 * component, 1 or 3 components, luma sampled 1x1, 2x1 or 2x2 with 1x1 chroma (4:4:4, 4:2:2, 4:2:0),
 * DRI restarts; APPn / COM segments are skipped.  The output equals libjpeg-turbo's default
 * decompression (islow IDCT, fancy upsampling) bit for bit.
 * fg_jpeg_info: host only, needs no GPU; C, H, W of a file from its markers (any may be NULL).  A
 * file outside the scope above is FG_ERR_UNSUPPORTED, a malformed header FG_ERR_INVALID, and
 * fg_last_error names the reason.
 * fg_dataset_upload_jpeg: file i = bytes[offsets[i] .. offsets[i+1]) (offsets has count+1 entries,
 * host memory) goes to row first+i, planar [Cs][Hs][Ws]; a 1-component file under Cs = 3 is
 * replicated to three planes, a 3-component file under Cs = 1 is refused.  Every header is checked
 * before anything is launched; a size other than Hs x Ws, an unsupported format or corrupt /
 * truncated entropy-coded data returns an error with *failed_out (may be NULL) = the index i of the
 * first failing file (a header failure is reported before any decode), else -1.  After an error the
 * rows [first, first+count) are unspecified.  Runs in bounded chunks on the ctx stream; returns once
 * the host buffers may be reused.                                                                  */
int fg_jpeg_info(const uint8_t* bytes, int64_t len, int* C, int* H, int* W);
int fg_dataset_upload_jpeg(fg_dataset* d, int64_t first, int64_t count, const uint8_t* bytes, const int64_t* offsets,
                           int64_t* failed_out);
/* The other direction (dataset/generate_dataset.py's misc.imsave): rows [first, first+count) as
 * baseline JFIF files, byte for byte what Pillow's Image.save(f, "JPEG", quality=quality) writes for
 * them (3 planes: YCbCr 4:2:0; 1 plane: grayscale; standard Huffman tables, no restart markers).
 * quality 1..100; any size the cache holds.
 * fg_dataset_encode_jpeg: offsets[count+1] (host) is always filled: file i = out[offsets[i] ..
 * offsets[i+1]).  If offsets[count] > cap, nothing is written to out and the call returns
 * FG_ERR_INVALID (the caller retries with that size); out may be NULL to ask for the sizes only.
 * out may be host or device memory.
 * fg_dataset_jpeg_roundtrip: rows [first, first+count) replaced in place by decode(encode(row,
 * quality)), what fg_dataset_upload_jpeg gives on fg_dataset_encode_jpeg's files, without leaving
 * the device.
 * An out-of-range span, a quality outside 1..100 or a NULL offsets is FG_ERR_INVALID and launches
 * nothing.  Both run in bounded chunks on the ctx stream and return once the work is done.          */
int fg_dataset_encode_jpeg(fg_dataset* d, int64_t first, int64_t count, int quality, uint8_t* out, int64_t cap,
                           int64_t* offsets);
int fg_dataset_jpeg_roundtrip(fg_dataset* d, int64_t first, int64_t count, int quality);
/* The same encoder on caller images (image.save(path, img) of sample.lua's sheets): count images
 * planar uint8 [count][C][H][W] (host or device), C = 1 or 3, 1 <= H, W <= 4096, quality 1..100 ->
 * baseline JFIF files byte for byte what Pillow's Image.save(f, "JPEG", quality=quality) writes
 * (4:2:0 colour, grayscale for C = 1).  offsets / cap / out: fg_dataset_encode_jpeg's contract.
 * Bad arguments are FG_ERR_INVALID and launch nothing.  Files of 2048 blocks or more (about 256x256
 * colour) are entropy-coded by many CTAs each, smaller ones by one CTA each; fg_set_option(ctx,
 * "jpeg_route", 1 | 2) forces one route for every encode on the ctx (tests only: same bytes).      */
int fg_jpeg_encode(fg_ctx* ctx, const uint8_t* images, int count, int C, int H, int W, int quality, uint8_t* out,
                   int64_t cap, int64_t* offsets);
/* image.toDisplayTensor{input=images[order[0..count)], nrow=nrow, padding=padding} followed by
 * image.saveJPG's clampImage (saturate to [0,1], *255, to bytes): planar uint8 [C][Hg][Wg] with
 * Hg = ceil(count / xmaps) * (H + padding), Wg = xmaps * (W + padding), xmaps = min(nrow, count).
 * images [N][C][H][W] float, host or device; order int32 [count] (host or device, NULL = 0..count-1;
 * host entries are range-checked, device ones clamped to [0, N)); out host or device, or NULL to ask
 * for Hg / Wg only (Hg_out / Wg_out may be NULL).  Cells outside an image hold the largest value of
 * the selected images; the grid is then normalised by image.minmax over those images.  NaN values
 * take no part in the minimum and maximum and give byte 0.  1 <= C <= 3, padding even and >= 0,
 * Hg, Wg <= 4096, nrow >= 1; anything else is FG_ERR_INVALID and launches nothing.               */
int fg_image_grid(fg_ctx* ctx, const float* images, int64_t N, int C, int H, int W, const int32_t* order, int count,
                  int nrow, int padding, uint8_t* out, int* Hg_out, int* Wg_out);
/* The augmented LFW training set (dataset/generate_dataset.py + ImageAugmenter.py): each output row
 * is LFW-crop's 84x84 box (rows 92..175, cols 83..166) of a source row, resized to the destination's
 * Ho x Wo as Pillow's Image.resize(BILINEAR) does (scipy.misc.imresize).  A descriptor with warp = 1
 * first flips the source horizontally (hflip = 1), scales it by `brightness` with truncation to
 * uint8, and warps it as skimage.transform.warp(img, m, mode="constant") at order 1: m is the
 * row-major 3x3 INVERSE map from output (x = col, y = row) to input coordinates, evaluated in
 * float64 without FMA contraction, bilinear taps outside the image read 0, the result is clipped to
 * the brightened source's [min, max] (exact zeros kept when min > 0) and truncated to uint8.  warp = 0
 * is the photo itself: crop and resize only (hflip, brightness and m are ignored).
 * fg_lfw_aug_params: host only, needs no GPU.  Fills n_src * (1 + n_aug) descriptors: row
 * (i - first_src) * (1 + n_aug) + a for source photo i in [first_src, first_src + n_src) and a in
 * [0, n_aug]; src = i, a = 0 is warp = 0, a >= 1 draws generate_dataset.py's distributions (scale
 * U[0.82, 1.10) on both axes, integer degrees in [-8, 8], integer translations in [-5, 5], hflip
 * with p = 1/2, brightness U[0.9, 1.1)) from counter-based streams keyed by (seed, i, a), so a slice
 * gives the same descriptors as the whole.  m = inverse of T(+shift) A T(-shift) with shift =
 * (src_h / 2, src_w / 2) for (x, y) (the reference's width/height swap), third row [0, 0, 1].
 * fg_dataset_augment: rows [dst_first, dst_first + n) of dst from the descriptors augs[0..n) (host
 * memory), on the ctx stream; returns when the rows are written.  Refused before anything is
 * launched (FG_ERR_INVALID, fg_last_error names the reason): caches on different contexts,
 * different channel counts, a source smaller than 176 x 167, a destination side outside [1, 84], a
 * descriptor whose src is out of range, whose warp / hflip is not 0 or 1, whose brightness is not
 * finite and >= 0 or whose m is not finite.                                                          */
typedef struct fg_aug {
  int64_t src;
  int32_t warp, hflip;
  double brightness;
  double m[9];
} fg_aug;
int fg_lfw_aug_params(uint64_t seed, int64_t first_src, int64_t n_src, int n_aug, int src_h, int src_w, fg_aug* out);
int fg_dataset_augment(fg_dataset* src, fg_dataset* dst, int64_t dst_first, const fg_aug* augs, int64_t n);
/* out [B][C][32][32] (host or device) for B 0-based indices (host or device int32)              */
int fg_dataset_gather(fg_dataset* d, const int32_t* idx, int B, float* out);
/* the counter-based streams fg_train_step_dataset draws from: B indices in [0,N) / n floats in
 * [-1,1) (NN_UTILS.createNoiseInputs, utils/nn_utils.lua:35-39); outputs host or device           */
int fg_dataset_draw(fg_dataset* d, uint64_t seed, int B, int32_t* idx_out);
int fg_noise_uniform(fg_ctx* ctx, uint64_t seed, int64_t n, float* out);
/* fg_train_step with every input produced on the device: real = gather(draw(4*seed, B/2)),
 * noise_D = uniform(4*seed+1), noise_G = uniform(4*seed+2), dropout masks from `seed`             */
int fg_train_step_dataset(fg_ctx* ctx, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats);
/* image.scale(image.load(...), size, size) (dataset.lua with setScale(size)) for B indices:
 * out [B][C][size][size], 1 <= size <= 32; size 32 is fg_dataset_gather                           */
int fg_dataset_gather_sized(fg_dataset* d, const int32_t* idx, int B, int size, float* out);
/* dataset_c2f.lua:49-62 _toResult for B indices at fineSize 32: fine = fg_dataset_gather(idx),
 * coarse = scale(scale(fine, cs, cs), 32, 32), diff = fine - coarse; [B][C][32][32] each, host or
 * device, any may be NULL; 1 <= coarse_size (train_c2f.lua --coarseSize) <= 32                     */
int fg_dataset_gather_c2f(fg_dataset* d, const int32_t* idx, int B, int coarse_size, float* fine, float* coarse,
                          float* diff);
/* the same at fineSize S in {16, 32, 64} (others: FG_ERR_UNSUPPORTED): fine = scale(image, S, S),
 * coarse = scale(scale(fine, cs, cs), S, S), diff = fine - coarse, [B][C][S][S] each; 1 <= cs <= S.
 * fine_size 32 is fg_dataset_gather_c2f.                                                           */
int fg_dataset_gather_c2f_sized(fg_dataset* d, const int32_t* idx, int B, int fine_size, int coarse_size, float* fine,
                                float* coarse, float* diff);
/* fg_s16_train_step (train.lua --scale 16) with every input produced on the device:
 * real = gather_sized(draw(4*seed, B/2), 16), noise_D = uniform(4*seed+1), noise_G = uniform(4*seed+2),
 * dropout masks from `seed` (the streams of fg_train_step_dataset).  d must belong to n's ctx.     */
int fg_s16_train_step_dataset(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats);
/* fg_c2f_train_step (one adversarial_c2f.lua:121-187 loop body) with every input produced on the device
 * (the draws of adversarial_c2f.lua:124-141 and :168-174):
 *   real pairs  = gather_c2f_sized(draw(8*seed,   B/2), S) -> real_diff, cond_D rows [0, B/2)
 *   fake cond   = gather_c2f_sized(draw(8*seed+1, B/2), S) -> cond_D rows [B/2, B)
 *   G-step cond = gather_c2f_sized(draw(8*seed+2, B), S)   -> cond_G
 *   noise_D = uniform(8*seed+3, B/2*S*S), noise_G = uniform(8*seed+4, B*S*S), dropout masks from `seed`.
 * coarse_size = train_c2f.lua --coarseSize (1..S).  d must belong to n's ctx.                         */
int fg_c2f_train_step_dataset(fg_c2f* n, fg_dataset* d, const fg_hyper* h, int B, int coarse_size, uint64_t seed,
                              fg_step_stats* stats);

/* ---- several D and G iterations per call (train.lua / train_c2f.lua --D_iterations, --G_iterations) ---- */
/* One call runs d_iters D iterations, then g_iters G iterations (adversarial.lua:240-288,
 * adversarial_c2f.lua:121-187), as one captured step.  D iteration j draws its own fakes from a
 * training-mode G forward (G's BatchNorm running statistics move once per D iteration), runs D
 * forward/backward, BCE, penalty, clamp and, for the 32x32 and 16x16 nets, the accuracy gate on its own
 * accuracy, then its own optimizer step; iteration j+1 sees the D that iteration j left.  G iteration j
 * is a full G step with its own optimizer step.  Inputs are those of the single-iteration entries,
 * stacked per iteration: real [d][B/2][C][S][S], noise_D [d][B/2][..], noise_G [g][B][..], masks_D
 * [d][B][mask], masks_G [g][B][mask] (or NULL: drawn from the stream roots below), c2f cond_D [d][B][..],
 * cond_G [g][B][..].  1 <= d_iters, g_iters <= 16, anything else is FG_ERR_UNSUPPORTED before any work
 * (D_iterations = 0 is not supported).  The statistics of a call: conf sums over the D iterations,
 * trained_D counts the D iterations that stepped, loss_D / acc_D are those of the last D iteration,
 * loss_G that of the last G iteration, t_D / t_G the counters after the call.  With d_iters = g_iters = 1
 * a call is bit for bit the single-iteration entry.
 * Stream roots: iteration j of a call with step seed s draws from the root r_j, r_0 = s and
 * r_j = 2^60 | s << 8 | j for j >= 1 (64-bit arithmetic; distinct from every r_0 while s < 2^52).
 * Its dropout masks use the streams of seed r_j (2*r_j+1 for D iteration j, 2*r_j+2 for G iteration j);
 * the _dataset_iters entries draw D iteration j's real half from fg_dataset_draw(4*r_j) and its noise
 * from fg_noise_uniform(4*r_j+1), G iteration j's noise from fg_noise_uniform(4*r_j+2); c2f: real pairs
 * 8*r_j, fake cond 8*r_j+1 and noise_D 8*r_j+3 for D iteration j, G cond 8*r_j+2 and noise_G 8*r_j+4 for
 * G iteration j.  For j = 0 these are the streams of the single-iteration entries.                   */
int fg_train_step_iters(fg_ctx* ctx, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                        const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                        fg_step_stats* stats);
int fg_s16_train_step_iters(fg_s16* n, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real,
                            const float* noise_D, const float* noise_G, const float* masks_D, const float* masks_G,
                            uint64_t seed, fg_step_stats* stats);
int fg_c2f_train_step_iters(fg_c2f* n, const fg_hyper* h, int B, int d_iters, int g_iters, const float* real_diff,
                            const float* cond_D, const float* noise_D, const float* cond_G, const float* noise_G,
                            const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats);
/* every input drawn on the device, inside the step (one graph launch per call once captured)          */
int fg_train_step_dataset_iters(fg_ctx* ctx, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters, uint64_t seed,
                                fg_step_stats* stats);
int fg_s16_train_step_dataset_iters(fg_s16* n, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters,
                                    uint64_t seed, fg_step_stats* stats);
int fg_c2f_train_step_dataset_iters(fg_c2f* n, fg_dataset* d, const fg_hyper* h, int B, int d_iters, int g_iters,
                                    int coarse_size, uint64_t seed, fg_step_stats* stats);

/* ---- scoring helpers of the sampler / the c2f trainer ------------------------------------------ */
/* device part of NN_UTILS.sortImagesByPrediction (utils/nn_utils.lua:90-98; sample.lua:84-85):
 * D's prediction for N images [N][C][32][32], `chunk` (= OPT.batchSize) at a time.  training=1 is
 * what sample.lua does (it never calls evaluate(): dropout live, masks from seed), 0 = evaluate(). */
int fg_D_score(fg_ctx* ctx, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out);
/* brute-force nearest neighbour by torch.dist (2-norm): for each of Q queries [Q][D] the index of
 * the closest of N candidates [N][D] and the distance (D <= 12288 = 3x64x64); ties -> lowest index */
int fg_nearest(fg_ctx* ctx, const float* queries, int Q, const float* cands, int64_t N, int D, int32_t* idx_out,
               float* dist_out);
/* findClosestNeighboursOf (sample.lua:141-159) against the device-resident training set            */
int fg_dataset_nearest(fg_dataset* d, const float* queries, int Q, int32_t* idx_out, float* dist_out);
/* the same against the size x size view of every cached image (1 <= size <= 64; DATASET.setScale
 * then loadImages: fg_dataset_gather_sized's arithmetic), queries [Q][C][size][size];
 * fg_dataset_nearest is fg_dataset_nearest_sized(d, 32, ...)                                         */
int fg_dataset_nearest_sized(fg_dataset* d, int size, const float* queries, int Q, int32_t* idx_out, float* dist_out);
/* fg_D_score on the --scale 16 discriminator: images [N][C][16][16], same chunking and seeds        */
int fg_s16_D_score(fg_s16* n, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out);
/* one sample of adversarial_c2f.lua:305-325 approxParzen: min_k || G({noise_k, coarse}) + coarse - fine ||,
 * noise [K][1][S][S], coarse / fine [C][S][S]                                                       */
int fg_c2f_parzen_dist(fg_c2f* n, const float* noise, const float* coarse, const float* fine, int K, float* dist_out);
/* image.scale(x, Wo, Ho) (default 'bilinear' mode) on fp32 NCHW: src [N][C][Hs][Ws] -> dst [N][C][Ho][Wo],
 * host or device; 1 <= Hs, Ws, Ho, Wo <= 256                                                        */
int fg_image_scale(fg_ctx* ctx, const float* src, int64_t N, int C, int Hs, int Ws, int Ho, int Wo, float* dst);
/* sample.lua:176-214 c2f(images, G, D, fineSize) on the net's fine size S (the coarse-to-fine pyramid step):
 *   up[i]     = image.scale(images[i], S, S)                     (a copy when in_size == S)
 *   diff[i,t] = G({noise[i,t], up[i]}),  pred[i,t] = D({diff[i,t], up[i]})   t < tries
 *   pick[i]   = the first t with the largest float32 pred (strict >, as the reference's loop; a NaN never
 *               wins except at t = 0)
 *   out[i]    = up[i] + diff[i, pick[i]]                          (no clamp, as torch.add)
 * images [N][C][in_size][in_size], 1 <= in_size <= 64; out [N][C][S][S]; pick_out [N] (0-based) and
 * pred_out [N][tries] may be NULL; every buffer host or device.  `chunk` images (chunk*tries rows <=
 * max_batch) per pass.  training = 1 is what sample.lua does (D's dropout live), 0 = evaluate().
 * noise [N][tries][1][S][S] or NULL = fg_noise_uniform(ctx, 2*seed, N*tries*S*S) (same element order);
 * masks [N][tries][fg_c2f_mask_per_sample_sized(S)] or NULL = fg_dropout_mask(.., N*tries*mask, 0.5,
 * 2*seed+1).  Both streams are indexed by the global row i*tries+t and neither net has a BatchNorm
 * layer, so the result does not depend on `chunk`.  Argument errors return before any launch.      */
int fg_c2f_refine(fg_c2f* n, const float* images, int64_t N, int in_size, int tries, int chunk, int training,
                  const float* noise, const float* masks, uint64_t seed, float* out, int32_t* pick_out, float* pred_out);

/* ---- the denoising autoencoders of train_denoiser.lua (train.lua --denoise) ------------------ */
/* AE = WhiteNoise(0, noise_std) + DECODER, AE2 = a second DECODER fed with AE's output
 * (train_denoiser.lua:83-117), images [B][C][S][S] with S = 16 or 32 and C = the ctx's channels.
 * DECODER = conv(C,8,3) SpatialBN LeakyReLU(0.333) conv(8,8,3) SpatialBN LeakyReLU Dropout(p)
 *           Linear(8(S-4)^2, 2048) BN LeakyReLU Dropout(p) Linear(2048, C S S) Sigmoid (no padding).
 * `net` is 0 for AE1's decoder (AE1_DECODER), 1 for AE2's (AE2_DECODER).  Single GPU only: a data-
 * parallel ctx gets FG_ERR_UNSUPPORTED.  Batches run from 2 (1 in evaluation) up to max_batch.     */
typedef struct fg_dn fg_dn;
typedef struct fg_dn_hyper {
  float lr, beta1, beta2, eps;  /* optim.adam: 1e-3, 0.9, 0.999, 1e-8 (OPTSTATE.adam = {})          */
  float L1, L2;                 /* --coefL1 / --coefL2: 0, 0 (loss, then grad += L1 sign(P) + L2 P)   */
  float clamp;                  /* --AE_clamp: 1 (gradients clamped to +-clamp; 0 = off)             */
  float p_drop;                 /* Dropout(0.2) of both dropout layers                                */
  float noise_std;              /* WhiteNoise(0, 0.1)                                                 */
} fg_dn_hyper;
typedef struct fg_dn_stats {
  float loss_AE1, loss_AE2;     /* BCE of the AE step and of the AE2 step (no penalty terms)          */
  int32_t t;                    /* the shared Adam step counter: 2 per batch                          */
} fg_dn_stats;
void fg_dn_hyper_default(fg_dn_hyper* h);
int fg_dn_create(fg_ctx* ctx, int size, fg_dn** out);     /* size 16 or 32, else FG_ERR_UNSUPPORTED */
int fg_dn_destroy(fg_dn* n);
int64_t fg_dn_param_count(int channels, int size);        /* one decoder; -1 for an unsupported shape */
/* dropout keep flags per sample: 8(S-4)^2 of the conv block ([8][S-4][S-4] order), then 2048       */
int fg_dn_mask_per_sample(int size);
int fg_dn_set_params(fg_dn* n, int net, const float* src); /* getParameters() order of one decoder   */
int fg_dn_get_params(fg_dn* n, int net, float* dst);
int fg_dn_get_grads(fg_dn* n, int net, float* dst);
int fg_dn_zero_grads(fg_dn* n, int net);
/* running statistics of one decoder's three BatchNorm layers: [mean1 8][var1 8][mean2 8][var2 8]
 * [mean3 2048][var3 2048] (4128 floats, the fg_t7_net_bn_state order)                             */
int fg_dn_set_bn_state(fg_dn* n, int net, const float* src);
int fg_dn_get_bn_state(fg_dn* n, int net, float* dst);
/* the ONE Adam state both updates of a batch use (m, v: fg_dn_param_count floats; t)              */
int fg_dn_set_adam_state(fg_dn* n, const float* m, const float* v, int t);
int fg_dn_get_adam_state(fg_dn* n, float* m, float* v, int* t);
/* forward of one decoder (net 0 with its WhiteNoise): x, out [B][C][S][S].  training != 0: batch
 * statistics (running statistics updated), noise [B][C][S][S] (net 0 only) and keep flags masks
 * [B][mps], each drawn from `seed` when NULL; 0: evaluate().  backward: dout = dL/d(out) of the last
 * forward of that decoder; its parameter gradients are ACCUMULATED (fg_dn_zero_grads).  A train step
 * leaves no forward to differentiate: call fg_dn_forward first (else FG_ERR_INVALID).              */
int fg_dn_forward(fg_dn* n, int net, const float* x, int B, int training, const float* noise, const float* masks,
                  uint64_t seed, float* out);
int fg_dn_backward(fg_dn* n, int net, const float* dout);
/* the per-batch body of train_denoiser.lua:247-341: fevalAE + adam, then fevalAE2 (AE forward again:
 * fresh noise and masks, AE's updated parameters, running statistics updated) + adam, on ONE Adam
 * state.  images [B][C][S][S] are inputs and targets; noise [2][B][C][S][S] (AE step, AE in the AE2
 * step) and masks [3][B][mps] (the same two, then AE2) may each be NULL: drawn from `seed`, streams
 * (8 seed + k) for noise k and (8 seed + 2 + k) for masks k.  Replays a captured CUDA graph.       */
int fg_dn_train_step(fg_dn* n, const fg_dn_hyper* h, int B, const float* images, const float* noise, const float* masks,
                     uint64_t seed, fg_dn_stats* stats);
/* train.lua --denoise: AE1_DECODER:evaluate():forward(images) for N images, `chunk` at a time       */
int fg_dn_denoise(fg_dn* n, const float* images, int N, int chunk, float* out);
/* the fg_*debug_tensor contract: what the last forwards drew, "noise0", "noise1" (NCHW), "masks0".."masks2";
 * each decoder's last forward "AE1.*" / "AE2.*": x z1 h1 z2 h2 z3 h3 z4 y (NHWC) and mean1..3 istd1..3; the
 * last backward's gradients dz4 dh3 dz3 dh2 dz2 dh1 dz1 (NHWC)                                      */
int64_t fg_dn_debug_tensor(fg_dn* n, const char* name, float* dst, int64_t max_elems);

/* ---- the autoencoder of train_autoencoder.lua ------------------------------------------------- */
/* MODEL_AE = View(I) Linear(I,512) ReLU Linear(512,d) Tanh Dropout(0.5) Linear(d,256) ReLU
 * Linear(256,I) Sigmoid View(1,S,S) (train_autoencoder.lua:80-92): grayscale images [B][1][S][S],
 * S = 16 or 32, I = S^2, d = --noiseDim (a multiple of 8 in [8, 1024]; a multiple of 64 keeps all four
 * Linear layers on the tensor cores).  Parameters in getParameters() order [L1W L1b .. L4W L4b],
 * weights [out][in].  The object borrows the ctx (destroy it before the ctx), which must have 1
 * channel and be single-GPU (else FG_ERR_UNSUPPORTED).  No BatchNorm: batches run from 1 to max_batch. */
typedef struct fg_ae fg_ae;
typedef struct fg_ae_hyper {
  float lr, beta1, beta2, eps;  /* optim.adam with OPTSTATE.adam = {}: 1e-3, 0.9, 0.999, 1e-8         */
  float L1, L2;                 /* --coefL1 / --coefL2: 0, 0 (grad += L1 sign(P) + L2 P)               */
  float p_drop;                 /* Dropout(0.5)                                                        */
} fg_ae_hyper;
typedef struct fg_ae_stats {
  float loss;                   /* nn.AbsCriterion: mean |output - input| (no penalty terms)           */
  int32_t t;                    /* the Adam step counter                                               */
} fg_ae_stats;
void fg_ae_hyper_default(fg_ae_hyper* h);
int fg_ae_create(fg_ctx* ctx, int size, int noise_dim, fg_ae** out);
int fg_ae_destroy(fg_ae* n);
int64_t fg_ae_param_count(int size, int noise_dim);       /* -1 for an unsupported shape              */
int fg_ae_set_params(fg_ae* n, const float* src);
int fg_ae_get_params(fg_ae* n, float* dst);
int fg_ae_get_grads(fg_ae* n, float* dst);
int fg_ae_zero_grads(fg_ae* n);
int fg_ae_set_adam_state(fg_ae* n, const float* m, const float* v, int t);
int fg_ae_get_adam_state(fg_ae* n, float* m, float* v, int* t);
/* forward: x [B][1][S][S] -> out (same shape) and the encoder's output code_out [B][d] (tanh, before
 * Dropout); either may be NULL.  training != 0: Dropout with the keep flags masks [B][d], drawn from
 * `seed` when NULL; 0: evaluate().  backward: dout = dL/d(out) of the last forward; the parameter
 * gradients are ACCUMULATED (fg_ae_zero_grads).  A train step or fg_ae_reconstruct leaves no forward
 * to differentiate: FG_ERR_STATE.                                                                   */
int fg_ae_forward(fg_ae* n, const float* x, int B, int training, const float* masks, uint64_t seed, float* code_out,
                  float* out);
int fg_ae_backward(fg_ae* n, const float* dout);
/* the per-batch body of train_autoencoder.lua:178-209: zero gradients, forward, nn.AbsCriterion with
 * the images as their own targets, backward, penalty gradients, optim.adam; no gradient clamp.  The
 * criterion's gradient is +1/n where output >= target (a tie counts as positive), -1/n elsewhere.
 * masks [B][d] keep flags or NULL (drawn from `seed`).  Replays a captured CUDA graph; with stats ==
 * NULL the call does not wait for the GPU.                                                          */
int fg_ae_train_step(fg_ae* n, const fg_ae_hyper* h, int B, const float* images, const float* masks, uint64_t seed,
                     fg_ae_stats* stats);
/* the same on images idx[0..B) (int32, host or device) of a dataset on the same ctx, gathered at S x S
 * on the device (fg_dataset_gather_sized); keep flags drawn from `seed`.  Nothing synchronises unless
 * stats != NULL: an epoch over a host-owned permutation can be enqueued without waiting.            */
int fg_ae_train_step_dataset(fg_ae* n, fg_dataset* d, const fg_ae_hyper* h, const int32_t* idx, int B, uint64_t seed,
                             fg_ae_stats* stats);
/* MODEL_AE:forward of N images, `chunk` (<= max_batch) at a time.  training != 0 keeps Dropout live, as
 * getSamples (train_autoencoder.lua:137-145) does; chunk k then draws its keep flags from seed + k.    */
int fg_ae_reconstruct(fg_ae* n, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* out);
/* the fg_*debug_tensor contract over the last forward (x z1 h1 z2 code h2 z3 h3 z4 y, and "masks" after
 * a training-mode one) and the last backward (dz4 dz3 dz2 dz1), each [B][features]; "loss": the last
 * step's criterion value, one float (into device memory the copy is asynchronous)                  */
int64_t fg_ae_debug_tensor(fg_ae* n, const char* name, float* dst, int64_t max_elems);
/* the same layers one at a time, flat tensors of n floats (host or device pointers): nn.ReLU (backward
 * from the input x), nn.Tanh (backward from the output y), nn.AbsCriterion size-averaged              */
int fg_relu_forward(fg_ctx* ctx, const float* x, float* y, int64_t n);
int fg_relu_backward(fg_ctx* ctx, const float* x, const float* dy, float* dx, int64_t n);
int fg_tanh_forward(fg_ctx* ctx, const float* x, float* y, int64_t n);
int fg_tanh_backward(fg_ctx* ctx, const float* y, const float* dy, float* dx, int64_t n);
int fg_abs_forward(fg_ctx* ctx, const float* x, const float* t, int64_t n, float* loss_out);
int fg_abs_backward(fg_ctx* ctx, const float* x, const float* t, int64_t n, float* dx);

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
/* the same for the coarse-to-fine and --scale 16 nets: dst == NULL returns the element count, -2 when
 * dst is too small, -1 (fg_last_error) for an unknown name or one not produced yet.  "Dstep.*" are the
 * D step's tensors of the last train step with option "debug_keep".
 *   c2f: G.x G.z1..G.z5  D.x D.z1..D.z4 D.p2 D.p4 D.zl1 D.logit D.out  Dstep.z1..z4 .zl1 .logit .out
 *   s16: G.z0..G.z3 G.bn_mean1/2 G.bn_istd1/2  D.z1..D.z4 (after the stride-2 sampling) D.p1 D.zf
 *        D.ze1 D.ze2 D.logit D.out  Dstep.z1..z4 .zf .ze1 .ze2 .logit .out                            */
int64_t fg_c2f_debug_tensor(fg_c2f* n, const char* name, float* dst, int64_t max_elems);
int64_t fg_s16_debug_tensor(fg_s16* n, const char* name, float* dst, int64_t max_elems);
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
