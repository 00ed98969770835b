-- fg_ffi.lua -- LuaJIT FFI binding of libfg_b200.so (include/fg_b200.h), 1:1 with face_generator_b200/lib.py.
-- NOTE: LuaJIT/Torch7 are not installed in the build image, so this file is delivered untested-by-execution;
-- it is deliberately thin (cdef + error check) and the identical call sequence is exercised through ctypes by
-- tests/ (face_generator_b200/lib.py is the executable mirror of this file).
local ffi = require 'ffi'

ffi.cdef[[
typedef struct fg_ctx fg_ctx;
typedef struct fg_hyper {
  float lr_D, lr_G, beta1, beta2, eps, D_L1, D_L2, G_L1, G_L2, D_clamp, G_clamp, D_maxAcc;
  int32_t accs_interval;
  float p_spatial, p_drop;
} fg_hyper;
typedef struct fg_step_stats {
  float loss_D, loss_G; int32_t conf[4]; int32_t trained_D; int32_t t_D, t_G; float acc_D;
} fg_step_stats;
const char* fg_version(void);
const char* fg_last_error(void);
void fg_hyper_default(fg_hyper* h);
int fg_create(fg_ctx** out, int device, int max_batch, int channels);
int fg_destroy(fg_ctx* ctx);
int fg_set_stream(fg_ctx* ctx, void* cuda_stream);
int fg_sync(fg_ctx* ctx);
int fg_set_option(fg_ctx* ctx, const char* key, int64_t value);
int64_t fg_get_option(fg_ctx* ctx, const char* key);
int fg_set_option_f(fg_ctx* ctx, const char* key, double value);
int64_t fg_param_count(int net, int channels);
int fg_set_params(fg_ctx* ctx, int net, const float* src);
int fg_get_params(fg_ctx* ctx, int net, float* dst);
int fg_get_grads(fg_ctx* ctx, int net, float* dst);
int fg_zero_grads(fg_ctx* ctx, int net);
int fg_bind_params(fg_ctx* ctx, int net, float* params_dev, float* grads_dev);
float* fg_params_ptr(fg_ctx* ctx, int net);
float* fg_grads_ptr(fg_ctx* ctx, int net);
int fg_set_adam_state(fg_ctx* ctx, int net, const float* m, const float* v, int t);
int fg_get_adam_state(fg_ctx* ctx, int net, float* m, float* v, int* t);
int fg_set_bn_state(fg_ctx* ctx, const float* src768);
int fg_get_bn_state(fg_ctx* ctx, float* dst768);
int fg_G_forward(fg_ctx* ctx, const float* noise, int B, int training, float* images_out);
int fg_G_backward(fg_ctx* ctx, const float* d_images, float* d_noise);
int fg_D_forward(fg_ctx* ctx, const float* images, int B, int training, const float* masks, uint64_t seed, float* out);
int fg_D_backward(fg_ctx* ctx, const float* d_out, int want_wgrad, float* d_images);
int fg_bce_forward(fg_ctx* ctx, const float* x, const float* t, int n, float* loss_out);
int fg_bce_backward(fg_ctx* ctx, const float* x, const float* t, int n, float* dx);
int fg_optim_step(fg_ctx* ctx, int net, const fg_hyper* h, float grad_scale);
int fg_adam_step(fg_ctx* ctx, float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1,
                 float beta2, float eps, int t, float l1_grad, float l2, float clampv, float grad_scale);
int fg_conv2d_forward(fg_ctx* ctx, const float* x, const float* w, const float* b, float* y, int N, int Cin, int H, int W, int Cout, int k);
int fg_conv2d_backward_data(fg_ctx* ctx, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W, int Cout, int k);
int fg_conv2d_backward_filter(fg_ctx* ctx, const float* x, const float* dy, float* dw, float* db, int N, int Cin, int H, int W, int Cout, int k);
int fg_scu_forward(fg_ctx* ctx, const float* x, const float* w, const float* b, float* y, int N, int Cin, int H, int W, int nOutputPlane, int k, int factor);
int fg_scu_backward_data(fg_ctx* ctx, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W, int nOutputPlane, int k, int factor);
int fg_scu_backward_filter(fg_ctx* ctx, const float* x, const float* dy, float* dw, float* db, int N, int Cin, int H, int W, int nOutputPlane, int k, int factor);
int fg_linear_forward(fg_ctx* ctx, const float* x, const float* w, const float* b, float* y, int N, int inp, int out);
int fg_linear_backward(fg_ctx* ctx, const float* x, const float* w, const float* dy, float* dx, float* dw, float* db, int N, int inp, int out);
int fg_bn_forward_train(fg_ctx* ctx, const float* x, const float* gamma, const float* beta, float* y, float* save_mean,
                        float* save_istd, float* run_mean, float* run_var, int N, int C, int HW);
int fg_bn_backward(fg_ctx* ctx, const float* x, const float* gamma, const float* save_mean, const float* save_istd,
                   const float* dy, float* dx, float* dgamma, float* dbeta, int N, int C, int HW);
int fg_prelu_forward(fg_ctx* ctx, const float* x, const float* slope, float* y, int64_t n);
int fg_prelu_backward(fg_ctx* ctx, const float* x, const float* slope, const float* dy, float* dx, float* dslope, int64_t n);
int fg_upsample2_forward(fg_ctx* ctx, const float* x, float* y, int N, int C, int H, int W);
int fg_upsample2_backward(fg_ctx* ctx, const float* dy, float* dx, int N, int C, int H, int W);
int fg_avgpool2_forward(fg_ctx* ctx, const float* x, float* y, int N, int C, int H, int W);
int fg_avgpool2_backward(fg_ctx* ctx, const float* dy, float* dx, int N, int C, int H, int W);
int fg_maxpool2_forward(fg_ctx* ctx, const float* x, float* y, int N, int C, int H, int W);
int fg_maxpool2_backward(fg_ctx* ctx, const float* x, const float* dy, float* dx, int N, int C, int H, int W);
int fg_dropout_forward(fg_ctx* ctx, const float* x, const float* mask, float p, int spatial, float* y, int N, int C, int HW);
int fg_dropout_backward(fg_ctx* ctx, const float* dy, const float* mask, float p, int spatial, float* dx, int N, int C, int HW);
int fg_dropout_mask(fg_ctx* ctx, float* mask_dev, int64_t n, float p, uint64_t seed);
int fg_sigmoid_forward(fg_ctx* ctx, const float* x, float* y, int64_t n);
int fg_sigmoid_backward(fg_ctx* ctx, const float* y, const float* dy, float* dx, int64_t n);
typedef struct fg_c2f fg_c2f;
int fg_c2f_create(fg_ctx* ctx, fg_c2f** out);
int fg_c2f_destroy(fg_c2f* n);
int64_t fg_c2f_param_count(int net, int channels);
int fg_c2f_mask_per_sample(void);
int fg_c2f_set_params(fg_c2f* n, int net, const float* src);
int fg_c2f_get_params(fg_c2f* n, int net, float* dst);
int fg_c2f_get_grads(fg_c2f* n, int net, float* dst);
int fg_c2f_zero_grads(fg_c2f* n, int net);
float* fg_c2f_params_ptr(fg_c2f* n, int net);
float* fg_c2f_grads_ptr(fg_c2f* n, int net);
int fg_c2f_set_adam_state(fg_c2f* n, int net, const float* m, const float* v, int t);
int fg_c2f_get_adam_state(fg_c2f* n, int net, float* m, float* v, int* t);
int fg_c2f_G_forward(fg_c2f* n, const float* noise, const float* cond, int B, float* diff_out);
int fg_c2f_G_backward(fg_c2f* n, const float* d_diff);
int fg_c2f_D_forward(fg_c2f* n, const float* diff, const float* cond, int B, int training, const float* masks, uint64_t seed, float* out);
int fg_c2f_D_backward(fg_c2f* n, const float* d_out, int want_wgrad, float* d_diff);
int fg_c2f_train_step(fg_c2f* n, const fg_hyper* h, int B, const float* real_diff, const float* cond_D, const float* noise_D,
                      const float* cond_G, const float* noise_G, const float* masks_D, const float* masks_G, uint64_t seed,
                      fg_step_stats* stats);
typedef struct fg_dataset fg_dataset;
int fg_dataset_create(fg_ctx* ctx, int64_t N, int Cs, int Hs, int Ws, fg_dataset** out);
int fg_dataset_destroy(fg_dataset* d);
int64_t fg_dataset_size(fg_dataset* d);
int fg_dataset_upload(fg_dataset* d, int64_t first, int64_t count, const uint8_t* images);
int fg_dataset_gather(fg_dataset* d, const int32_t* idx, int B, float* out);
int fg_dataset_draw(fg_dataset* d, uint64_t seed, int B, int32_t* idx_out);
int fg_noise_uniform(fg_ctx* ctx, uint64_t seed, int64_t n, float* out);
int fg_train_step_dataset(fg_ctx* ctx, fg_dataset* d, const fg_hyper* h, int B, uint64_t seed, fg_step_stats* stats);
int fg_D_score(fg_ctx* ctx, const float* images, int64_t N, int chunk, int training, uint64_t seed, float* preds_out);
int fg_nearest(fg_ctx* ctx, const float* queries, int Q, const float* cands, int64_t N, int D, int32_t* idx_out, float* dist_out);
int fg_dataset_nearest(fg_dataset* d, const float* queries, int Q, int32_t* idx_out, float* dist_out);
int fg_c2f_parzen_dist(fg_c2f* n, const float* noise, const float* coarse, const float* fine, int K, float* dist_out);
typedef struct fg_t7 fg_t7;
int fg_t7_open(const char* path, fg_t7** out);
int fg_t7_close(fg_t7* f);
int fg_t7_kind(fg_t7* f, const char* path);
int fg_t7_number(fg_t7* f, const char* path, double* out);
int64_t fg_t7_string(fg_t7* f, const char* path, char* dst, int64_t cap);
int64_t fg_t7_tensor(fg_t7* f, const char* path, float* dst, int64_t cap, int64_t* dims8);
int64_t fg_t7_net_params(fg_t7* f, const char* path, float* dst, int64_t cap);
int64_t fg_t7_net_bn_state(fg_t7* f, const char* path, float* dst, int64_t cap);
int64_t fg_t7_net_describe(fg_t7* f, const char* path, char* dst, int64_t cap);
typedef struct fg_t7_writer fg_t7_writer;
int fg_t7_writer_open(const char* path, fg_t7_writer** out);
int fg_t7_writer_add_tensor(fg_t7_writer* w, const char* key, const float* data, const int64_t* dims, int ndim);
int fg_t7_writer_add_number(fg_t7_writer* w, const char* key, double v);
int fg_t7_writer_add_string(fg_t7_writer* w, const char* key, const char* s);
int fg_t7_writer_close(fg_t7_writer* w);
int fg_train_step(fg_ctx* ctx, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                  const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats);
int fg_sample(fg_ctx* ctx, const float* noise, int N, int chunk, float* images_out);
int fg_dp_unique_id(void* out128);
int fg_dp_init(fg_ctx* ctx, const void* id128, int nranks, int rank);
int fg_dp_broadcast_params(fg_ctx* ctx);
typedef struct fg_s16 fg_s16;
int fg_s16_create(fg_ctx* ctx, fg_s16** out);
int fg_s16_destroy(fg_s16* n);
int64_t fg_s16_param_count(int net, int channels);
int fg_s16_mask_per_sample(void);
int fg_s16_set_params(fg_s16* n, int net, const float* src);
int fg_s16_get_params(fg_s16* n, int net, float* dst);
int fg_s16_get_grads(fg_s16* n, int net, float* dst);
int fg_s16_zero_grads(fg_s16* n, int net);
float* fg_s16_params_ptr(fg_s16* n, int net);
float* fg_s16_grads_ptr(fg_s16* n, int net);
int fg_s16_set_adam_state(fg_s16* n, int net, const float* m, const float* v, int t);
int fg_s16_get_adam_state(fg_s16* n, int net, float* m, float* v, int* t);
int fg_s16_set_bn_state(fg_s16* n, const float* src768);
int fg_s16_get_bn_state(fg_s16* n, float* dst768);
int fg_s16_G_forward(fg_s16* n, const float* noise, int B, int training, float* img_out);
int fg_s16_G_backward(fg_s16* n, const float* d_img, float* d_noise);
int fg_s16_D_forward(fg_s16* n, const float* img, int B, int training, const float* masks, uint64_t seed, float* out);
int fg_s16_D_backward(fg_s16* n, const float* d_out, int want_wgrad, float* d_img);
int fg_s16_train_step(fg_s16* n, const fg_hyper* h, int B, const float* real, const float* noise_D, const float* noise_G,
                      const float* masks_D, const float* masks_G, uint64_t seed, fg_step_stats* stats);
int fg_c2f_dp_broadcast_params(fg_c2f* n);
int fg_s16_dp_broadcast_params(fg_s16* n);
int fg_dp_world(fg_ctx* ctx);
void* fg_dev_alloc(size_t bytes);
int fg_dev_free(void* p);
void* fg_host_alloc_pinned(size_t bytes);
int fg_host_free_pinned(void* p);
int fg_memcpy(fg_ctx* ctx, void* dst, const void* src, size_t bytes);
int64_t fg_kernel_launches(fg_ctx* ctx);
int64_t fg_debug_tensor(fg_ctx* ctx, const char* name, float* dst, int64_t max_elems);
int fg_bench_tf32_peak(fg_ctx* ctx, int iters, double* tflops);
int fg_event_record(fg_ctx* ctx, int slot);
int fg_event_elapsed_ms(fg_ctx* ctx, int slot_a, int slot_b, double* ms);
int fg_timing_enable(fg_ctx* ctx, int on);
int fg_timing_get(fg_ctx* ctx, const char* name, double* ms_total, int64_t* launches);
]]

local M = {}
M.NET_G, M.NET_D = 0, 1
M.C = ffi.load(os.getenv('FG_B200_LIB') or 'fg_b200')  -- libfg_b200.so on LD_LIBRARY_PATH

function M.check(rc, what)
  if rc ~= 0 then
    error(string.format('%s failed (%d): %s', what, tonumber(rc), ffi.string(M.C.fg_last_error())))
  end
end

-- float* of a contiguous torch.FloatTensor / torch.CudaTensor (the library classifies host vs device itself)
function M.ptr(t)
  if t == nil then return nil end
  assert(t:isContiguous(), 'b200: tensors must be contiguous')
  return ffi.cast('float*', torch.pointer(t:storage():data()) ) + (t:storageOffset() - 1)
end

return M
