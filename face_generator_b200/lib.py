"""ctypes binding of libfg_b200.so -- a 1:1 mirror of face_generator_b200/lua/fg_ffi.lua.

Fails loudly when the shared library is missing or a call returns an error; never falls back to
a CPU implementation (the CPU oracle under oracle/ is test infrastructure and is not imported here).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfg_b200.so")
MASK_PER_SAMPLE = 1984
NOISE_DIM = 100
NET_G, NET_D = 0, 1
CONV_SIMT, CONV_TC_DENSE, CONV_TC_COLLAPSED = 0, 1, 2


class FGError(RuntimeError):
    pass


class Hyper(C.Structure):
    _fields_ = [("lr_D", C.c_float), ("lr_G", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float), ("D_L1", C.c_float), ("D_L2", C.c_float), ("G_L1", C.c_float),
                ("G_L2", C.c_float), ("D_clamp", C.c_float), ("G_clamp", C.c_float), ("D_maxAcc", C.c_float),
                ("accs_interval", C.c_int32), ("p_spatial", C.c_float), ("p_drop", C.c_float)]


class StepStats(C.Structure):
    _fields_ = [("loss_D", C.c_float), ("loss_G", C.c_float), ("conf", C.c_int32 * 4), ("trained_D", C.c_int32),
                ("t_D", C.c_int32), ("t_G", C.c_int32), ("acc_D", C.c_float)]


class DnHyper(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("L1", C.c_float),
                ("L2", C.c_float), ("clamp", C.c_float), ("p_drop", C.c_float), ("noise_std", C.c_float)]


class DnStats(C.Structure):
    _fields_ = [("loss_AE1", C.c_float), ("loss_AE2", C.c_float), ("t", C.c_int32)]


class AeHyper(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("L1", C.c_float),
                ("L2", C.c_float), ("p_drop", C.c_float)]


class AeStats(C.Structure):
    _fields_ = [("loss", C.c_float), ("t", C.c_int32)]


# every symbol include/fg_b200.h declares: name -> (restype, argtypes)
_P, _F, _I, _L, _U64, _SZ = C.c_void_p, C.c_float, C.c_int, C.c_int64, C.c_uint64, C.c_size_t
SYMBOLS = {
    "fg_version": (C.c_char_p, []),
    "fg_last_error": (C.c_char_p, []),
    "fg_hyper_default": (None, [C.POINTER(Hyper)]),
    "fg_create": (_I, [C.POINTER(_P), _I, _I, _I]),
    "fg_destroy": (_I, [_P]),
    "fg_set_stream": (_I, [_P, _P]),
    "fg_sync": (_I, [_P]),
    "fg_set_option": (_I, [_P, C.c_char_p, _L]),
    "fg_get_option": (_L, [_P, C.c_char_p]),
    "fg_set_option_f": (_I, [_P, C.c_char_p, C.c_double]),
    "fg_param_count": (_L, [_I, _I]),
    "fg_create_disc": (_I, [C.POINTER(_P), _I, _I, _I, _I]),
    "fg_get_disc": (_I, [_P]),
    "fg_disc_param_count": (_L, [_I, _I]),
    "fg_disc_mask_per_sample": (_I, [_I]),
    "fg_disc_side": (_I, [_I]),
    "fg_set_params": (_I, [_P, _I, _P]),
    "fg_get_params": (_I, [_P, _I, _P]),
    "fg_get_grads": (_I, [_P, _I, _P]),
    "fg_bind_params": (_I, [_P, _I, _P, _P]),
    "fg_zero_grads": (_I, [_P, _I]),
    "fg_params_ptr": (_P, [_P, _I]),
    "fg_grads_ptr": (_P, [_P, _I]),
    "fg_set_adam_state": (_I, [_P, _I, _P, _P, _I]),
    "fg_get_adam_state": (_I, [_P, _I, _P, _P, C.POINTER(_I)]),
    "fg_set_bn_state": (_I, [_P, _P]),
    "fg_get_bn_state": (_I, [_P, _P]),
    "fg_G_forward": (_I, [_P, _P, _I, _I, _P]),
    "fg_G_backward": (_I, [_P, _P, _P]),
    "fg_D_forward": (_I, [_P, _P, _I, _I, _P, _U64, _P]),
    "fg_D_backward": (_I, [_P, _P, _I, _P]),
    "fg_bce_forward": (_I, [_P, _P, _P, _I, _P]),
    "fg_bce_backward": (_I, [_P, _P, _P, _I, _P]),
    "fg_optim_step": (_I, [_P, _I, C.POINTER(Hyper), _F]),
    "fg_adam_step": (_I, [_P, _P, _P, _P, _P, _L, _F, _F, _F, _F, _I, _F, _F, _F, _F]),
    "fg_conv2d_forward": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I]),
    "fg_conv2d_backward_data": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I]),
    "fg_conv2d_backward_filter": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I]),
    "fg_scu_forward": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I]),
    "fg_scu_backward_data": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I]),
    "fg_scu_backward_filter": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I]),
    "fg_linear_forward": (_I, [_P, _P, _P, _P, _P, _I, _I, _I]),
    "fg_linear_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I]),
    "fg_bn_forward_train": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I]),
    "fg_bn_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I]),
    "fg_prelu_forward": (_I, [_P, _P, _P, _P, _L]),
    "fg_prelu_backward": (_I, [_P, _P, _P, _P, _P, _P, _L]),
    "fg_upsample2_forward": (_I, [_P, _P, _P, _I, _I, _I, _I]),
    "fg_upsample2_backward": (_I, [_P, _P, _P, _I, _I, _I, _I]),
    "fg_avgpool2_forward": (_I, [_P, _P, _P, _I, _I, _I, _I]),
    "fg_avgpool2_backward": (_I, [_P, _P, _P, _I, _I, _I, _I]),
    "fg_maxpool2_forward": (_I, [_P, _P, _P, _I, _I, _I, _I]),
    "fg_maxpool2_backward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I]),
    "fg_dropout_forward": (_I, [_P, _P, _P, _F, _I, _P, _I, _I, _I]),
    "fg_dropout_backward": (_I, [_P, _P, _P, _F, _I, _P, _I, _I, _I]),
    "fg_dropout_mask": (_I, [_P, _P, _L, _F, _U64]),
    "fg_sigmoid_forward": (_I, [_P, _P, _P, _L]),
    "fg_sigmoid_backward": (_I, [_P, _P, _P, _P, _L]),
    "fg_c2f_create": (_I, [_P, C.POINTER(_P)]),
    "fg_c2f_create_sized": (_I, [_P, _I, C.POINTER(_P)]),
    "fg_c2f_fine_size": (_I, [_P]),
    "fg_c2f_param_count_sized": (_L, [_I, _I, _I]),
    "fg_c2f_mask_per_sample_sized": (_I, [_I]),
    "fg_c2f_create_nets": (_I, [_P, _I, _I, _I, C.POINTER(_P)]),
    "fg_c2f_get_gen": (_I, [_P]),
    "fg_c2f_get_disc": (_I, [_P]),
    "fg_c2f_gen_param_count": (_L, [_I, _I]),
    "fg_c2f_disc_param_count": (_L, [_I, _I, _I]),
    "fg_c2f_disc_mask_per_sample": (_I, [_I, _I]),
    "fg_c2f_destroy": (_I, [_P]),
    "fg_c2f_param_count": (_L, [_I, _I]),
    "fg_c2f_mask_per_sample": (_I, []),
    "fg_c2f_set_params": (_I, [_P, _I, _P]),
    "fg_c2f_get_params": (_I, [_P, _I, _P]),
    "fg_c2f_get_grads": (_I, [_P, _I, _P]),
    "fg_c2f_zero_grads": (_I, [_P, _I]),
    "fg_c2f_params_ptr": (_P, [_P, _I]),
    "fg_c2f_grads_ptr": (_P, [_P, _I]),
    "fg_c2f_set_adam_state": (_I, [_P, _I, _P, _P, _I]),
    "fg_c2f_get_adam_state": (_I, [_P, _I, _P, _P, C.POINTER(_I)]),
    "fg_c2f_G_forward": (_I, [_P, _P, _P, _I, _P]),
    "fg_c2f_G_backward": (_I, [_P, _P]),
    "fg_c2f_D_forward": (_I, [_P, _P, _P, _I, _I, _P, _U64, _P]),
    "fg_c2f_D_backward": (_I, [_P, _P, _I, _P]),
    "fg_c2f_train_step": (_I, [_P, C.POINTER(Hyper), _I, _P, _P, _P, _P, _P, _P, _P, _U64, C.POINTER(StepStats)]),
    "fg_dataset_create": (_I, [_P, _L, _I, _I, _I, C.POINTER(_P)]),
    "fg_dataset_destroy": (_I, [_P]),
    "fg_dataset_size": (_L, [_P]),
    "fg_dataset_upload": (_I, [_P, _L, _L, _P]),
    "fg_dataset_download": (_I, [_P, _L, _L, _P]),
    "fg_jpeg_info": (_I, [_P, _L, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "fg_dataset_upload_jpeg": (_I, [_P, _L, _L, _P, _P, C.POINTER(_L)]),
    "fg_dataset_encode_jpeg": (_I, [_P, _L, _L, _I, _P, _L, _P]),
    "fg_dataset_jpeg_roundtrip": (_I, [_P, _L, _L, _I]),
    "fg_jpeg_encode": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _L, _P]),
    "fg_image_grid": (_I, [_P, _P, _L, _I, _I, _I, _P, _I, _I, _I, _P, _P, _P]),
    "fg_lfw_aug_params": (_I, [_U64, _L, _L, _I, _I, _I, _P]),
    "fg_dataset_augment": (_I, [_P, _P, _L, _P, _L]),
    "fg_dataset_gather": (_I, [_P, _P, _I, _P]),
    "fg_dataset_draw": (_I, [_P, _U64, _I, _P]),
    "fg_noise_uniform": (_I, [_P, _U64, _L, _P]),
    "fg_train_step_dataset": (_I, [_P, _P, C.POINTER(Hyper), _I, _U64, C.POINTER(StepStats)]),
    "fg_dataset_gather_sized": (_I, [_P, _P, _I, _I, _P]),
    "fg_dataset_gather_c2f": (_I, [_P, _P, _I, _I, _P, _P, _P]),
    "fg_dataset_gather_c2f_sized": (_I, [_P, _P, _I, _I, _I, _P, _P, _P]),
    "fg_s16_train_step_dataset": (_I, [_P, _P, C.POINTER(Hyper), _I, _U64, C.POINTER(StepStats)]),
    "fg_c2f_train_step_dataset": (_I, [_P, _P, C.POINTER(Hyper), _I, _I, _U64, C.POINTER(StepStats)]),
    "fg_D_score": (_I, [_P, _P, _L, _I, _I, _U64, _P]),
    "fg_nearest": (_I, [_P, _P, _I, _P, _L, _I, _P, _P]),
    "fg_dataset_nearest": (_I, [_P, _P, _I, _P, _P]),
    "fg_dataset_nearest_sized": (_I, [_P, _I, _P, _I, _P, _P]),
    "fg_s16_D_score": (_I, [_P, _P, _L, _I, _I, _U64, _P]),
    "fg_c2f_parzen_dist": (_I, [_P, _P, _P, _P, _I, _P]),
    "fg_image_scale": (_I, [_P, _P, _L, _I, _I, _I, _I, _I, _P]),
    "fg_c2f_refine": (_I, [_P, _P, _L, _I, _I, _I, _I, _P, _P, _U64, _P, _P, _P]),
    "fg_t7_open": (_I, [C.c_char_p, C.POINTER(_P)]),
    "fg_t7_close": (_I, [_P]),
    "fg_t7_kind": (_I, [_P, C.c_char_p]),
    "fg_t7_number": (_I, [_P, C.c_char_p, C.POINTER(C.c_double)]),
    "fg_t7_string": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_t7_tensor": (_L, [_P, C.c_char_p, _P, _L, C.POINTER(_L)]),
    "fg_t7_net_params": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_t7_net_bn_state": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_t7_net_describe": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_t7_writer_open": (_I, [C.c_char_p, C.POINTER(_P)]),
    "fg_t7_writer_add_tensor": (_I, [_P, C.c_char_p, _P, C.POINTER(_L), _I]),
    "fg_t7_writer_add_number": (_I, [_P, C.c_char_p, C.c_double]),
    "fg_t7_writer_add_string": (_I, [_P, C.c_char_p, C.c_char_p]),
    "fg_t7_writer_close": (_I, [_P]),
    "fg_train_step": (_I, [_P, C.POINTER(Hyper), _I, _P, _P, _P, _P, _P, _U64, C.POINTER(StepStats)]),
    "fg_sample": (_I, [_P, _P, _I, _I, _P]),
    "fg_dp_unique_id": (_I, [_P]),
    "fg_dp_init": (_I, [_P, _P, _I, _I]),
    "fg_dp_broadcast_params": (_I, [_P]),
    "fg_c2f_dp_broadcast_params": (_I, [_P]),
    "fg_s16_dp_broadcast_params": (_I, [_P]),
    "fg_s16_create": (_I, [_P, C.POINTER(_P)]),
    "fg_s16_destroy": (_I, [_P]),
    "fg_s16_param_count": (_L, [_I, _I]),
    "fg_s16_mask_per_sample": (_I, []),
    "fg_s16_create_disc": (_I, [_P, _I, C.POINTER(_P)]),
    "fg_s16_get_disc": (_I, [_P]),
    "fg_s16_set_params": (_I, [_P, _I, _P]),
    "fg_s16_get_params": (_I, [_P, _I, _P]),
    "fg_s16_get_grads": (_I, [_P, _I, _P]),
    "fg_s16_zero_grads": (_I, [_P, _I]),
    "fg_s16_params_ptr": (_P, [_P, _I]),
    "fg_s16_grads_ptr": (_P, [_P, _I]),
    "fg_s16_set_adam_state": (_I, [_P, _I, _P, _P, _I]),
    "fg_s16_get_adam_state": (_I, [_P, _I, _P, _P, C.POINTER(_I)]),
    "fg_s16_set_bn_state": (_I, [_P, _P]),
    "fg_s16_get_bn_state": (_I, [_P, _P]),
    "fg_s16_G_forward": (_I, [_P, _P, _I, _I, _P]),
    "fg_s16_G_backward": (_I, [_P, _P, _P]),
    "fg_s16_D_forward": (_I, [_P, _P, _I, _I, _P, _U64, _P]),
    "fg_s16_D_backward": (_I, [_P, _P, _I, _P]),
    "fg_s16_train_step": (_I, [_P, C.POINTER(Hyper), _I, _P, _P, _P, _P, _P, _U64, C.POINTER(StepStats)]),
    "fg_dp_world": (_I, [_P]),
    "fg_dev_alloc": (_P, [_SZ]),
    "fg_dev_free": (_I, [_P]),
    "fg_host_alloc_pinned": (_P, [_SZ]),
    "fg_host_free_pinned": (_I, [_P]),
    "fg_memcpy": (_I, [_P, _P, _P, _SZ]),
    "fg_kernel_launches": (_L, [_P]),
    "fg_debug_tensor": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_c2f_debug_tensor": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_s16_debug_tensor": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_bench_tf32_peak": (_I, [_P, _I, C.POINTER(C.c_double)]),
    "fg_event_record": (_I, [_P, _I]),
    "fg_event_elapsed_ms": (_I, [_P, _I, _I, C.POINTER(C.c_double)]),
    "fg_timing_enable": (_I, [_P, _I]),
    "fg_timing_get": (_I, [_P, C.c_char_p, C.POINTER(C.c_double), C.POINTER(_L)]),
    "fg_train_step_iters": (_I, [_P, C.POINTER(Hyper), _I, _I, _I, _P, _P, _P, _P, _P, _U64, C.POINTER(StepStats)]),
    "fg_s16_train_step_iters": (_I, [_P, C.POINTER(Hyper), _I, _I, _I, _P, _P, _P, _P, _P, _U64, C.POINTER(StepStats)]),
    "fg_c2f_train_step_iters": (_I, [_P, C.POINTER(Hyper), _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _U64,
                                     C.POINTER(StepStats)]),
    "fg_train_step_dataset_iters": (_I, [_P, _P, C.POINTER(Hyper), _I, _I, _I, _U64, C.POINTER(StepStats)]),
    "fg_s16_train_step_dataset_iters": (_I, [_P, _P, C.POINTER(Hyper), _I, _I, _I, _U64, C.POINTER(StepStats)]),
    "fg_c2f_train_step_dataset_iters": (_I, [_P, _P, C.POINTER(Hyper), _I, _I, _I, _I, _U64, C.POINTER(StepStats)]),
    "fg_dn_hyper_default": (None, [C.POINTER(DnHyper)]),
    "fg_dn_create": (_I, [_P, _I, C.POINTER(_P)]),
    "fg_dn_destroy": (_I, [_P]),
    "fg_dn_param_count": (_L, [_I, _I]),
    "fg_dn_mask_per_sample": (_I, [_I]),
    "fg_dn_set_params": (_I, [_P, _I, _P]),
    "fg_dn_get_params": (_I, [_P, _I, _P]),
    "fg_dn_get_grads": (_I, [_P, _I, _P]),
    "fg_dn_zero_grads": (_I, [_P, _I]),
    "fg_dn_set_bn_state": (_I, [_P, _I, _P]),
    "fg_dn_get_bn_state": (_I, [_P, _I, _P]),
    "fg_dn_set_adam_state": (_I, [_P, _P, _P, _I]),
    "fg_dn_get_adam_state": (_I, [_P, _P, _P, C.POINTER(_I)]),
    "fg_dn_forward": (_I, [_P, _I, _P, _I, _I, _P, _P, _U64, _P]),
    "fg_dn_backward": (_I, [_P, _I, _P]),
    "fg_dn_train_step": (_I, [_P, C.POINTER(DnHyper), _I, _P, _P, _P, _U64, C.POINTER(DnStats)]),
    "fg_dn_denoise": (_I, [_P, _P, _I, _I, _P]),
    "fg_dn_debug_tensor": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_ae_hyper_default": (None, [C.POINTER(AeHyper)]),
    "fg_ae_create": (_I, [_P, _I, _I, C.POINTER(_P)]),
    "fg_ae_destroy": (_I, [_P]),
    "fg_ae_param_count": (_L, [_I, _I]),
    "fg_ae_set_params": (_I, [_P, _P]),
    "fg_ae_get_params": (_I, [_P, _P]),
    "fg_ae_get_grads": (_I, [_P, _P]),
    "fg_ae_zero_grads": (_I, [_P]),
    "fg_ae_set_adam_state": (_I, [_P, _P, _P, _I]),
    "fg_ae_get_adam_state": (_I, [_P, _P, _P, C.POINTER(_I)]),
    "fg_ae_forward": (_I, [_P, _P, _I, _I, _P, _U64, _P, _P]),
    "fg_ae_backward": (_I, [_P, _P]),
    "fg_ae_train_step": (_I, [_P, C.POINTER(AeHyper), _I, _P, _P, _U64, C.POINTER(AeStats)]),
    "fg_ae_train_step_dataset": (_I, [_P, _P, C.POINTER(AeHyper), _P, _I, _U64, C.POINTER(AeStats)]),
    "fg_ae_reconstruct": (_I, [_P, _P, _L, _I, _I, _U64, _P]),
    "fg_ae_debug_tensor": (_L, [_P, C.c_char_p, _P, _L]),
    "fg_relu_forward": (_I, [_P, _P, _P, _L]),
    "fg_relu_backward": (_I, [_P, _P, _P, _P, _L]),
    "fg_tanh_forward": (_I, [_P, _P, _P, _L]),
    "fg_tanh_backward": (_I, [_P, _P, _P, _P, _L]),
    "fg_abs_forward": (_I, [_P, _P, _P, _L, _P]),
    "fg_abs_backward": (_I, [_P, _P, _P, _L, _P]),
}

MAX_ITERS = 16  # the most D or G iterations one call runs (fg_train_step_iters)


def check_iters(D_iterations, G_iterations):
    """train.lua --D_iterations / --G_iterations as the _iters entry points take them: integers in [1, 16].
    D_iterations = 0 is not supported.  Raises ValueError before anything runs."""
    for name, v in (("D_iterations", D_iterations), ("G_iterations", G_iterations)):
        if int(v) != v or not 1 <= int(v) <= MAX_ITERS:
            raise ValueError("%s = %r: must be an integer in [1, %d]" % (name, v, MAX_ITERS))
    return int(D_iterations), int(G_iterations)


def iteration_root(seed, j):
    """The stream root of iteration j of a multi-iteration step with step seed `seed` (fg_b200.h): the seed itself for
    j = 0, else 2^60 | seed << 8 | j (64-bit).  Dropout masks of iteration j use 2*root+1 (D) / 2*root+2 (G); the
    device-fed steps draw from 4*root+k (8*root+k for c2f)."""
    seed = int(seed) & (2 ** 64 - 1)
    if j == 0:
        return seed
    return ((1 << 60) | (seed << 8) | int(j)) & (2 ** 64 - 1)

_lib = None


def load_library(path=None):
    """Load libfg_b200.so and bind every declared symbol.  Raises FGError if it is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or _SO
    if not os.path.exists(path):
        raise FGError("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                      "(there is no CPU fallback)" % path)
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError => the .so does not match include/fg_b200.h
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _check(rc, what):
    if rc != 0:
        raise FGError("%s failed (%d): %s" % (what, rc, load_library().fg_last_error().decode()))


def hyper_default(**kw):
    h = Hyper()
    load_library().fg_hyper_default(C.byref(h))
    for k, v in kw.items():
        if not hasattr(h, k):
            raise KeyError(k)
        setattr(h, k, v)
    return h


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.dtype == np.float32 and a.flags.c_contiguous, "float32 C-contiguous arrays only"
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))  # raw (device or pinned host) address


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


class PinnedArray:
    """float32 numpy view over cudaMallocHost memory (so H2D copies in the e2e path are truly async)."""

    def __init__(self, shape):
        self.shape = tuple(shape)
        n = int(np.prod(self.shape))
        self.addr = load_library().fg_host_alloc_pinned(max(n, 1) * 4)
        if not self.addr:
            raise FGError("fg_host_alloc_pinned failed: " + load_library().fg_last_error().decode())
        buf = (C.c_float * n).from_address(self.addr)
        self.array = np.frombuffer(buf, dtype=np.float32).reshape(self.shape)

    def free(self):
        if self.addr:
            load_library().fg_host_free_pinned(self.addr)
            self.addr = None


def _stats(st):
    """fg_step_stats -> dict (None when no statistics were asked for)"""
    if st is None:
        return None
    return dict(loss_D=st.loss_D, loss_G=st.loss_G, conf=list(st.conf), trained_D=st.trained_D, t_D=st.t_D,
                t_G=st.t_G, acc_D=st.acc_D)


class _NetPair:
    """What Context, C2f and S16 share: the flat parameters, gradients and optimizer state of one G/D pair, reached
    through the C entry points _prefix + "set_params", _prefix + "get_grads", ..."""
    _prefix = "fg_"  # "fg_", "fg_c2f_" or "fg_s16_"
    _what = ""       # how errors of _sized name the nets: "", "c2f ", "s16 "

    def _call(self, name, *args):
        fn = self._prefix + name
        _check(getattr(self.lib, fn)(self.h, *args), fn)

    def count(self, net):
        return self.nD if net == NET_D else self.nG

    def _sized(self, what, a, n):
        """the C ABI copies exactly n floats from the pointer it is given: a shorter buffer (a checkpoint written by a
        1- vs 3-channel build, a truncated or hostile file) would be read out of bounds, so sizes are checked here
        with a real error (asserts vanish under python -O)"""
        a = f32(a)
        if a.size != n:
            raise FGError("%s%s: expected %d floats, got %d" % (self._what, what, n, a.size))
        return a

    def _masks(self, what, m, rows):
        """host keep flags for `rows` samples of this pair's D: the C ABI reads rows * mask_per_sample floats, so a
        shorter array (flags of another discriminator) is refused.  Raw addresses pass as they are."""
        if m is None or not hasattr(m, "shape"):
            return m
        m = f32(m)
        n = rows * self.mask_per_sample
        if m.size < n:
            raise FGError("%s%s: %d keep flags for %d samples of %d, got %d"
                          % (self._what, what, n, rows, self.mask_per_sample, m.size))
        return m

    def set_params(self, net, p):
        self._call("set_params", net, _ptr(self._sized("set_params", p, self.count(net))))

    def get_params(self, net):
        out = np.empty(self.count(net), np.float32)
        self._call("get_params", net, _ptr(out))
        return out

    def get_grads(self, net):
        out = np.empty(self.count(net), np.float32)
        self._call("get_grads", net, _ptr(out))
        return out

    def zero_grads(self, net):
        self._call("zero_grads", net)

    def set_adam_state(self, net, m, v, t):
        m = None if m is None else self._sized("set_adam_state m", m, self.count(net))
        v = None if v is None else self._sized("set_adam_state v", v, self.count(net))
        self._call("set_adam_state", net, _ptr(m), _ptr(v), int(t))

    def get_adam_state(self, net):
        m, v, t = np.empty(self.count(net), np.float32), np.empty(self.count(net), np.float32), C.c_int(0)
        self._call("get_adam_state", net, _ptr(m), _ptr(v), C.byref(t))
        return m, v, t.value

    def dp_broadcast_params(self):
        self._call("dp_broadcast_params")

    def debug_tensor(self, name):
        """an internal tensor of the last forward / train step as stored (NHWC), flat float32 (tests)"""
        fn = getattr(self.lib, self._prefix + "debug_tensor")
        n = fn(self.h, name.encode(), None, 0)
        if n < 0:
            raise FGError("%sdebug_tensor(%s): %d: %s" % (self._prefix, name, n, self.lib.fg_last_error().decode()))
        out = np.empty(n, np.float32)
        r = fn(self.h, name.encode(), _ptr(out), n)
        if r < 0:
            raise FGError("%sdebug_tensor(%s): %d" % (self._prefix, name, r))
        return out


class _BatchNormNetPair(_NetPair):
    """A pair whose G has BatchNorm layers: their running statistics, [mean1 256][var1 256][mean2 128][var2 128]."""

    def set_bn_state(self, s):
        self._call("set_bn_state", _ptr(self._sized("set_bn_state", s, 768)))

    def get_bn_state(self):
        out = np.empty(768, np.float32)
        self._call("get_bn_state", _ptr(out))
        return out


# models.lua's discriminators by the name of the function that builds them (include/fg_b200.h FG_DISC_*)
DISCRIMINATORS = {"create_D32b": 1, "create_D16_d": 2, "create_D32": 3, "create_D16": 4, "create_D16_b": 5,
                  "create_D16_c": 6}


def disc_id(name):
    """FG_DISC_* of a models.lua discriminator name ("create_D32", ...)"""
    if name not in DISCRIMINATORS:
        raise FGError("unknown discriminator %r: models.lua defines %s" % (name, ", ".join(sorted(DISCRIMINATORS))))
    return DISCRIMINATORS[name]


def disc_param_count(name, channels):
    """length of the discriminator's getParameters() vector"""
    return int(load_library().fg_disc_param_count(disc_id(name), channels))


def disc_mask_per_sample(name):
    """the discriminator's (Spatial)Dropout keep flags per sample, in module order"""
    return int(load_library().fg_disc_mask_per_sample(disc_id(name)))


class Context(_BatchNormNetPair):
    """One fg_ctx (one GPU).  Mirrors face_generator_b200/lua/b200.lua's `b200.Context`.  discriminator: the 32x32
    D, "create_D32b" (models.lua's choice) or "create_D32"."""

    def __init__(self, device=0, max_batch=256, channels=3, discriminator="create_D32b"):
        self.lib = load_library()
        h = C.c_void_p()
        disc = disc_id(discriminator)
        _check(self.lib.fg_create_disc(C.byref(h), device, max_batch, channels, disc), "fg_create_disc")
        self.h, self.C, self.max_batch, self.device = h, channels, max_batch, device
        self.discriminator = discriminator
        self.nG = int(self.lib.fg_param_count(NET_G, channels))
        self.nD = int(self.lib.fg_disc_param_count(disc, channels))
        self.mask_per_sample = int(self.lib.fg_disc_mask_per_sample(disc))

    def close(self):
        if self.h:
            self.lib.fg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key, value):
        _check(self.lib.fg_set_option(self.h, key.encode(), int(value)), "fg_set_option(%s)" % key)

    def get_option(self, key):
        return int(self.lib.fg_get_option(self.h, key.encode()))

    def set_optimizer(self, net, method, momentum=0.0):
        """OPT.D_optmethod / G_optmethod: "adam" | "adagrad" | "sgd" (train.lua:38-39); momentum only for sgd."""
        which = "D" if net == NET_D else "G"
        self.set_option("optimizer_" + which, {"adam": 0, "adagrad": 1, "sgd": 2}[method])
        _check(self.lib.fg_set_option_f(self.h, ("sgd_momentum_" + which).encode(), float(momentum)), "fg_set_option_f")

    def sync(self):
        _check(self.lib.fg_sync(self.h), "fg_sync")

    # ---- L-net ----
    def G_forward(self, noise, training=True, want_images=True):
        noise = f32(noise)
        B = noise.shape[0]
        out = np.empty((B, self.C, 32, 32), np.float32) if want_images else None
        _check(self.lib.fg_G_forward(self.h, _ptr(noise), B, int(training), _ptr(out)), "fg_G_forward")
        return out

    def G_backward(self, d_images, want_dnoise=False):
        d_images = f32(d_images)
        dn = np.empty((d_images.shape[0], NOISE_DIM), np.float32) if want_dnoise else None
        _check(self.lib.fg_G_backward(self.h, _ptr(d_images), _ptr(dn)), "fg_G_backward")
        return dn

    def D_forward(self, images, masks=None, training=True, seed=0):
        images = f32(images)
        B = images.shape[0]
        masks = self._masks("D_forward", masks, B)
        out = np.empty(B, np.float32)
        _check(self.lib.fg_D_forward(self.h, _ptr(images), B, int(training), _ptr(masks), seed, _ptr(out)), "fg_D_forward")
        return out

    def D_backward(self, d_out, want_wgrad=True, want_dimages=True):
        d_out = f32(d_out)
        B = d_out.shape[0]
        di = np.empty((B, self.C, 32, 32), np.float32) if want_dimages else None
        _check(self.lib.fg_D_backward(self.h, _ptr(d_out), int(want_wgrad), _ptr(di)), "fg_D_backward")
        return di

    def bce_forward(self, x, t):
        x, t = f32(x).ravel(), f32(t).ravel()
        out = np.empty(1, np.float32)
        _check(self.lib.fg_bce_forward(self.h, _ptr(x), _ptr(t), x.size, _ptr(out)), "fg_bce_forward")
        return float(out[0])

    def bce_backward(self, x, t):
        x, t = f32(x).ravel(), f32(t).ravel()
        dx = np.empty(x.size, np.float32)
        _check(self.lib.fg_bce_backward(self.h, _ptr(x), _ptr(t), x.size, _ptr(dx)), "fg_bce_backward")
        return dx

    def optim_step(self, net, hyper, grad_scale=1.0):
        _check(self.lib.fg_optim_step(self.h, net, C.byref(hyper), grad_scale), "fg_optim_step")

    # ---- L-step ----
    def train_step(self, hyper, B, real, noise_D, noise_G, masks_D=None, masks_G=None, seed=0, want_stats=True):
        """Pointers may be numpy float32 arrays (host) or raw addresses (device / pinned)."""
        masks_D, masks_G = self._masks("train_step masks_D", masks_D, B), self._masks("train_step masks_G", masks_G, B)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_train_step(self.h, C.byref(hyper), B, _ptr(real), _ptr(noise_D), _ptr(noise_G),
                                      _ptr(masks_D), _ptr(masks_G), seed, C.byref(st) if st is not None else None),
               "fg_train_step")
        return _stats(st)

    def train_step_iters(self, hyper, B, D_iterations, G_iterations, real, noise_D, noise_G, masks_D=None, masks_G=None,
                         seed=0, want_stats=True):
        """D_iterations D iterations + G_iterations G iterations in one call (fg_train_step_iters); the inputs of
        train_step stacked per iteration: real [d][B/2][C][32][32], noise_D [d][B/2][100], noise_G [g][B][100],
        masks_* [d|g][B][mask_per_sample] or None (mask_per_sample: 1984 for create_D32b)."""
        d, g = check_iters(D_iterations, G_iterations)
        masks_D = self._masks("train_step_iters masks_D", masks_D, d * B)
        masks_G = self._masks("train_step_iters masks_G", masks_G, g * B)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_train_step_iters(self.h, C.byref(hyper), B, d, g, _ptr(real), _ptr(noise_D), _ptr(noise_G),
                                            _ptr(masks_D), _ptr(masks_G), seed, C.byref(st) if st is not None else None),
               "fg_train_step_iters")
        return _stats(st)

    def sample(self, noise, chunk):
        noise = f32(noise)
        N = noise.shape[0]
        out = np.empty((N, self.C, 32, 32), np.float32)
        _check(self.lib.fg_sample(self.h, _ptr(noise), N, chunk, _ptr(out)), "fg_sample")
        return out

    # ---- device memory helpers ----
    def dev_array(self, host):
        host = f32(host)
        p = self.lib.fg_dev_alloc(max(host.nbytes, 4))
        if not p:
            raise FGError("fg_dev_alloc failed")
        _check(self.lib.fg_memcpy(self.h, p, _ptr(host), host.nbytes), "fg_memcpy")
        return p

    def dev_free(self, p):
        self.lib.fg_dev_free(p)

    def tf32_peak(self, iters=20000):
        """measured tf32 wgmma issue rate in TFLOP/s (roofline denominator of the 3xTF32 convolutions)"""
        v = C.c_double(0)
        _check(self.lib.fg_bench_tf32_peak(self.h, iters, C.byref(v)), "fg_bench_tf32_peak")
        return v.value

    def launches(self):
        return int(self.lib.fg_kernel_launches(self.h))

    def event_record(self, slot):
        _check(self.lib.fg_event_record(self.h, slot), "fg_event_record")

    def event_elapsed_ms(self, a, b):
        ms = C.c_double(0)
        _check(self.lib.fg_event_elapsed_ms(self.h, a, b, C.byref(ms)), "fg_event_elapsed_ms")
        return ms.value

    def timing_enable(self, on=True):
        _check(self.lib.fg_timing_enable(self.h, int(on)), "fg_timing_enable")

    def timing_get(self, prefix):
        ms, n = C.c_double(0), C.c_int64(0)
        _check(self.lib.fg_timing_get(self.h, prefix.encode(), C.byref(ms), C.byref(n)), "fg_timing_get")
        return ms.value, n.value

    # ---- data parallel ----
    def dp_unique_id(self):
        buf = (C.c_ubyte * 128)()
        _check(self.lib.fg_dp_unique_id(buf), "fg_dp_unique_id")
        return bytes(buf)

    def dp_init(self, id_bytes, nranks, rank):
        buf = (C.c_ubyte * 128).from_buffer_copy(id_bytes)
        _check(self.lib.fg_dp_init(self.h, buf, nranks, rank), "fg_dp_init")

    # ---- L-op: resampling / pooling / dropout / sigmoid at the nn.Module boundary (NCHW numpy in/out) ----
    def upsample2_forward(self, x):
        x = f32(x)
        N, Cc, H, W = x.shape
        y = np.empty((N, Cc, 2 * H, 2 * W), np.float32)
        _check(self.lib.fg_upsample2_forward(self.h, _ptr(x), _ptr(y), N, Cc, H, W), "fg_upsample2_forward")
        return y

    def upsample2_backward(self, dy):
        dy = f32(dy)
        N, Cc, H2, W2 = dy.shape
        dx = np.empty((N, Cc, H2 // 2, W2 // 2), np.float32)
        _check(self.lib.fg_upsample2_backward(self.h, _ptr(dy), _ptr(dx), N, Cc, H2 // 2, W2 // 2), "fg_upsample2_backward")
        return dx

    def avgpool2_forward(self, x):
        x = f32(x)
        N, Cc, H, W = x.shape
        y = np.empty((N, Cc, H // 2, W // 2), np.float32)
        _check(self.lib.fg_avgpool2_forward(self.h, _ptr(x), _ptr(y), N, Cc, H, W), "fg_avgpool2_forward")
        return y

    def avgpool2_backward(self, dy):
        dy = f32(dy)
        N, Cc, Ho, Wo = dy.shape
        dx = np.empty((N, Cc, 2 * Ho, 2 * Wo), np.float32)
        _check(self.lib.fg_avgpool2_backward(self.h, _ptr(dy), _ptr(dx), N, Cc, 2 * Ho, 2 * Wo), "fg_avgpool2_backward")
        return dx

    def maxpool2_forward(self, x):
        x = f32(x)
        N, Cc, H, W = x.shape
        y = np.empty((N, Cc, H // 2, W // 2), np.float32)
        _check(self.lib.fg_maxpool2_forward(self.h, _ptr(x), _ptr(y), N, Cc, H, W), "fg_maxpool2_forward")
        return y

    def maxpool2_backward(self, x, dy):
        x, dy = f32(x), f32(dy)
        N, Cc, H, W = x.shape
        dx = np.empty_like(x)
        _check(self.lib.fg_maxpool2_backward(self.h, _ptr(x), _ptr(dy), _ptr(dx), N, Cc, H, W), "fg_maxpool2_backward")
        return dx

    def dropout_forward(self, x, mask, p, spatial=False):
        """x [N][C][H][W] (or [N][F]); mask: keep flags (same shape as x, or [N][C] when spatial) / None = evaluate()."""
        x = f32(x)
        N, Cc = x.shape[0], x.shape[1]
        HW = int(np.prod(x.shape[2:])) if x.ndim > 2 else 1
        mask = f32(mask) if mask is not None else None
        y = np.empty_like(x)
        _check(self.lib.fg_dropout_forward(self.h, _ptr(x), _ptr(mask), p, int(spatial), _ptr(y), N, Cc, HW),
               "fg_dropout_forward")
        return y

    def dropout_backward(self, dy, mask, p, spatial=False):
        dy = f32(dy)
        N, Cc = dy.shape[0], dy.shape[1]
        HW = int(np.prod(dy.shape[2:])) if dy.ndim > 2 else 1
        mask = f32(mask) if mask is not None else None
        dx = np.empty_like(dy)
        _check(self.lib.fg_dropout_backward(self.h, _ptr(dy), _ptr(mask), p, int(spatial), _ptr(dx), N, Cc, HW),
               "fg_dropout_backward")
        return dx

    def dropout_mask(self, n, p, seed):
        """keep flags drawn on the device (throughput mode), returned as a host array for inspection."""
        dev = self.lib.fg_dev_alloc(n * 4)
        if not dev:
            raise FGError("fg_dev_alloc failed")
        try:
            _check(self.lib.fg_dropout_mask(self.h, dev, n, p, seed), "fg_dropout_mask")
            out = np.empty(n, np.float32)
            _check(self.lib.fg_memcpy(self.h, _ptr(out), dev, n * 4), "fg_memcpy")
            self.sync()
        finally:
            self.lib.fg_dev_free(dev)
        return out

    def sigmoid_forward(self, x):
        x = f32(x)
        y = np.empty_like(x)
        _check(self.lib.fg_sigmoid_forward(self.h, _ptr(x), _ptr(y), x.size), "fg_sigmoid_forward")
        return y

    def sigmoid_backward(self, y, dy):
        y, dy = f32(y), f32(dy)
        dx = np.empty_like(y)
        _check(self.lib.fg_sigmoid_backward(self.h, _ptr(y), _ptr(dy), _ptr(dx), y.size), "fg_sigmoid_backward")
        return dx


C2F_MASK_PER_SAMPLE = 16384 + 512
C2F_FINE_SIZES = (16, 32, 64)


# models_c2f.lua's generators and discriminators by the name of the function that builds them (include/fg_b200.h
# FG_C2F_G_* / FG_C2F_D_*); create_G / create_D resolve to create_G_d / create_D_c
C2F_GENERATORS = {"create_G_d": 1, "create_G_a": 2, "create_G_b": 3, "create_G_c": 4}
C2F_DISCRIMINATORS = {"create_D_c": 1, "create_D_a": 2, "create_D_b": 3}


def c2f_gen_id(name):
    """FG_C2F_G_* of a models_c2f.lua generator name ("create_G_a", ...)"""
    if name not in C2F_GENERATORS:
        raise FGError("unknown c2f generator %r: models_c2f.lua defines %s" % (name, ", ".join(sorted(C2F_GENERATORS))))
    return C2F_GENERATORS[name]


def c2f_disc_id(name):
    """FG_C2F_D_* of a models_c2f.lua discriminator name ("create_D_a", ...)"""
    if name not in C2F_DISCRIMINATORS:
        raise FGError("unknown c2f discriminator %r: models_c2f.lua defines %s"
                      % (name, ", ".join(sorted(C2F_DISCRIMINATORS))))
    return C2F_DISCRIMINATORS[name]


def _c2f_size(n, what):
    """a count of the C ABI, or FGError for its -1 (a channel count below 1 or a fine size other than 16, 32, 64)"""
    n = int(n)
    if n < 0:
        raise FGError("%s is not supported (channels >= 1; fine size 16, 32 or 64)" % what)
    return n


def c2f_gen_param_count(name, channels):
    """length of the c2f generator's getParameters() vector"""
    n = load_library().fg_c2f_gen_param_count(c2f_gen_id(name), channels)
    return _c2f_size(n, "%s with %d channels" % (name, channels))


def c2f_disc_param_count(name, channels, fine_size):
    """length of the c2f discriminator's getParameters() vector at fine size S"""
    n = load_library().fg_c2f_disc_param_count(c2f_disc_id(name), channels, fine_size)
    return _c2f_size(n, "%s with %d channels at fine size %d" % (name, channels, fine_size))


def c2f_mask_per_sample(fine_size=32, discriminator="create_D_c"):
    """nn.Dropout keep flags per sample of a coarse-to-fine D at fine size S: its last pooled map (create_D_c:
    [256][S/4][S/4]) then [512]"""
    n = load_library().fg_c2f_disc_mask_per_sample(c2f_disc_id(discriminator), fine_size)
    return _c2f_size(n, "%s at fine size %d" % (discriminator, fine_size))


class C2f(_NetPair):
    """Coarse-to-fine nets + loop (train_c2f.lua) on a Context at fine size S = train_c2f.lua --fineSize (16, 32 or
    64).  generator / discriminator: models_c2f.lua's nets by name (C2F_GENERATORS, C2F_DISCRIMINATORS; the defaults
    are models_c2f.lua's create_G / create_D).  Mirrors lua/adversarial_c2f_b200.lua."""
    _prefix, _what = "fg_c2f_", "c2f "

    def __init__(self, ctx, fine_size=32, generator="create_G_d", discriminator="create_D_c"):
        self.ctx, self.lib, self.C = ctx, ctx.lib, ctx.C
        gen, disc = c2f_gen_id(generator), c2f_disc_id(discriminator)
        h = C.c_void_p()
        _check(self.lib.fg_c2f_create_nets(ctx.h, fine_size, gen, disc, C.byref(h)), "fg_c2f_create_nets")
        self.h = h
        self.generator, self.discriminator = generator, discriminator
        self.S = int(self.lib.fg_c2f_fine_size(h))
        self.mask_per_sample = int(self.lib.fg_c2f_disc_mask_per_sample(disc, self.S))
        self.nG = int(self.lib.fg_c2f_gen_param_count(gen, self.C))
        self.nD = int(self.lib.fg_c2f_disc_param_count(disc, self.C, self.S))

    def close(self):
        if self.h:
            self.lib.fg_c2f_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h:
                self.close()
        except Exception:
            pass

    def G_forward(self, noise, cond, want_diff=True):
        noise, cond = f32(noise), f32(cond)
        B = cond.shape[0]
        out = np.empty((B, self.C, self.S, self.S), np.float32) if want_diff else None
        _check(self.lib.fg_c2f_G_forward(self.h, _ptr(noise), _ptr(cond), B, _ptr(out)), "fg_c2f_G_forward")
        return out

    def G_backward(self, d_diff):
        _check(self.lib.fg_c2f_G_backward(self.h, _ptr(f32(d_diff))), "fg_c2f_G_backward")

    def D_forward(self, diff, cond, masks=None, training=True, seed=0):
        diff, cond = f32(diff), f32(cond)
        B = diff.shape[0]
        masks = self._masks("D_forward masks", masks, B)
        out = np.empty(B, np.float32)
        _check(self.lib.fg_c2f_D_forward(self.h, _ptr(diff), _ptr(cond), B, int(training), _ptr(masks), seed, _ptr(out)),
               "fg_c2f_D_forward")
        return out

    def D_backward(self, d_out, want_wgrad=True, want_ddiff=True):
        d_out = f32(d_out)
        dd = np.empty((d_out.shape[0], self.C, self.S, self.S), np.float32) if want_ddiff else None
        _check(self.lib.fg_c2f_D_backward(self.h, _ptr(d_out), int(want_wgrad), _ptr(dd)), "fg_c2f_D_backward")
        return dd

    def train_step(self, hyper, B, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D=None, masks_G=None, seed=0,
                   want_stats=True):
        """Pointers may be numpy float32 arrays (host) or raw addresses (device / pinned)."""
        masks_D, masks_G = self._masks("train_step masks_D", masks_D, B), self._masks("train_step masks_G", masks_G, B)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_c2f_train_step(self.h, C.byref(hyper), B, _ptr(real_diff), _ptr(cond_D), _ptr(noise_D),
                                          _ptr(cond_G), _ptr(noise_G), _ptr(masks_D), _ptr(masks_G), seed,
                                          C.byref(st) if st is not None else None), "fg_c2f_train_step")
        return _stats(st)

    def train_step_dataset(self, dataset, hyper, B, coarse_size, seed, want_stats=True):
        """train_step with the pairs, conditions and noise drawn on the device from a DeviceDataset of this ctx
        (fg_c2f_train_step_dataset); coarse_size = train_c2f.lua --coarseSize."""
        st = StepStats() if want_stats else None
        _check(self.lib.fg_c2f_train_step_dataset(self.h, dataset.h, C.byref(hyper), B, coarse_size, seed,
                                                  C.byref(st) if st is not None else None), "fg_c2f_train_step_dataset")
        return _stats(st)

    def train_step_iters(self, hyper, B, D_iterations, G_iterations, real_diff, cond_D, noise_D, cond_G, noise_G,
                         masks_D=None, masks_G=None, seed=0, want_stats=True):
        """D_iterations D iterations + G_iterations G iterations in one call (fg_c2f_train_step_iters); the train_step
        inputs stacked per iteration: real_diff [d][B/2], cond_D [d][B], noise_D [d][B/2], cond_G / noise_G [g][B],
        masks_* [d|g][B][mask_per_sample] or None."""
        d, g = check_iters(D_iterations, G_iterations)
        masks_D = self._masks("train_step_iters masks_D", masks_D, d * B)
        masks_G = self._masks("train_step_iters masks_G", masks_G, g * B)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_c2f_train_step_iters(self.h, C.byref(hyper), B, d, g, _ptr(real_diff), _ptr(cond_D),
                                                _ptr(noise_D), _ptr(cond_G), _ptr(noise_G), _ptr(masks_D), _ptr(masks_G),
                                                seed, C.byref(st) if st is not None else None), "fg_c2f_train_step_iters")
        return _stats(st)

    def train_step_dataset_iters(self, dataset, hyper, B, D_iterations, G_iterations, coarse_size, seed, want_stats=True):
        """train_step_iters with every input drawn on the device, inside the step (fg_c2f_train_step_dataset_iters)."""
        d, g = check_iters(D_iterations, G_iterations)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_c2f_train_step_dataset_iters(self.h, dataset.h, C.byref(hyper), B, d, g, coarse_size, seed,
                                                        C.byref(st) if st is not None else None),
               "fg_c2f_train_step_dataset_iters")
        return _stats(st)


S16_MASK_PER_SAMPLE = 1024 + 128


class S16(_BatchNormNetPair):
    """The --scale 16 nets (models.lua:27-51 G16, :279-316 D16_d) + the adversarial.lua loop on a Context.
    discriminator: "create_D16_d" (models.lua's choice), "create_D16", "create_D16_b" or "create_D16_c"."""
    _prefix, _what = "fg_s16_", "s16 "

    def __init__(self, ctx, discriminator="create_D16_d"):
        self.ctx, self.lib, self.C = ctx, ctx.lib, ctx.C
        h = C.c_void_p()
        disc = disc_id(discriminator)
        _check(self.lib.fg_s16_create_disc(ctx.h, disc, C.byref(h)), "fg_s16_create_disc")
        self.h = h
        self.discriminator = discriminator
        self.nG = int(self.lib.fg_s16_param_count(NET_G, self.C))
        self.nD = int(self.lib.fg_disc_param_count(disc, self.C))
        self.mask_per_sample = int(self.lib.fg_disc_mask_per_sample(disc))

    def close(self):
        if self.h:
            self.lib.fg_s16_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h:
                self.close()
        except Exception:
            pass

    def G_forward(self, noise, training=True, want_img=True):
        noise = f32(noise)
        B = noise.shape[0]
        out = np.empty((B, self.C, 16, 16), np.float32) if want_img else None
        _check(self.lib.fg_s16_G_forward(self.h, _ptr(noise), B, int(training), _ptr(out)), "fg_s16_G_forward")
        return out

    def G_backward(self, d_img, want_dnoise=False):
        d_img = f32(d_img)
        dn = np.empty((d_img.shape[0], NOISE_DIM), np.float32) if want_dnoise else None
        _check(self.lib.fg_s16_G_backward(self.h, _ptr(d_img), _ptr(dn)), "fg_s16_G_backward")
        return dn

    def D_forward(self, img, masks=None, training=True, seed=0):
        img = f32(img)
        B = img.shape[0]
        masks = self._masks("D_forward", masks, B)
        out = np.empty(B, np.float32)
        _check(self.lib.fg_s16_D_forward(self.h, _ptr(img), B, int(training), _ptr(masks), seed, _ptr(out)), "fg_s16_D_forward")
        return out

    def D_backward(self, d_out, want_wgrad=True, want_dimg=True):
        d_out = f32(d_out)
        dd = np.empty((d_out.shape[0], self.C, 16, 16), np.float32) if want_dimg else None
        _check(self.lib.fg_s16_D_backward(self.h, _ptr(d_out), int(want_wgrad), _ptr(dd)), "fg_s16_D_backward")
        return dd

    def train_step(self, hyper, B, real, noise_D, noise_G, masks_D=None, masks_G=None, seed=0, want_stats=True):
        """Pointers may be numpy float32 arrays (host) or raw addresses (device / pinned)."""
        masks_D, masks_G = self._masks("train_step masks_D", masks_D, B), self._masks("train_step masks_G", masks_G, B)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_s16_train_step(self.h, C.byref(hyper), B, _ptr(real), _ptr(noise_D), _ptr(noise_G), _ptr(masks_D),
                                          _ptr(masks_G), seed, C.byref(st) if st is not None else None), "fg_s16_train_step")
        return _stats(st)

    def train_step_dataset(self, dataset, hyper, B, seed, want_stats=True):
        """train_step with the 16x16 real half and the noise drawn on the device from a DeviceDataset of this ctx
        (fg_s16_train_step_dataset)."""
        st = StepStats() if want_stats else None
        _check(self.lib.fg_s16_train_step_dataset(self.h, dataset.h, C.byref(hyper), B, seed,
                                                  C.byref(st) if st is not None else None), "fg_s16_train_step_dataset")
        return _stats(st)

    def train_step_iters(self, hyper, B, D_iterations, G_iterations, real, noise_D, noise_G, masks_D=None, masks_G=None,
                         seed=0, want_stats=True):
        """fg_s16_train_step_iters: train_step's inputs stacked per iteration (real [d][B/2][C][16][16], noise_D
        [d][B/2][100], noise_G [g][B][100], masks_* [d|g][B][mask_per_sample] or None; 1152 for create_D16_d)."""
        d, g = check_iters(D_iterations, G_iterations)
        masks_D = self._masks("train_step_iters masks_D", masks_D, d * B)
        masks_G = self._masks("train_step_iters masks_G", masks_G, g * B)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_s16_train_step_iters(self.h, C.byref(hyper), B, d, g, _ptr(real), _ptr(noise_D), _ptr(noise_G),
                                                _ptr(masks_D), _ptr(masks_G), seed, C.byref(st) if st is not None else None),
               "fg_s16_train_step_iters")
        return _stats(st)

    def train_step_dataset_iters(self, dataset, hyper, B, D_iterations, G_iterations, seed, want_stats=True):
        """train_step_iters with every input drawn on the device, inside the step (fg_s16_train_step_dataset_iters)."""
        d, g = check_iters(D_iterations, G_iterations)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_s16_train_step_dataset_iters(self.h, dataset.h, C.byref(hyper), B, d, g, seed,
                                                        C.byref(st) if st is not None else None),
               "fg_s16_train_step_dataset_iters")
        return _stats(st)
