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
    "fg_dataset_gather": (_I, [_P, _P, _I, _P]),
    "fg_dataset_draw": (_I, [_P, _U64, _I, _P]),
    "fg_noise_uniform": (_I, [_P, _U64, _L, _P]),
    "fg_train_step_dataset": (_I, [_P, _P, C.POINTER(Hyper), _I, _U64, C.POINTER(StepStats)]),
    "fg_D_score": (_I, [_P, _P, _L, _I, _I, _U64, _P]),
    "fg_nearest": (_I, [_P, _P, _I, _P, _L, _I, _P, _P]),
    "fg_dataset_nearest": (_I, [_P, _P, _I, _P, _P]),
    "fg_c2f_parzen_dist": (_I, [_P, _P, _P, _P, _I, _P]),
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
    "fg_bench_tf32_peak": (_I, [_P, _I, C.POINTER(C.c_double)]),
    "fg_event_record": (_I, [_P, _I]),
    "fg_event_elapsed_ms": (_I, [_P, _I, _I, C.POINTER(C.c_double)]),
    "fg_timing_enable": (_I, [_P, _I]),
    "fg_timing_get": (_I, [_P, C.c_char_p, C.POINTER(C.c_double), C.POINTER(_L)]),
}

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


class Context:
    """One fg_ctx (one GPU).  Mirrors face_generator_b200/lua/b200.lua's `b200.Context`."""

    def __init__(self, device=0, max_batch=256, channels=3):
        self.lib = load_library()
        h = C.c_void_p()
        _check(self.lib.fg_create(C.byref(h), device, max_batch, channels), "fg_create")
        self.h, self.C, self.max_batch, self.device = h, channels, max_batch, device
        self.nG = int(self.lib.fg_param_count(NET_G, channels))
        self.nD = int(self.lib.fg_param_count(NET_D, channels))

    def close(self):
        if self.h:
            self.lib.fg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters ----
    def count(self, net):
        return self.nD if net == NET_D else self.nG

    def _sized(self, what, a, n):
        """the C ABI copies exactly n floats from the pointer it is given: a shorter buffer (a checkpoint written by a
        1- vs 3-channel build, a truncated or hostile file) would be read out of bounds, so sizes are checked here
        with a real error (asserts vanish under python -O)"""
        a = f32(a)
        if a.size != n:
            raise FGError("%s: expected %d floats, got %d" % (what, n, a.size))
        return a

    def set_params(self, net, p):
        p = self._sized("set_params", p, self.count(net))
        _check(self.lib.fg_set_params(self.h, net, _ptr(p)), "fg_set_params")

    def get_params(self, net):
        out = np.empty(self.count(net), np.float32)
        _check(self.lib.fg_get_params(self.h, net, _ptr(out)), "fg_get_params")
        return out

    def get_grads(self, net):
        out = np.empty(self.count(net), np.float32)
        _check(self.lib.fg_get_grads(self.h, net, _ptr(out)), "fg_get_grads")
        return out

    def zero_grads(self, net):
        _check(self.lib.fg_zero_grads(self.h, net), "fg_zero_grads")

    def set_adam_state(self, net, m, v, t):
        m = None if m is None else self._sized("set_adam_state m", m, self.count(net))
        v = None if v is None else self._sized("set_adam_state v", v, self.count(net))
        _check(self.lib.fg_set_adam_state(self.h, net, _ptr(m), _ptr(v), int(t)), "fg_set_adam_state")

    def get_adam_state(self, net):
        m, v, t = np.empty(self.count(net), np.float32), np.empty(self.count(net), np.float32), C.c_int(0)
        _check(self.lib.fg_get_adam_state(self.h, net, _ptr(m), _ptr(v), C.byref(t)), "fg_get_adam_state")
        return m, v, t.value

    def set_bn_state(self, s):
        _check(self.lib.fg_set_bn_state(self.h, _ptr(self._sized("set_bn_state", s, 768))), "fg_set_bn_state")

    def get_bn_state(self):
        out = np.empty(768, np.float32)
        _check(self.lib.fg_get_bn_state(self.h, _ptr(out)), "fg_get_bn_state")
        return out

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
        masks = f32(masks) if masks is not None else None
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
        st = StepStats() if want_stats else None
        _check(self.lib.fg_train_step(self.h, C.byref(hyper), B, _ptr(real), _ptr(noise_D), _ptr(noise_G),
                                      _ptr(masks_D), _ptr(masks_G), seed, C.byref(st) if st is not None else None),
               "fg_train_step")
        if st is None:
            return None
        return dict(loss_D=st.loss_D, loss_G=st.loss_G, conf=list(st.conf), trained_D=st.trained_D, t_D=st.t_D,
                    t_G=st.t_G, acc_D=st.acc_D)

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

    def debug_tensor(self, name):
        n = self.lib.fg_debug_tensor(self.h, name.encode(), None, 0)
        if n < 0:
            raise FGError("fg_debug_tensor(%s): %d" % (name, n))
        out = np.empty(n, np.float32)
        r = self.lib.fg_debug_tensor(self.h, name.encode(), _ptr(out), n)
        if r < 0:
            raise FGError("fg_debug_tensor(%s): %d" % (name, r))
        return out

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

    def dp_broadcast_params(self):
        _check(self.lib.fg_dp_broadcast_params(self.h), "fg_dp_broadcast_params")

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


class C2f:
    """Coarse-to-fine nets + loop (train_c2f.lua) on a Context.  Mirrors lua/adversarial_c2f_b200.lua."""

    def __init__(self, ctx):
        self.ctx, self.lib, self.C = ctx, ctx.lib, ctx.C
        h = C.c_void_p()
        _check(self.lib.fg_c2f_create(ctx.h, C.byref(h)), "fg_c2f_create")
        self.h = h
        self.nG = int(self.lib.fg_c2f_param_count(NET_G, self.C))
        self.nD = int(self.lib.fg_c2f_param_count(NET_D, self.C))

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

    def count(self, net):
        return self.nD if net == NET_D else self.nG

    def _sized(self, what, a, n):
        a = f32(a)
        if a.size != n:
            raise FGError("%s: expected %d floats, got %d" % (what, n, a.size))
        return a

    def set_params(self, net, p):
        p = self._sized("c2f set_params", p, self.count(net))
        _check(self.lib.fg_c2f_set_params(self.h, net, _ptr(p)), "fg_c2f_set_params")

    def get_params(self, net):
        out = np.empty(self.count(net), np.float32)
        _check(self.lib.fg_c2f_get_params(self.h, net, _ptr(out)), "fg_c2f_get_params")
        return out

    def get_grads(self, net):
        out = np.empty(self.count(net), np.float32)
        _check(self.lib.fg_c2f_get_grads(self.h, net, _ptr(out)), "fg_c2f_get_grads")
        return out

    def zero_grads(self, net):
        _check(self.lib.fg_c2f_zero_grads(self.h, net), "fg_c2f_zero_grads")

    def set_adam_state(self, net, m, v, t):
        m = None if m is None else self._sized("c2f set_adam_state m", m, self.count(net))
        v = None if v is None else self._sized("c2f set_adam_state v", v, self.count(net))
        _check(self.lib.fg_c2f_set_adam_state(self.h, net, _ptr(m), _ptr(v), int(t)), "fg_c2f_set_adam_state")

    def get_adam_state(self, net):
        m, v, t = np.empty(self.count(net), np.float32), np.empty(self.count(net), np.float32), C.c_int(0)
        _check(self.lib.fg_c2f_get_adam_state(self.h, net, _ptr(m), _ptr(v), C.byref(t)), "fg_c2f_get_adam_state")
        return m, v, t.value

    def G_forward(self, noise, cond, want_diff=True):
        noise, cond = f32(noise), f32(cond)
        B = cond.shape[0]
        out = np.empty((B, self.C, 32, 32), np.float32) if want_diff else None
        _check(self.lib.fg_c2f_G_forward(self.h, _ptr(noise), _ptr(cond), B, _ptr(out)), "fg_c2f_G_forward")
        return out

    def G_backward(self, d_diff):
        _check(self.lib.fg_c2f_G_backward(self.h, _ptr(f32(d_diff))), "fg_c2f_G_backward")

    def D_forward(self, diff, cond, masks=None, training=True, seed=0):
        diff, cond = f32(diff), f32(cond)
        B = diff.shape[0]
        masks = f32(masks) if masks is not None else None
        out = np.empty(B, np.float32)
        _check(self.lib.fg_c2f_D_forward(self.h, _ptr(diff), _ptr(cond), B, int(training), _ptr(masks), seed, _ptr(out)),
               "fg_c2f_D_forward")
        return out

    def D_backward(self, d_out, want_wgrad=True, want_ddiff=True):
        d_out = f32(d_out)
        dd = np.empty((d_out.shape[0], self.C, 32, 32), np.float32) if want_ddiff else None
        _check(self.lib.fg_c2f_D_backward(self.h, _ptr(d_out), int(want_wgrad), _ptr(dd)), "fg_c2f_D_backward")
        return dd

    def dp_broadcast_params(self):
        _check(self.lib.fg_c2f_dp_broadcast_params(self.h), "fg_c2f_dp_broadcast_params")

    def train_step(self, hyper, B, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D=None, masks_G=None, seed=0,
                   want_stats=True):
        """Pointers may be numpy float32 arrays (host) or raw addresses (device / pinned)."""
        st = StepStats() if want_stats else None
        _check(self.lib.fg_c2f_train_step(self.h, C.byref(hyper), B, _ptr(real_diff), _ptr(cond_D), _ptr(noise_D),
                                          _ptr(cond_G), _ptr(noise_G), _ptr(masks_D), _ptr(masks_G), seed,
                                          C.byref(st) if st is not None else None), "fg_c2f_train_step")
        if st is None:
            return None
        return dict(loss_D=st.loss_D, loss_G=st.loss_G, conf=list(st.conf), t_D=st.t_D, t_G=st.t_G, acc_D=st.acc_D)


S16_MASK_PER_SAMPLE = 1024 + 128


class S16:
    """The --scale 16 nets (models.lua:27-51 G16, :279-316 D16_d) + the adversarial.lua loop on a Context."""

    def __init__(self, ctx):
        self.ctx, self.lib, self.C = ctx, ctx.lib, ctx.C
        h = C.c_void_p()
        _check(self.lib.fg_s16_create(ctx.h, C.byref(h)), "fg_s16_create")
        self.h = h
        self.nG = int(self.lib.fg_s16_param_count(NET_G, self.C))
        self.nD = int(self.lib.fg_s16_param_count(NET_D, self.C))

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

    def count(self, net):
        return self.nD if net == NET_D else self.nG

    def _sized(self, what, a, n):
        a = f32(a)
        if a.size != n:
            raise FGError("%s: expected %d floats, got %d" % (what, n, a.size))
        return a

    def set_params(self, net, p):
        p = self._sized("s16 set_params", p, self.count(net))
        _check(self.lib.fg_s16_set_params(self.h, net, _ptr(p)), "fg_s16_set_params")

    def get_params(self, net):
        out = np.empty(self.count(net), np.float32)
        _check(self.lib.fg_s16_get_params(self.h, net, _ptr(out)), "fg_s16_get_params")
        return out

    def get_grads(self, net):
        out = np.empty(self.count(net), np.float32)
        _check(self.lib.fg_s16_get_grads(self.h, net, _ptr(out)), "fg_s16_get_grads")
        return out

    def zero_grads(self, net):
        _check(self.lib.fg_s16_zero_grads(self.h, net), "fg_s16_zero_grads")

    def set_adam_state(self, net, m, v, t):
        m = None if m is None else self._sized("s16 set_adam_state m", m, self.count(net))
        v = None if v is None else self._sized("s16 set_adam_state v", v, self.count(net))
        _check(self.lib.fg_s16_set_adam_state(self.h, net, _ptr(m), _ptr(v), int(t)), "fg_s16_set_adam_state")

    def get_adam_state(self, net):
        m, v, t = np.empty(self.count(net), np.float32), np.empty(self.count(net), np.float32), C.c_int(0)
        _check(self.lib.fg_s16_get_adam_state(self.h, net, _ptr(m), _ptr(v), C.byref(t)), "fg_s16_get_adam_state")
        return m, v, t.value

    def set_bn_state(self, s):
        s = self._sized("s16 set_bn_state", s, 768)
        _check(self.lib.fg_s16_set_bn_state(self.h, _ptr(s)), "fg_s16_set_bn_state")

    def get_bn_state(self):
        out = np.empty(768, np.float32)
        _check(self.lib.fg_s16_get_bn_state(self.h, _ptr(out)), "fg_s16_get_bn_state")
        return out

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
        masks = f32(masks) if masks is not None else None
        out = np.empty(B, np.float32)
        _check(self.lib.fg_s16_D_forward(self.h, _ptr(img), B, int(training), _ptr(masks), seed, _ptr(out)), "fg_s16_D_forward")
        return out

    def D_backward(self, d_out, want_wgrad=True, want_dimg=True):
        d_out = f32(d_out)
        dd = np.empty((d_out.shape[0], self.C, 16, 16), np.float32) if want_dimg else None
        _check(self.lib.fg_s16_D_backward(self.h, _ptr(d_out), int(want_wgrad), _ptr(dd)), "fg_s16_D_backward")
        return dd

    def dp_broadcast_params(self):
        _check(self.lib.fg_s16_dp_broadcast_params(self.h), "fg_s16_dp_broadcast_params")

    def train_step(self, hyper, B, real, noise_D, noise_G, masks_D=None, masks_G=None, seed=0, want_stats=True):
        """Pointers may be numpy float32 arrays (host) or raw addresses (device / pinned)."""
        st = StepStats() if want_stats else None
        _check(self.lib.fg_s16_train_step(self.h, C.byref(hyper), B, _ptr(real), _ptr(noise_D), _ptr(noise_G), _ptr(masks_D),
                                          _ptr(masks_G), seed, C.byref(st) if st is not None else None), "fg_s16_train_step")
        if st is None:
            return None
        return dict(loss_D=st.loss_D, loss_G=st.loss_G, conf=list(st.conf), trained_D=st.trained_D, t_D=st.t_D, t_G=st.t_G,
                    acc_D=st.acc_D)
