"""The denoising autoencoders of train_denoiser.lua on the GPU (fg_dn_* entry points), and the host side of its epoch
loop.  Mirrors face_generator_b200/lua/denoiser_b200.lua.

    dn = Denoiser(ctx, 32)                    # AE1 = WhiteNoise + DECODER, AE2 = DECODER:clone(), at ctx.C x 32 x 32
    dn.set_params(0, P1); dn.set_params(1, P2)
    st = dn.train_step(hyper, images)         # fevalAE + adam, fevalAE2 + adam, on one Adam state
    clean = dn.denoise(images)                # train.lua --denoise: AE1_DECODER:evaluate():forward(images)
"""
import ctypes as C

import numpy as np

from .lib import DnHyper, DnStats, FGError, _check, _ptr, f32, load_library

AE1, AE2 = 0, 1
BN_STATE = 2 * (8 + 8 + 2048)  # [mean1 8][var1 8][mean2 8][var2 8][mean3 2048][var3 2048] per decoder


def dn_hyper_default(**kw):
    """lr 1e-3, betas 0.9 / 0.999, eps 1e-8 (optim.adam), L1 = L2 = 0, clamp 1 (--coefL1 / --coefL2 / --AE_clamp),
    p_drop 0.2, noise_std 0.1 (train_denoiser.lua:83-113)."""
    h = DnHyper()
    load_library().fg_dn_hyper_default(C.byref(h))
    for k, v in kw.items():
        if not hasattr(h, k):
            raise KeyError(k)
        setattr(h, k, v)
    return h


def param_count(channels, size):
    return int(load_library().fg_dn_param_count(channels, size))


def mask_per_sample(size):
    return int(load_library().fg_dn_mask_per_sample(size))


def layout(channels, size):
    """getParameters() order of one DECODER: [(name, shape)] of conv1 W/b, bn1 gamma/beta, conv2, bn2, lin1, bn3, lin2"""
    A, H, O = 8 * (size - 4) ** 2, 2048, channels * size * size
    return [("c1W", (8, channels, 3, 3)), ("c1b", (8,)), ("g1", (8,)), ("b1", (8,)), ("c2W", (8, 8, 3, 3)), ("c2b", (8,)),
            ("g2", (8,)), ("b2", (8,)), ("L1W", (H, A)), ("L1b", (H,)), ("g3", (H,)), ("b3", (H,)), ("L2W", (O, H)),
            ("L2b", (O,))]


def init_params(channels, size, rng):
    """NN_UTILS.initializeWeights(DECODER) (utils/nn_utils.lua:8-29): every module's weight ~ N(0, 1) * 0.005 and bias
    ~ N(0, 1) * 0.001, BatchNorm's gamma / beta included."""
    parts = [rng.standard_normal(int(np.prod(shape))) * (0.005 if name[-1] == "W" or name[0] == "g" else 0.001)
             for name, shape in layout(channels, size)]
    return np.concatenate(parts).astype(np.float32)


class Denoiser:
    """AE1 and AE2 of train_denoiser.lua at images [C][S][S], S = --scale (16 or 32), C = the context's channels."""

    def __init__(self, ctx, size=16):
        self.ctx, self.lib, self.C, self.S = ctx, ctx.lib, ctx.C, int(size)
        h = C.c_void_p()
        _check(self.lib.fg_dn_create(ctx.h, self.S, C.byref(h)), "fg_dn_create")
        self.h = h
        self.n = param_count(self.C, self.S)
        self.mps = mask_per_sample(self.S)

    def close(self):
        if self.h:
            self.lib.fg_dn_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h:
                self.close()
        except Exception:
            pass

    def _call(self, name, *args):
        _check(getattr(self.lib, name)(self.h, *args), name)

    def _sized(self, what, a, n):
        a = f32(a)
        if a.size != n:
            raise FGError("denoiser %s: expected %d floats, got %d" % (what, n, a.size))
        return a

    def _images(self, what, x):
        x = f32(x)
        if x.ndim != 4 or x.shape[1:] != (self.C, self.S, self.S):
            raise FGError("denoiser %s: expected [B][%d][%d][%d] images, got %s" % (what, self.C, self.S, self.S, x.shape))
        return x

    # ---- state ----
    def set_params(self, net, p):
        self._call("fg_dn_set_params", net, _ptr(self._sized("set_params", p, self.n)))

    def get_params(self, net):
        out = np.empty(self.n, np.float32)
        self._call("fg_dn_get_params", net, _ptr(out))
        return out

    def get_grads(self, net):
        out = np.empty(self.n, np.float32)
        self._call("fg_dn_get_grads", net, _ptr(out))
        return out

    def zero_grads(self, net):
        self._call("fg_dn_zero_grads", net)

    def set_bn_state(self, net, s):
        self._call("fg_dn_set_bn_state", net, _ptr(self._sized("set_bn_state", s, BN_STATE)))

    def get_bn_state(self, net):
        out = np.empty(BN_STATE, np.float32)
        self._call("fg_dn_get_bn_state", net, _ptr(out))
        return out

    def set_adam_state(self, m, v, t):
        m = None if m is None else self._sized("set_adam_state m", m, self.n)
        v = None if v is None else self._sized("set_adam_state v", v, self.n)
        self._call("fg_dn_set_adam_state", _ptr(m), _ptr(v), int(t))

    def get_adam_state(self):
        m, v, t = np.empty(self.n, np.float32), np.empty(self.n, np.float32), C.c_int(0)
        self._call("fg_dn_get_adam_state", _ptr(m), _ptr(v), C.byref(t))
        return m, v, t.value

    # ---- L-net ----
    def forward(self, net, x, training=True, noise=None, masks=None, seed=0):
        x = self._images("forward", x)
        B = x.shape[0]
        noise = None if noise is None else self._sized("forward noise", noise, x.size)
        masks = None if masks is None else self._sized("forward masks", masks, B * self.mps)
        out = np.empty_like(x)
        self._call("fg_dn_forward", net, _ptr(x), B, int(training), _ptr(noise), _ptr(masks), seed, _ptr(out))
        return out

    def backward(self, net, dout):
        self._call("fg_dn_backward", net, _ptr(f32(dout)))

    # ---- L-step ----
    def train_step(self, hyper, images, noise=None, masks=None, seed=0, B=None):
        """images: [B][C][S][S] numpy array, or a raw device address with B given; noise [2][B][C][S][S] and masks
        [3][B][mps] or None (drawn from seed).  Returns {loss_AE1, loss_AE2, t}."""
        if isinstance(images, np.ndarray):
            images = self._images("train_step", images)
            B = images.shape[0]
        if noise is not None:
            noise = self._sized("train_step noise", noise, 2 * B * self.C * self.S * self.S)
        if masks is not None:
            masks = self._sized("train_step masks", masks, 3 * B * self.mps)
        st = DnStats()
        self._call("fg_dn_train_step", C.byref(hyper), B, _ptr(images), _ptr(noise), _ptr(masks), seed, C.byref(st))
        return dict(loss_AE1=st.loss_AE1, loss_AE2=st.loss_AE2, t=st.t)

    def denoise(self, images, chunk=None):
        """train.lua --denoise (nn_utils.lua:144-155): AE1_DECODER:evaluate():forward(images)."""
        images = self._images("denoise", images)
        out = np.empty_like(images)
        chunk = chunk or self.ctx.max_batch
        self._call("fg_dn_denoise", _ptr(images), images.shape[0], int(chunk), _ptr(out))
        return out

    def debug_tensor(self, name):
        """what the last forwards drew: "noise0", "noise1", "masks0".."masks2" (tests)"""
        fn = self.lib.fg_dn_debug_tensor
        n = fn(self.h, name.encode(), None, 0)
        if n < 0:
            raise FGError("fg_dn_debug_tensor(%s): %s" % (name, self.lib.fg_last_error().decode()))
        out = np.empty(n, np.float32)
        if fn(self.h, name.encode(), _ptr(out), n) < 0:
            raise FGError("fg_dn_debug_tensor(%s) failed" % name)
        return out


def train(dn, dataset, hyper, batch_size=128, epochs=1, rng=None, seed=0, log=print):
    """train_denoiser.lua train() (:230-370) on a DeviceDataset: per epoch a random permutation of the training set
    (torch.randperm), batches of batch_size with a ragged last batch, each gathered at --scale on the device
    (fg_dataset_gather_sized) and trained by one fg_dn_train_step.  Returns the per-epoch mean losses (AE1, AE2) the
    script prints: sum of batch losses / (N / batchSize)."""
    rng = rng or np.random.default_rng(seed)
    N, ctx = dataset.size(), dn.ctx
    if batch_size > ctx.max_batch:
        raise FGError("batch_size %d exceeds the context's max_batch %d" % (batch_size, ctx.max_batch))
    buf = ctx.lib.fg_dev_alloc(batch_size * dn.C * dn.S * dn.S * 4)
    if not buf:
        raise FGError("fg_dev_alloc failed")
    history, step = [], 0
    try:
        for epoch in range(epochs):
            shuffle = rng.permutation(N).astype(np.int32)
            s1 = s2 = 0.0
            for t in range(0, N, batch_size):
                idx = np.ascontiguousarray(shuffle[t:t + batch_size])
                B = idx.size
                if B < 2:  # BatchNorm needs two samples; torch would fail on such a batch as well
                    continue
                _check(ctx.lib.fg_dataset_gather_sized(dataset.h, idx.ctypes.data_as(C.c_void_p), B, dn.S, C.c_void_p(buf)),
                       "fg_dataset_gather_sized")
                st = dn.train_step(hyper, buf, seed=(seed << 32) + step, B=B)
                s1 += st["loss_AE1"]
                s2 += st["loss_AE2"]
                step += 1
            l1, l2 = s1 / (N / batch_size), s2 / (N / batch_size)
            if log:
                log("<trainer> epoch %d: loss AE1 = %.4f, loss AE2 = %.4f" % (epoch + 1, l1, l2))
            history.append((l1, l2))
    finally:
        ctx.lib.fg_dev_free(buf)
    return history
