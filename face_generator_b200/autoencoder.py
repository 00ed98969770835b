"""The autoencoder of train_autoencoder.lua on the GPU (fg_ae_* entry points), and the host side of its epoch loop.
Mirrors face_generator_b200/lua/autoencoder_b200.lua.

    ae = Autoencoder(ctx, 32, 256)            # grayscale 32x32, --noiseDim 256; ctx has 1 channel
    ae.set_params(init_params(32, 256, rng))
    st = ae.train_step(hyper, images)         # fevalAE + optim.adam on one batch
    code = ae.encode(images)                  # the Tanh output, [N][256]
    out = ae.reconstruct(images)              # MODEL_AE:evaluate():forward(images)
"""
import ctypes as C

import numpy as np

from .lib import AeHyper, AeStats, FGError, _check, _ptr, f32, load_library

H1, H3 = 512, 256  # the two hidden widths of the script


def ae_hyper_default(**kw):
    """lr 1e-3, betas 0.9 / 0.999, eps 1e-8 (optim.adam with an empty config), L1 = L2 = 0 (--coefL1 / --coefL2),
    p_drop 0.5 (train_autoencoder.lua:87, :129-134).  --learningRate and --momentum only reach the script's unused sgd table."""
    h = AeHyper()
    load_library().fg_ae_hyper_default(C.byref(h))
    for k, v in kw.items():
        if not hasattr(h, k):
            raise KeyError(k)
        setattr(h, k, v)
    return h


def param_count(size, noise_dim):
    return int(load_library().fg_ae_param_count(size, noise_dim))


def layout(size, noise_dim):
    """getParameters() order: [(name, shape)] of the four Linear layers, weights [out][in]"""
    I, d = size * size, noise_dim
    return [("L1W", (H1, I)), ("L1b", (H1,)), ("L2W", (d, H1)), ("L2b", (d,)), ("L3W", (H3, d)), ("L3b", (H3,)),
            ("L4W", (I, H3)), ("L4b", (I,))]


def init_params(size, noise_dim, rng):
    """initializeWeights(MODEL_AE) (train_autoencoder.lua:66-78): weights ~ N(0, 1) * 0.005, biases ~ N(0, 1) * 0.001"""
    parts = [rng.standard_normal(int(np.prod(shape))) * (0.005 if name[-1] == "W" else 0.001)
             for name, shape in layout(size, noise_dim)]
    return np.concatenate(parts).astype(np.float32)


class Autoencoder:
    """MODEL_AE of train_autoencoder.lua at images [1][S][S], S = --scale (16 or 32), code width d = --noiseDim."""

    def __init__(self, ctx, size=32, noise_dim=256):
        self.ctx, self.lib, self.S, self.d = ctx, ctx.lib, int(size), int(noise_dim)
        h = C.c_void_p()
        _check(self.lib.fg_ae_create(ctx.h, self.S, self.d, C.byref(h)), "fg_ae_create")
        self.h = h
        self.I = self.S * self.S
        self.n = param_count(self.S, self.d)

    def close(self):
        if self.h:
            self.lib.fg_ae_destroy(self.h)
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
            raise FGError("autoencoder %s: expected %d floats, got %d" % (what, n, a.size))
        return a

    def _images(self, what, x):
        x = f32(x)
        if x.ndim != 4 or x.shape[1:] != (1, self.S, self.S):
            raise FGError("autoencoder %s: expected [B][1][%d][%d] images, got %s" % (what, self.S, self.S, x.shape))
        return x

    # ---- state ----
    def set_params(self, p):
        self._call("fg_ae_set_params", _ptr(self._sized("set_params", p, self.n)))

    def _vec(self, name):
        out = np.empty(self.n, np.float32)
        self._call(name, _ptr(out))
        return out

    def get_params(self):
        return self._vec("fg_ae_get_params")

    def get_grads(self):
        return self._vec("fg_ae_get_grads")

    def zero_grads(self):
        self._call("fg_ae_zero_grads")

    def set_adam_state(self, m, v, t):
        m = None if m is None else self._sized("set_adam_state m", m, self.n)
        v = None if v is None else self._sized("set_adam_state v", v, self.n)
        self._call("fg_ae_set_adam_state", _ptr(m), _ptr(v), int(t))

    def get_adam_state(self):
        m, v, t = np.empty(self.n, np.float32), np.empty(self.n, np.float32), C.c_int(0)
        self._call("fg_ae_get_adam_state", _ptr(m), _ptr(v), C.byref(t))
        return m, v, t.value

    # ---- L-net ----
    def forward(self, x, training=True, masks=None, seed=0):
        """-> (code [B][d], out [B][1][S][S]); masks: [B][d] keep flags or None (drawn from seed)"""
        x = self._images("forward", x)
        B = x.shape[0]
        masks = None if masks is None else self._sized("forward masks", masks, B * self.d)
        code, out = np.empty((B, self.d), np.float32), np.empty_like(x)
        self._call("fg_ae_forward", _ptr(x), B, int(training), _ptr(masks), seed, _ptr(code), _ptr(out))
        return code, out

    def backward(self, dout):
        self._call("fg_ae_backward", _ptr(f32(dout)))

    # ---- L-step ----
    def train_step(self, hyper, images, masks=None, seed=0, B=None, sync=True):
        """images: [B][1][S][S] numpy array, or a raw device address with B given; masks [B][d] or None (drawn from
        seed).  Returns {loss, t}, or None without waiting for the GPU when sync is False."""
        if isinstance(images, np.ndarray):
            images = self._images("train_step", images)
            B = images.shape[0]
        if masks is not None:
            masks = self._sized("train_step masks", masks, B * self.d)
        st = AeStats()
        self._call("fg_ae_train_step", C.byref(hyper), B, _ptr(images), _ptr(masks), seed, C.byref(st) if sync else None)
        return dict(loss=st.loss, t=st.t) if sync else None

    def train_step_dataset(self, dataset, hyper, idx, seed=0, sync=True):
        """one step on images idx (int32 array) of a DeviceDataset, gathered at S x S on the device"""
        idx = np.ascontiguousarray(idx, np.int32)
        st = AeStats()
        self._call("fg_ae_train_step_dataset", dataset.h, C.byref(hyper), idx.ctypes.data_as(C.c_void_p), idx.size, seed,
                   C.byref(st) if sync else None)
        return dict(loss=st.loss, t=st.t) if sync else None

    def reconstruct(self, images, chunk=None, training=False, seed=0):
        """MODEL_AE:forward(images) chunk by chunk.  training=True keeps Dropout live as the script's getSamples does
        (:137-145 never calls evaluate()); chunk k then draws its keep flags from seed + k."""
        images = self._images("reconstruct", images)
        out = np.empty_like(images)
        self._call("fg_ae_reconstruct", _ptr(images), images.shape[0], int(chunk or self.ctx.max_batch), int(training), seed,
                   _ptr(out))
        return out

    def encode(self, images, chunk=None):
        """the encoder half in evaluation mode: Tanh(Linear(ReLU(Linear(images)))), [N][d]"""
        images = self._images("encode", images)
        chunk = int(chunk or self.ctx.max_batch)
        out = np.empty((images.shape[0], self.d), np.float32)
        for s in range(0, images.shape[0], chunk):
            b = min(chunk, images.shape[0] - s)
            self._call("fg_ae_forward", _ptr(images[s:s + b]), b, 0, None, 0, _ptr(out[s:s + b]), None)
        return out

    def debug_tensor(self, name):
        """x z1 h1 z2 code h2 z3 h3 z4 y masks of the last forward, dz4 dz3 dz2 dz1 of the last backward (tests)"""
        fn = self.lib.fg_ae_debug_tensor
        n = fn(self.h, name.encode(), None, 0)
        if n < 0:
            raise FGError("fg_ae_debug_tensor(%s): %s" % (name, self.lib.fg_last_error().decode()))
        out = np.empty(n, np.float32)
        if fn(self.h, name.encode(), _ptr(out), n) < 0:
            raise FGError("fg_ae_debug_tensor(%s) failed" % name)
        return out


def epoch_batches(N, batch_size, rng):
    """train_autoencoder.lua:153-167: a random permutation cut into batches, the last one whatever is left"""
    shuffle = rng.permutation(N).astype(np.int32)
    return [np.ascontiguousarray(shuffle[t:t + batch_size]) for t in range(0, N, batch_size)]


def train(ae, dataset, hyper, batch_size=128, epochs=1, seed=0, log=print):
    """train() of train_autoencoder.lua (:148-239) on a DeviceDataset.  Per epoch: a permutation from
    np.random.default_rng(seed), every batch one fg_ae_train_step_dataset with step seed (seed << 32) + step, none of
    which waits for the GPU; the losses are read once the epoch is enqueued.  Returns the mean batch loss per epoch."""
    rng = np.random.default_rng(seed)
    N, ctx = dataset.size(), ae.ctx
    if batch_size > ctx.max_batch:
        raise FGError("batch_size %d exceeds the context's max_batch %d" % (batch_size, ctx.max_batch))
    history, step = [], 0
    for epoch in range(epochs):
        batches = epoch_batches(N, batch_size, rng)
        losses = ctx.lib.fg_dev_alloc(4 * len(batches))
        if not losses:
            raise FGError("fg_dev_alloc failed")
        try:
            for k, idx in enumerate(batches):
                ae.train_step_dataset(dataset, hyper, idx, seed=(seed << 32) + step, sync=False)
                step += 1
                # the step's loss stays on the device until the epoch is enqueued
                n = ae.lib.fg_ae_debug_tensor(ae.h, b"loss", C.c_void_p(losses + 4 * k), 1)
                if n != 1:
                    raise FGError("fg_ae_debug_tensor(loss): %s" % ae.lib.fg_last_error().decode())
            host = np.empty(len(batches), np.float32)
            _check(ctx.lib.fg_memcpy(ctx.h, _ptr(host), C.c_void_p(losses), host.nbytes), "fg_memcpy")
            _check(ctx.lib.fg_sync(ctx.h), "fg_sync")
        finally:
            ctx.lib.fg_dev_free(losses)
        mean = float(host.astype(np.float64).mean())
        if log:
            log("<trainer> epoch %d: loss = %.4f" % (epoch + 1, mean))
        history.append(mean)
    return history
