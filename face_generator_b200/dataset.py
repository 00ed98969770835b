"""Host-side mirror of dataset.lua for the device-resident path: decoded uint8 images live on the GPU, the batch
(`inputs[i] = dataset[math.random(dataset:size())]`, adversarial.lua:244-249) is assembled by one kernel.

    ds = DeviceDataset(ctx, images_u8)            # [N][Cs][Hs][Ws] uint8, e.g. the 64x64 faces of dataset.lua:10
    real = ds.gather(indices)                     # == image.scale(image.load(...), 32, 32) for those images
    real16 = ds.gather(indices, 16)               # the same at 16x16 (train.lua --scale 16)
    fine, coarse, diff = ds.gather_c2f(indices, 16)   # dataset_c2f.lua _toResult (train_c2f.lua --coarseSize 16)
    stats = ds.train_step(hyper, B, seed)         # adversarial.lua loop body with no host->device traffic
    stats = ds.train_step_iters(hyper, B, 2, 1, seed)          # --D_iterations 2: two D iterations, one G iteration
    S16(ctx).train_step_dataset(ds, hyper, B, seed)            # the same for the --scale 16 nets
    C2f(ctx).train_step_dataset(ds, hyper, B, 16, seed)        # and for the coarse-to-fine nets
    C2f(ctx, 64).train_step_dataset(ds, hyper, B, 32, seed)    # the pyramid level 32x32 -> 64x64 (--fineSize 64)
"""
import ctypes as C

import numpy as np

from .lib import Context, StepStats, _check, _stats, check_iters


class DeviceDataset:
    def __init__(self, ctx: Context, images_u8, chunk=8192):
        images_u8 = np.ascontiguousarray(images_u8, np.uint8)
        assert images_u8.ndim == 4, "[N][Cs][Hs][Ws] uint8"
        N, Cs, Hs, Ws = images_u8.shape
        self.ctx, self.lib, self.N = ctx, ctx.lib, N
        h = C.c_void_p()
        _check(self.lib.fg_dataset_create(ctx.h, N, Cs, Hs, Ws, C.byref(h)), "fg_dataset_create")
        self.h = h
        for s in range(0, N, chunk):  # dataset.loadImages(startAt, count) granularity
            part = images_u8[s:s + chunk]
            _check(self.lib.fg_dataset_upload(self.h, s, part.shape[0], part.ctypes.data_as(C.c_void_p)), "fg_dataset_upload")

    def close(self):
        if self.h:
            self.lib.fg_dataset_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h:
                self.close()
        except Exception:
            pass

    def size(self):
        return int(self.lib.fg_dataset_size(self.h))

    def gather(self, indices, size=32):
        """image.scale(image.load(...), size, size) of those images (dataset.lua setScale(size)), [B][C][size][size]."""
        idx = np.ascontiguousarray(indices, np.int32)
        out = np.empty((idx.size, self.ctx.C, size, size), np.float32)
        _check(self.lib.fg_dataset_gather_sized(self.h, idx.ctypes.data_as(C.c_void_p), idx.size, size,
                                                out.ctypes.data_as(C.c_void_p)), "fg_dataset_gather_sized")
        return out

    def gather_c2f(self, indices, coarse_size, fine_size=32):
        """dataset_c2f.lua _toResult of those images at fineSize S = fine_size (16, 32 or 64): (fine, coarse, diff),
        each [B][C][S][S]."""
        idx = np.ascontiguousarray(indices, np.int32)
        S = fine_size
        fine, coarse, diff = (np.empty((idx.size, self.ctx.C, S, S), np.float32) for _ in range(3))
        _check(self.lib.fg_dataset_gather_c2f_sized(self.h, idx.ctypes.data_as(C.c_void_p), idx.size, S, coarse_size,
                                                    fine.ctypes.data_as(C.c_void_p), coarse.ctypes.data_as(C.c_void_p),
                                                    diff.ctypes.data_as(C.c_void_p)), "fg_dataset_gather_c2f_sized")
        return fine, coarse, diff

    def draw(self, seed, B):
        idx = np.empty(B, np.int32)
        _check(self.lib.fg_dataset_draw(self.h, seed, B, idx.ctypes.data_as(C.c_void_p)), "fg_dataset_draw")
        return idx

    def train_step(self, hyper, B, seed, want_stats=True):
        st = StepStats() if want_stats else None
        _check(self.lib.fg_train_step_dataset(self.ctx.h, self.h, C.byref(hyper), B, seed,
                                              C.byref(st) if st is not None else None), "fg_train_step_dataset")
        return _stats(st)

    def train_step_iters(self, hyper, B, D_iterations, G_iterations, seed, want_stats=True):
        """D_iterations D iterations + G_iterations G iterations of the 32x32 nets in one call, every input drawn on
        the device inside the step (fg_train_step_dataset_iters; the streams are in fg_b200.h)."""
        d, g = check_iters(D_iterations, G_iterations)
        st = StepStats() if want_stats else None
        _check(self.lib.fg_train_step_dataset_iters(self.ctx.h, self.h, C.byref(hyper), B, d, g, seed,
                                                    C.byref(st) if st is not None else None), "fg_train_step_dataset_iters")
        return _stats(st)


def noise_uniform(ctx: Context, seed, shape):
    """NN_UTILS.createNoiseInputs drawn on the device (the stream fg_train_step_dataset uses)."""
    out = np.empty(shape, np.float32)
    _check(ctx.lib.fg_noise_uniform(ctx.h, seed, out.size, out.ctypes.data_as(C.c_void_p)), "fg_noise_uniform")
    return out
