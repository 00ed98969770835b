"""Host-side mirror of dataset.lua for the device-resident path: decoded uint8 images live on the GPU, the batch
(`inputs[i] = dataset[math.random(dataset:size())]`, adversarial.lua:244-249) is assembled by one kernel.

    ds = DeviceDataset(ctx, images_u8)            # [N][Cs][Hs][Ws] uint8, e.g. the 64x64 faces of dataset.lua:10
    real = ds.gather(indices)                     # == image.scale(image.load(...), 32, 32) for those images
    real16 = ds.gather(indices, 16)               # the same at 16x16 (train.lua --scale 16)
    fine, coarse, diff = ds.gather_c2f(indices, 16)   # dataset_c2f.lua _toResult (train_c2f.lua --coarseSize 16)
    ds = DeviceDataset.from_dirs(ctx, ["faces/"])  # dataset.loadImagesFromDirs: .jpg files decoded on the GPU
    ds = DeviceDataset.from_lfw(ctx, ["lfw/"])     # generate_dataset.py's out_aug_64x64, built on the GPU from LFW
    ds = DeviceDataset.from_lfw(ctx, ["lfw/"], jpeg_quality=75)  # ... as its quality-75 .jpg files decode
    ds.save_jpeg("out_aug_64x64/")                # and those files themselves, {i:06}_{a:03}.jpg, encoded on the GPU
    stats = ds.train_step(hyper, B, seed)         # adversarial.lua loop body with no host->device traffic
    stats = ds.train_step_iters(hyper, B, 2, 1, seed)          # --D_iterations 2: two D iterations, one G iteration
    S16(ctx).train_step_dataset(ds, hyper, B, seed)            # the same for the --scale 16 nets
    C2f(ctx).train_step_dataset(ds, hyper, B, 16, seed)        # and for the coarse-to-fine nets
    C2f(ctx, 64).train_step_dataset(ds, hyper, B, 32, seed)    # the pyramid level 32x32 -> 64x64 (--fineSize 64)
"""
import ctypes as C
import os

import numpy as np

from .lib import Context, FGError, StepStats, _check, _stats, check_iters, load_library


def list_image_files(dirs, ext="jpg", start_at=1, count=None):
    """dataset.lua:156-190 loadImagesFromDirs' file list: the files of each directory whose name ends in `ext`, in the
    order the directories are given, sorted by full path (byte order, as Lua's `<` on strings), then the 1-based
    range [start_at, start_at + count)."""
    files = []
    for d in dirs:
        files += [os.path.join(d, f) for f in os.listdir(d) if f.endswith(ext)]
        if not files:
            raise FileNotFoundError("given directory doesnt contain any files of type: " + ext)
    files.sort(key=os.fsencode)
    end = len(files) if count is None else min(start_at + count - 1, len(files))
    return files[start_at - 1:end]


def list_lfw_files(dirs):
    """dataset/generate_dataset.py's walk: the files of each given directory and of its direct subdirectories whose
    name matches `.jpg$`, sorted by full path in byte order (as list_image_files).  The reference took the files in
    the order of a set() of directories and os.listdir, which is unspecified; sorting makes the row order, and with
    it every augmentation drawn for a photo, reproducible."""
    files = []
    for d in dirs:
        subs = [d] + sorted(os.path.join(d, s) for s in os.listdir(d) if os.path.isdir(os.path.join(d, s)))
        for sd in subs:
            files += [os.path.join(sd, f) for f in os.listdir(sd)
                      if f.endswith(".jpg") and os.path.isfile(os.path.join(sd, f))]
    files = sorted(set(files), key=os.fsencode)
    return files


# fg_aug (include/fg_b200.h)
AUG_DTYPE = np.dtype([("src", "<i8"), ("warp", "<i4"), ("hflip", "<i4"), ("brightness", "<f8"), ("m", "<f8", (9,))])


def lfw_aug_params(seed, first_src, n_src, n_aug, src_h, src_w):
    """fg_lfw_aug_params (host only): the n_src * (1 + n_aug) descriptors of photos [first_src, first_src + n_src),
    photo-major, as an AUG_DTYPE array; src is the global photo index."""
    out = np.zeros(n_src * (1 + n_aug), AUG_DTYPE)
    lib = load_library()
    _check(lib.fg_lfw_aug_params(seed, first_src, n_src, n_aug, src_h, src_w, out.ctypes.data_as(C.c_void_p)),
           "fg_lfw_aug_params")
    return out


def read_pgm(data):
    """Binary (P5) 8-bit PGM bytes -> [1][H][W] uint8 (train_autoencoder.lua's lfwcrop_grey set)."""
    fields, p = [], 2
    if data[:2] != b"P5":
        raise ValueError("not a binary PGM (P5) file")
    while len(fields) < 3:
        while p < len(data) and data[p:p + 1].isspace():
            p += 1
        if data[p:p + 1] == b"#":
            while p < len(data) and data[p:p + 1] not in (b"\n", b"\r"):
                p += 1
            continue
        q = p
        while q < len(data) and not data[q:q + 1].isspace():
            q += 1
        if q == p:
            raise ValueError("truncated PGM header")
        fields.append(int(data[p:q]))
        p = q
    W, H, maxval = fields
    if not 0 < maxval < 256:
        raise ValueError("PGM maxval %d: only 8-bit PGM is supported" % maxval)
    p += 1  # the single whitespace byte after maxval
    if len(data) < p + W * H:
        raise ValueError("truncated PGM data")
    return np.frombuffer(data, np.uint8, W * H, p).reshape(1, H, W)


def jpeg_info(data):
    """(C, H, W) of JPEG bytes from their markers (fg_jpeg_info; host only)."""
    lib = load_library()
    c, h, w = C.c_int(), C.c_int(), C.c_int()
    buf = np.frombuffer(data, np.uint8)
    _check(lib.fg_jpeg_info(buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(c), C.byref(h), C.byref(w)), "fg_jpeg_info")
    return c.value, h.value, w.value


class DeviceDataset:
    def __init__(self, ctx: Context, images_u8=None, chunk=8192, shape=None):
        """From decoded images [N][Cs][Hs][Ws] uint8, or an empty cache of `shape` = (N, Cs, Hs, Ws) to fill with
        upload / upload_jpeg."""
        if images_u8 is not None:
            images_u8 = np.ascontiguousarray(images_u8, np.uint8)
            assert images_u8.ndim == 4, "[N][Cs][Hs][Ws] uint8"
            shape = images_u8.shape
        N, Cs, Hs, Ws = shape
        self.ctx, self.lib, self.N = ctx, ctx.lib, N
        self.shape = (N, Cs, Hs, Ws)
        h = C.c_void_p()
        _check(self.lib.fg_dataset_create(ctx.h, N, Cs, Hs, Ws, C.byref(h)), "fg_dataset_create")
        self.h = h
        if images_u8 is not None:
            for s in range(0, N, chunk):  # dataset.loadImages(startAt, count) granularity
                self.upload(s, images_u8[s:s + chunk])

    @classmethod
    def from_dirs(cls, ctx: Context, dirs, ext="jpg", start_at=1, count=None, channels=None, chunk=16384):
        """dataset.loadImagesFromDirs(dirs, ext, startAt, count, doSort = true) into a device cache at the files'
        own size (image.load(path, nbChannels, 'byte')): the cache is sized from the first file, every file must
        match it.  JPEG files are decoded on the GPU, `chunk` files per call; ext "pgm" reads binary PGM on the host
        (nothing to decode).  channels = the cache's Cs: default 3 for colour JPEG files (a 1-channel context then
        gathers image.rgb2y of them), else the context's channel count."""
        files = list_image_files(dirs, ext, start_at, count)
        if not files:
            raise FileNotFoundError("no %s files in the requested range" % ext)
        pgm = ext.lower().endswith("pgm")
        with open(files[0], "rb") as f:
            head = f.read()
        C0, Hs, Ws = read_pgm(head).shape if pgm else jpeg_info(head)
        Cs = channels if channels is not None else (3 if C0 == 3 else ctx.C)
        ds = cls(ctx, shape=(len(files), Cs, Hs, Ws))
        try:
            for s in range(0, len(files), chunk):
                blobs = []
                for fn in files[s:s + chunk]:
                    with open(fn, "rb") as f:
                        blobs.append(f.read())
                if pgm:
                    imgs = np.stack([read_pgm(b) for b in blobs])
                    if imgs.shape[2:] != (Hs, Ws):
                        raise ValueError("PGM files of different sizes in %s" % dirs)
                    ds.upload(s, np.repeat(imgs, Cs, axis=1) if Cs == 3 else imgs)
                else:
                    try:
                        ds.upload_jpeg(s, blobs)
                    except FGError as e:
                        raise FGError("%s (%s)" % (e, files[s + e.index] if e.index is not None else dirs)) from None
        except Exception:
            ds.close()
            raise
        return ds

    @classmethod
    def from_lfw(cls, ctx: Context, dirs, augmentations=19, seed=43, size=64, chunk=2048, jpeg_quality=None):
        """dataset/generate_dataset.py on the GPU: the augmented LFW training set (out_aug_64x64 with the defaults,
        out_unaug_64x64 with augmentations=0) straight into a device cache of len(files) * (1 + augmentations) rows,
        3 planes (a 1-channel context gathers image.rgb2y of them), size x size.  Row i * (1 + augmentations) + a is
        augmentation a of photo i of list_lfw_files(dirs), a = 0 the photo itself: the order of the reference's file
        names {i:06}_{a:03}.jpg.  The photos are decoded on the GPU `chunk` at a time into a scratch cache that the
        chunk's rows are built from (fg_dataset_upload_jpeg, fg_dataset_augment); the descriptors come from
        fg_lfw_aug_params(seed), so the result does not depend on `chunk`.  jpeg_quality = q (75 for the reference's
        misc.imsave) then passes every row through jpeg_roundtrip(q): the rows are what the reference's files decode
        to.  save_jpeg writes those files."""
        files = list_lfw_files(dirs)
        if not files:
            raise FileNotFoundError("no .jpg files in %s or their direct subdirectories" % (dirs,))
        with open(files[0], "rb") as f:
            _, Hs, Ws = jpeg_info(f.read())
        per = 1 + augmentations
        ds = cls(ctx, shape=(len(files) * per, 3, size, size))
        ds.per = per
        try:
            for s in range(0, len(files), chunk):
                blobs = []
                for fn in files[s:s + chunk]:
                    with open(fn, "rb") as f:
                        blobs.append(f.read())
                scratch = cls(ctx, shape=(len(blobs), 3, Hs, Ws))
                try:
                    try:
                        scratch.upload_jpeg(0, blobs)
                    except FGError as e:
                        raise FGError("%s (%s)" % (e, files[s + e.index] if e.index is not None else dirs)) from None
                    augs = lfw_aug_params(seed, s, len(blobs), augmentations, Hs, Ws)
                    augs["src"] -= s  # rows of the scratch cache
                    ds.augment(scratch, s * per, augs)
                finally:
                    scratch.close()
            if jpeg_quality is not None:
                ds.jpeg_roundtrip(quality=jpeg_quality)
        except Exception:
            ds.close()
            raise
        return ds

    def augment(self, src, first, augs):
        """fg_dataset_augment: rows [first, first + len(augs)) of this cache from rows of `src` (a cache on the same
        context), one AUG_DTYPE descriptor per row."""
        a = np.ascontiguousarray(augs, AUG_DTYPE)
        _check(self.lib.fg_dataset_augment(src.h, self.h, first, a.ctypes.data_as(C.c_void_p), a.size),
               "fg_dataset_augment")

    def upload(self, first, images_u8):
        """fg_dataset_upload: decoded images [n][Cs][Hs][Ws] uint8 into rows [first, first + n)."""
        a = np.ascontiguousarray(images_u8, np.uint8)
        _check(self.lib.fg_dataset_upload(self.h, first, a.shape[0], a.ctypes.data_as(C.c_void_p)), "fg_dataset_upload")

    def upload_jpeg(self, first, files):
        """fg_dataset_upload_jpeg: a list of JPEG files (bytes) decoded on the GPU into rows [first, first + n).
        On failure the FGError carries .index, the position in `files` of the first failing file."""
        offsets = np.zeros(len(files) + 1, np.int64)
        offsets[1:] = np.cumsum([len(b) for b in files])
        data = np.frombuffer(b"".join(files), np.uint8) if offsets[-1] else np.zeros(1, np.uint8)
        failed = C.c_int64(-1)
        rc = self.lib.fg_dataset_upload_jpeg(self.h, first, len(files), data.ctypes.data_as(C.c_void_p),
                                             offsets.ctypes.data_as(C.c_void_p), C.byref(failed))
        if rc != 0:
            err = FGError("fg_dataset_upload_jpeg failed (%d): %s" % (rc, self.lib.fg_last_error().decode()))
            err.rc, err.index = rc, (failed.value if failed.value >= 0 else None)
            raise err

    def encode_jpeg(self, first=0, count=None, quality=75):
        """fg_dataset_encode_jpeg: rows [first, first + count) as JPEG files (list of bytes), byte for byte what
        Pillow's Image.save(f, "JPEG", quality=quality) writes (3 planes: YCbCr 4:2:0, 1 plane: grayscale).  The
        output buffer is sized from a guess first and, when that is short, once more from the sizes reported."""
        count = self.N - first if count is None else count
        offsets = np.zeros(count + 1, np.int64)
        _, Cs, Hs, Ws = self.shape
        cap = count * (700 + Cs * Hs * Ws // 2)
        for attempt in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            rc = self.lib.fg_dataset_encode_jpeg(self.h, first, count, quality, out.ctypes.data_as(C.c_void_p), cap,
                                                 offsets.ctypes.data_as(C.c_void_p))
            if rc == 0:
                break
            if attempt or offsets[-1] <= cap:
                _check(rc, "fg_dataset_encode_jpeg")
            cap = int(offsets[-1])
        data = out.tobytes()
        return [data[offsets[i]:offsets[i + 1]] for i in range(count)]

    def jpeg_roundtrip(self, first=0, count=None, quality=75):
        """fg_dataset_jpeg_roundtrip: rows [first, first + count) replaced in place by what upload_jpeg gives on
        encode_jpeg's files, without leaving the device."""
        count = self.N - first if count is None else count
        _check(self.lib.fg_dataset_jpeg_roundtrip(self.h, first, count, quality), "fg_dataset_jpeg_roundtrip")

    def save_jpeg(self, directory, quality=75, names=None, per=None, chunk=16384):
        """Every row as a JPEG file in `directory` (created if missing), encoded on the GPU `chunk` rows at a time.
        names: one file name per row; by default generate_dataset.py's {i:06}_{a:03}.jpg for a cache of `per` rows
        per photo (row i * per + a), `per` defaulting to the 1 + augmentations of from_lfw, else 1."""
        per = per or getattr(self, "per", 1)
        if names is None:
            names = ["%06d_%03d.jpg" % (r // per, r % per) for r in range(self.N)]
        if len(names) != self.N:
            raise ValueError("%d names for %d rows" % (len(names), self.N))
        os.makedirs(directory, exist_ok=True)
        for s in range(0, self.N, chunk):
            for name, b in zip(names[s:s + chunk], self.encode_jpeg(s, min(chunk, self.N - s), quality)):
                with open(os.path.join(directory, name), "wb") as f:
                    f.write(b)

    def download(self, first=0, count=None):
        """fg_dataset_download: rows [first, first + count) of the cache, [count][Cs][Hs][Ws] uint8."""
        count = self.N - first if count is None else count
        out = np.empty((count,) + self.shape[1:], np.uint8)
        _check(self.lib.fg_dataset_download(self.h, first, count, out.ctypes.data_as(C.c_void_p)), "fg_dataset_download")
        return out

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
