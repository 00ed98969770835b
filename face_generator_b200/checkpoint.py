"""Torch7 checkpoint files (`torch.save` binary format) through the C ABI's fg_t7_* entry points.

Reading: the reference's `adversarial.net` = {D = MODEL_D, G = MODEL_G, opt = OPT, epoch = EPOCH}
(adversarial.lua:328, adversarial_c2f.lua:216; consumed by sample.lua:251-258 and train.lua:104-124).
Writing: flat float tensors + numbers + strings in one root table, readable with stock `torch.load`
(parameters, Adam moments and step counters -- the reference itself drops its optimizer state, train.lua:122).
Host-side only: nothing here touches the GPU.
"""
import ctypes as C

import numpy as np

from .lib import (FGError, NET_D, NET_G, c2f_disc_param_count, c2f_gen_param_count, disc_param_count,
                  load_library)

KINDS = {0: "nil", 1: "number", 2: "string", 3: "table", 4: "object", 5: "boolean", 6: "function", 16: "tensor",
         17: "storage", -1: None}


def _err(what):
    raise FGError("%s: %s" % (what, load_library().fg_last_error().decode()))


class T7File:
    def __init__(self, path):
        self.lib = load_library()
        h = C.c_void_p()
        if self.lib.fg_t7_open(str(path).encode(), C.byref(h)) != 0:
            _err("fg_t7_open")
        self.h = h

    def close(self):
        if self.h:
            self.lib.fg_t7_close(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def kind(self, path):
        return KINDS.get(int(self.lib.fg_t7_kind(self.h, path.encode())), "?")

    def number(self, path):
        v = C.c_double(0)
        if self.lib.fg_t7_number(self.h, path.encode(), C.byref(v)) != 0:
            _err("fg_t7_number(%s)" % path)
        return v.value

    def string(self, path):
        n = int(self.lib.fg_t7_string(self.h, path.encode(), None, 0))
        if n < 0:
            raise FGError("fg_t7_string(%s): not a string / object" % path)
        buf = C.create_string_buffer(n + 1)
        self.lib.fg_t7_string(self.h, path.encode(), buf, n + 1)
        return buf.value.decode()

    def tensor(self, path):
        dims = (C.c_int64 * 8)()
        n = int(self.lib.fg_t7_tensor(self.h, path.encode(), None, 0, dims))
        if n < 0:
            _err("fg_t7_tensor(%s)" % path)
        shape = [int(d) for d in dims if d > 0]
        out = np.empty(n, np.float32)
        if n and self.lib.fg_t7_tensor(self.h, path.encode(), out.ctypes.data_as(C.c_void_p), n, None) < 0:
            _err("fg_t7_tensor(%s)" % path)
        return out.reshape(shape) if n else out

    def _vec(self, fn, path):
        n = int(fn(self.h, path.encode(), None, 0))
        if n < 0:
            _err("%s(%s)" % (fn.__name__, path))
        out = np.empty(n, np.float32)
        if n and fn(self.h, path.encode(), out.ctypes.data_as(C.c_void_p), n) < 0:
            _err("%s(%s)" % (fn.__name__, path))
        return out

    def net_params(self, path):
        """Flat parameter vector of the module tree at `path` in getParameters() order."""
        return self._vec(self.lib.fg_t7_net_params, path)

    def net_bn_state(self, path):
        return self._vec(self.lib.fg_t7_net_bn_state, path)

    def net_describe(self, path):
        n = int(self.lib.fg_t7_net_describe(self.h, path.encode(), None, 0))
        if n < 0:
            raise FGError("fg_t7_net_describe(%s): no such entry" % path)
        buf = C.create_string_buffer(n + 1)
        self.lib.fg_t7_net_describe(self.h, path.encode(), buf, n + 1)
        return buf.value.decode()


class T7Writer:
    def __init__(self, path):
        self.lib = load_library()
        h = C.c_void_p()
        if self.lib.fg_t7_writer_open(str(path).encode(), C.byref(h)) != 0:
            _err("fg_t7_writer_open")
        self.h = h

    def add(self, key, value):
        k = key.encode()
        if isinstance(value, str):
            rc = self.lib.fg_t7_writer_add_string(self.h, k, value.encode())
        elif isinstance(value, (int, float, np.integer, np.floating)):
            rc = self.lib.fg_t7_writer_add_number(self.h, k, float(value))
        else:
            a = np.ascontiguousarray(value, np.float32)
            dims = (C.c_int64 * a.ndim)(*a.shape)
            rc = self.lib.fg_t7_writer_add_tensor(self.h, k, a.ctypes.data_as(C.c_void_p), dims, a.ndim)
        if rc != 0:
            _err("fg_t7_writer_add(%s)" % key)

    def close(self):
        if self.h:
            rc = self.lib.fg_t7_writer_close(self.h)
            self.h = None
            if rc != 0:
                _err("fg_t7_writer_close")


# models.lua's discriminators as module lists (nn.Module class names, containers with their children in braces), one
# letter per leaf: C SpatialConvolution, P PReLU, M SpatialMaxPooling, A SpatialAveragePooling, S SpatialDropout,
# V View, L Linear, D Dropout, J JoinTable, G Sigmoid
_LEAF = dict(C="nn.SpatialConvolution", P="nn.PReLU", M="nn.SpatialMaxPooling", A="nn.SpatialAveragePooling",
             S="nn.SpatialDropout", V="nn.View", L="nn.Linear", D="nn.Dropout", J="nn.JoinTable", G="nn.Sigmoid")
_DENSE = "VLPDLP"
_DISC_TREES = {  # (branches of the ConcatTable or None, modules of the Sequential after it)
    "create_D32b": (None, "CPSA" * 4 + "VLPDLPDLG"),
    "create_D16_d": (["CPCPACPCPSVLP", "VLPDLP"], "JLG"),
    "create_D32": (["CPCPMSVLP", "CPCPMCPCPMSVLPDLP", _DENSE], "JLPDLG"),
    "create_D16": (["CPCPMSVLPD", "CPCPMSVLPD", _DENSE], "JLPDLG"),
    "create_D16_b": (["CPCPCPCPSVLPD", "CPCPCPCPSVLPD", _DENSE], "JLPDLG"),
    "create_D16_c": (["CPCPCPCPCPSVLP", "CPCPCPCPCPSVLP", _DENSE], "JLPDLG"),
}


def disc_module_list(name):
    """the fg_t7_net_describe skeleton of models.lua's discriminator `name` (without the CUDA-mode Copy wrapper)"""
    branches, tail = _DISC_TREES[name]
    seq = lambda letters: "nn.Sequential{%s}" % ",".join(_LEAF[c] for c in letters)
    mods = ([] if branches is None else ["nn.ConcatTable{%s}" % ",".join(seq(b) for b in branches)])
    return "nn.Sequential{%s}" % ",".join(mods + [_LEAF[c] for c in tail])


def recognise_disc(describe):
    """the models.lua discriminator whose module list `describe` (fg_t7_net_describe) is, or None.  The CUDA-mode
    wrapper nn.Sequential{nn.Copy, net, nn.Copy} (utils/nn_utils.lua:328-363) and cudnn.* classes are accepted."""
    d = describe.replace("cudnn.", "nn.")
    pre, post = "nn.Sequential{nn.Copy,", ",nn.Copy}"
    if d.startswith(pre) and d.endswith(post):
        d = d[len(pre):-len(post)]
    for name in _DISC_TREES:
        if d == disc_module_list(name):
            return name
    return None


def _check_disc(f, want, channels, what):
    """D of checkpoint f against the net's discriminator `want`: a recognised other D is refused naming both; any D
    whose length is not `want`'s is refused"""
    desc = f.net_describe("D")
    have = recognise_disc(desc)
    if have is not None and have != want:
        raise FGError("checkpoint D is %s; %s has %s" % (have, what, want))
    pd = f.net_params("D")
    n = disc_param_count(want, channels)
    if pd.size != n:
        raise FGError("checkpoint D has %d parameters (%s); %s has %s with %d" % (pd.size, desc, what, want, n))
    return pd


def load_reference_checkpoint(ctx, path, want_D=True):
    """sample.lua:247-258 `loadModels`: upload G (and D) of a reference `adversarial.net` into a Context.
    Raises if G is not the 32x32 generator or D is not the discriminator the Context was created with."""
    with T7File(path) as f:
        pg = f.net_params("G")
        if pg.size != ctx.count(NET_G):
            raise FGError("checkpoint G has %d parameters (%s); this build implements create_G_decoder_upsampling32 with %d"
                          % (pg.size, f.net_describe("G"), ctx.count(NET_G)))
        ctx.set_params(NET_G, pg)
        bn = f.net_bn_state("G")
        if bn.size == 768:
            ctx.set_bn_state(bn)
        elif bn.size:
            raise FGError("checkpoint G carries %d BatchNorm running statistics, expected 768 (2 layers: 256 + 128 channels)"
                          % bn.size)
        else:
            # prepareNetworkForSave never strips running_mean / running_var (utils/nn_utils.lua:259-279), so a stock
            # checkpoint always has them; without them evaluate()-mode G would silently use stale statistics
            import warnings
            warnings.warn("checkpoint G holds no BatchNorm running statistics: evaluate()-mode forwards will use the "
                          "context's current ones (training-mode forwards, incl. sample.lua's, are unaffected)")
        if want_D and f.kind("D") is not None:
            ctx.set_params(NET_D, _check_disc(f, ctx.discriminator, ctx.C, "this 32x32 net"))
        return int(f.number("epoch")) if f.kind("epoch") == "number" else None


# models_c2f.lua's nets: G's "same" SpatialConvolutionUpsample layers (Cout, k) after the C+1 joined planes, Cout 0 =
# the C image channels; D's 3x3 convolutions (Cout, 2x2 max pool after) (include/fg_b200.h FG_C2F_G_* / FG_C2F_D_*)
C2F_G_LAYERS = {
    "create_G_d": [(64, 3), (64, 3), (128, 5), (256, 5), (0, 7)],
    "create_G_a": [(64, 3), (128, 7), (0, 5)],
    "create_G_b": [(64, 3), (64, 3), (256, 5), (0, 7)],
    "create_G_c": [(64, 3), (128, 3), (256, 5), (0, 7)],
}
C2F_D_LAYERS = {
    "create_D_c": [(64, False), (64, True), (128, False), (256, True)],
    "create_D_a": [(64, False), (64, True)],
    "create_D_b": [(64, False), (64, True), (128, False), (128, True)],
}


def c2f_G_module_list(name):
    """the fg_t7_net_describe skeleton of models_c2f.lua's generator `name` (cuda = false: no Copy layers)"""
    inner = ["nn.SpatialConvolutionUpsample", "nn.PReLU"] * (len(C2F_G_LAYERS[name]) - 1)
    return "nn.Sequential{nn.JoinTable,nn.Sequential{%s}}" % ",".join(inner + ["nn.SpatialConvolutionUpsample", "nn.View"])


def c2f_D_module_list(name):
    """the fg_t7_net_describe skeleton of models_c2f.lua's discriminator `name` (cuda = false: no Copy layers)"""
    inner = []
    for _, pool in C2F_D_LAYERS[name]:
        inner += ["nn.SpatialConvolution", "nn.PReLU"] + (["nn.SpatialMaxPooling"] if pool else [])
    inner += ["nn.Dropout", "nn.View", "nn.Linear", "nn.PReLU", "nn.Dropout", "nn.Linear", "nn.Sigmoid"]
    return "nn.Sequential{nn.CAddTable,nn.Sequential{%s}}" % ",".join(inner)


def c2f_G_conv_shapes(name, channels):
    """the weight shapes (Cout, Cin, k, k) of the generator's convolutions in module order"""
    out, cin = [], channels + 1
    for cout, k in C2F_G_LAYERS[name]:
        cout = cout or channels
        out.append((cout, cin, k, k))
        cin = cout
    return out


def c2f_D_conv_shapes(name, channels):
    out, cin = [], channels
    for cout, _ in C2F_D_LAYERS[name]:
        out.append((cout, cin, 3, 3))
        cin = cout
    return out


def _c2f_plain(describe):
    """describe without the CUDA-mode Copy layers models_c2f.lua inserts (cuda = true) and with cudnn.* as nn.*"""
    return describe.replace("cudnn.", "nn.").replace(",nn.Copy", "")


def _recognise(describe, conv_shapes, names, module_list, shapes):
    d = _c2f_plain(describe)
    for name in names:
        if d != module_list(name):
            continue
        for C in (1, 3):
            if [tuple(s) for s in conv_shapes] == shapes(name, C):
                return name
    return None


def recognise_c2f_G(describe, conv_shapes):
    """the models_c2f.lua generator whose module list `describe` (fg_t7_net_describe) and convolution weight shapes
    `conv_shapes` (module order) these are, or None.  The CUDA-mode Copy layers and cudnn.* classes are accepted."""
    return _recognise(describe, conv_shapes, C2F_G_LAYERS, c2f_G_module_list, c2f_G_conv_shapes)


def recognise_c2f_D(describe, conv_shapes):
    """the models_c2f.lua discriminator of `describe` and `conv_shapes`, as recognise_c2f_G"""
    return _recognise(describe, conv_shapes, C2F_D_LAYERS, c2f_D_module_list, c2f_D_conv_shapes)


def conv_weight_shapes(f, path, limit=256):
    """the weight shapes of every (Spatial)Convolution* leaf of the module tree at `path`, in module order (at most
    `limit` modules are visited, so a cyclic or huge tree ends the walk)"""
    out, seen = [], [0]

    def walk(p, depth):
        seen[0] += 1
        if seen[0] > limit or depth > 16:
            raise FGError("%s is not a plausible module tree" % path)
        if f.kind(p + ".modules") == "table":
            i = 1
            while f.kind("%s.modules.%d" % (p, i)) is not None:
                walk("%s.modules.%d" % (p, i), depth + 1)
                i += 1
        elif "Convolution" in f.string(p) and f.kind(p + ".weight") == "tensor":
            out.append(f.tensor(p + ".weight").shape)

    walk(path, 0)
    return out


def _c2f_fit(n_params, count):
    """' (the count of a c2f D with C channels at fine size S)' for the (C, S) whose count(C, S) is n_params, else ''"""
    fits = ["%d channels at fine size %d" % (c, s) for c in (1, 3) for s in (16, 32, 64) if count(c, s) == n_params]
    return " (that of %s)" % " or ".join(fits) if fits else ""


def read_c2f_checkpoint(path, channels, fine_size, generator="create_G_d", discriminator="create_D_c"):
    """adversarial_c2f.lua:207-216's `adversarial_c2f_<cs>_to_<S>.net` ({D, G, opt, epoch}) as flat vectors:
    dict(PG, PD, epoch) in getParameters() order.  Refuses a G or D that does not fit the c2f nets `generator` /
    `discriminator` with `channels` channels at fine size `fine_size` (create_D_c's Linear reads 256*(S/4)^2
    features): a recognised other models_c2f.lua net is named, any other tree is refused by its length.  Needs no
    GPU."""
    if fine_size not in (16, 32, 64):
        raise FGError("fine size %d is not supported (16, 32 or 64)" % fine_size)
    nG = c2f_gen_param_count(generator, channels)
    nD = c2f_disc_param_count(discriminator, channels, fine_size)
    with T7File(path) as f:
        for key, want, recognise in (("G", generator, recognise_c2f_G), ("D", discriminator, recognise_c2f_D)):
            have = recognise(f.net_describe(key), conv_weight_shapes(f, key))
            if have is not None and have != want:
                raise FGError("checkpoint %s is %s; the c2f net has %s" % (key, have, want))
        pg = f.net_params("G")
        if pg.size != nG:
            raise FGError("checkpoint G has %d parameters (%s); the c2f G with %d channels has %d (%s)"
                          % (pg.size, f.net_describe("G"), channels, nG, generator))
        pd = f.net_params("D")
        if pd.size != nD:
            fit = _c2f_fit(pd.size, lambda c, s: c2f_disc_param_count(discriminator, c, s))
            raise FGError("checkpoint D has %d parameters%s (%s); the c2f D with %d channels at fine size %d has %d (%s)"
                          % (pd.size, fit, f.net_describe("D"), channels, fine_size, nD, discriminator))
        epoch = int(f.number("epoch")) if f.kind("epoch") == "number" else None
    return dict(PG=pg, PD=pd, epoch=epoch)


def load_c2f_checkpoint(net, path):
    """load G and D of an `adversarial_c2f_<cs>_to_<S>.net` into a C2f of the same nets, channels and fine size;
    returns the epoch (None when the file has none)"""
    ck = read_c2f_checkpoint(path, net.C, net.S, net.generator, net.discriminator)
    net.set_params(NET_G, ck["PG"])
    net.set_params(NET_D, ck["PD"])
    return ck["epoch"]


def read_s16_checkpoint(path, channels, discriminator="create_D16_d"):
    """an `adversarial.net` trained with train.lua --scale 16 (create_G_decoder_upsampling16 and `discriminator`:
    create_D16_d, or create_D16 / _b / _c) as flat vectors: dict(PG, bn, PD, epoch); bn = G's 768 BatchNorm running
    statistics, PD None when the file has no D.  Needs no GPU."""
    lib = load_library()
    nG = int(lib.fg_s16_param_count(NET_G, channels))
    with T7File(path) as f:
        pg = f.net_params("G")
        if pg.size != nG:
            raise FGError("checkpoint G has %d parameters (%s); the --scale 16 G with %d channels has %d"
                          % (pg.size, f.net_describe("G"), channels, nG))
        bn = f.net_bn_state("G")
        if bn.size != 768:
            raise FGError("checkpoint G carries %d BatchNorm running statistics, expected 768 (2 layers: 256 + 128 channels)"
                          % bn.size)
        pd = None
        if f.kind("D") is not None:
            pd = _check_disc(f, discriminator, channels, "the --scale 16 D with %d channels" % channels)
        epoch = int(f.number("epoch")) if f.kind("epoch") == "number" else None
    return dict(PG=pg, bn=bn, PD=pd, epoch=epoch)


def load_s16_checkpoint(net, path):
    """load G (with its BatchNorm running statistics) and, when present, D of a --scale 16 `adversarial.net` into an
    S16; returns the epoch (None when the file has none)"""
    ck = read_s16_checkpoint(path, net.C, net.discriminator)
    net.set_params(NET_G, ck["PG"])
    net.set_bn_state(ck["bn"])
    if ck["PD"] is not None:
        net.set_params(NET_D, ck["PD"])
    return ck["epoch"]


def save_flat_checkpoint(ctx, path, epoch=0, extra=None):
    """Everything needed to resume: parameters, Adam moments and step counters, BN running statistics."""
    w = T7Writer(path)
    for name, net in (("G", NET_G), ("D", NET_D)):
        w.add(name, ctx.get_params(net))
        m, v, t = ctx.get_adam_state(net)
        w.add("adam_%s_m" % name, m)
        w.add("adam_%s_v" % name, v)
        w.add("adam_%s_t" % name, t)
    w.add("bn_G", ctx.get_bn_state())
    w.add("epoch", epoch)
    w.add("format", "fg_b200 flat checkpoint: getParameters()-ordered vectors of create_G_decoder_upsampling32 / create_D32b")
    for k, v in (extra or {}).items():
        w.add(k, v)
    w.close()


def load_flat_checkpoint(ctx, path):
    with T7File(path) as f:
        for name, net in (("G", NET_G), ("D", NET_D)):
            ctx.set_params(net, f.tensor(name))
            ctx.set_adam_state(net, f.tensor("adam_%s_m" % name), f.tensor("adam_%s_v" % name),
                               int(f.number("adam_%s_t" % name)))
        ctx.set_bn_state(f.tensor("bn_G"))
        return int(f.number("epoch"))


def read_denoiser_checkpoint(path, channels, size):
    """train_denoiser.lua's `denoiser_CxHxW.net` ({AE1_ENCODER, AE1_DECODER, AE2_DECODER}, :360-362) as flat vectors:
    dict(P1, P2, bn1, bn2), the getParameters() order and BatchNorm running statistics of the two decoders (AE2_DECODER
    may be absent: P2 / bn2 None).  Needs no GPU."""
    from .denoiser import BN_STATE, param_count
    n = param_count(channels, size)
    out = {}
    with T7File(path) as f:
        for key, pk, bk in (("AE1_DECODER", "P1", "bn1"), ("AE2_DECODER", "P2", "bn2")):
            if f.kind(key) is None:
                if key == "AE1_DECODER":
                    raise FGError("%s holds no AE1_DECODER" % path)
                out[pk] = out[bk] = None
                continue
            p = f.net_params(key)
            if p.size != n:
                raise FGError("checkpoint %s has %d parameters (%s); the %dx%dx%d denoiser has %d"
                              % (key, p.size, f.net_describe(key), channels, size, size, n))
            bn = f.net_bn_state(key)
            if bn.size != BN_STATE:
                raise FGError("checkpoint %s carries %d BatchNorm running statistics, expected %d (8 + 8 + 2048 channels)"
                              % (key, bn.size, BN_STATE))
            out[pk], out[bk] = p, bn
    return out


def load_denoiser_checkpoint(dn, path):
    """train.lua --denoise (:101-110): load `denoiser_CxHxW.net` into a Denoiser (both decoders when present)."""
    ck = read_denoiser_checkpoint(path, dn.C, dn.S)
    for net, pk, bk in ((0, "P1", "bn1"), (1, "P2", "bn2")):
        if ck[pk] is not None:
            dn.set_params(net, ck[pk])
            dn.set_bn_state(net, ck[bk])
    return ck


def read_autoencoder_checkpoint(path, size, noise_dim):
    """train_autoencoder.lua's `autoencoder.net` ({AE = MODEL_AE, optstate = OPTSTATE}, :234): MODEL_AE's parameters in
    getParameters() order.  The script's Adam state is per-parameter-tensor tables inside optstate and is not read:
    training resumes with fresh moments, as the script itself does after a restart.  Needs no GPU."""
    from .autoencoder import param_count
    n = param_count(size, noise_dim)
    with T7File(path) as f:
        if f.kind("AE") is None:
            raise FGError("%s holds no AE" % path)
        p = f.net_params("AE")
        if p.size != n:
            raise FGError("checkpoint AE has %d parameters (%s); the %dx%d autoencoder with noiseDim %d has %d"
                          % (p.size, f.net_describe("AE"), size, size, noise_dim, n))
        return p


def load_autoencoder_checkpoint(ae, path):
    """load the AE of an `autoencoder.net` into an Autoencoder of the same --scale and --noiseDim"""
    p = read_autoencoder_checkpoint(path, ae.S, ae.d)
    ae.set_params(p)
    return p


def save_autoencoder_flat(ae, path, epoch=0):
    """Everything needed to resume an Autoencoder: parameters, Adam moments and step counter, as flat tensors in one root
    table that stock torch.load reads."""
    w = T7Writer(path)
    w.add("AE", ae.get_params())
    m, v, t = ae.get_adam_state()
    w.add("adam_m", m)
    w.add("adam_v", v)
    w.add("adam_t", t)
    w.add("scale", ae.S)
    w.add("noiseDim", ae.d)
    w.add("epoch", epoch)
    w.add("format", "fg_b200 flat checkpoint: getParameters()-ordered vector of train_autoencoder.lua's MODEL_AE")
    w.close()


def load_autoencoder_flat(ae, path):
    with T7File(path) as f:
        if int(f.number("scale")) != ae.S or int(f.number("noiseDim")) != ae.d:
            raise FGError("%s was saved at scale %d, noiseDim %d; this autoencoder has %d, %d"
                          % (path, f.number("scale"), f.number("noiseDim"), ae.S, ae.d))
        ae.set_params(f.tensor("AE"))
        ae.set_adam_state(f.tensor("adam_m"), f.tensor("adam_v"), int(f.number("adam_t")))
        return int(f.number("epoch"))
