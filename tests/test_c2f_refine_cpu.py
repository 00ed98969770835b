"""CPU: the pieces of the coarse-to-fine refinement (fg_c2f_refine, sample.lua:176-214) that need no GPU.

 * image.scale's enlarge rule (oracle_data.scale) is bilinear interpolation with aligned corners; equal sizes copy.
 * The float64 restatement's pick rule is sample.lua's loop, ties at a saturated 1.0f and NaNs included.
 * Reference-like `adversarial_c2f_<cs>_to_<S>.net` and --scale 16 `adversarial.net` files read back exactly, and a
   wrong fine size or channel count is refused.  The file writer is test_t7.py's, restated here.
"""
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import c2f_refine_ref as RR  # noqa: E402
from face_generator_b200 import layouts as LY  # noqa: E402
from face_generator_b200.lib import FGError  # noqa: E402
from oracle import oracle_data as OD  # noqa: E402


# ------------------------------------------------------------------ torch7 writer (as in test_t7.py)
class Obj:
    def __init__(self, cls, fields):
        self.cls, self.fields = cls, fields


class Tensor:
    def __init__(self, storage, size, stride=None, offset=0, cls="torch.FloatTensor"):
        self.storage, self.size, self.offset, self.cls = storage, list(size), offset, cls
        if stride is None:
            stride, s = [], 1
            for d in reversed(self.size):
                stride.insert(0, s)
                s *= d
        self.stride = list(stride)


class Storage:
    def __init__(self, data, cls="torch.FloatStorage"):
        self.data, self.cls = data, cls


class W:
    def __init__(self):
        self.buf, self.ids = bytearray(), {}

    def i32(self, v):
        self.buf += struct.pack("<i", v)

    def i64(self, v):
        self.buf += struct.pack("<q", v)

    def s(self, v):
        b = v.encode()
        self.i32(len(b))
        self.buf += b

    def ref(self, o, typ):
        self.i32(typ)
        if id(o) in self.ids:
            self.i32(self.ids[id(o)])
            return True
        self.ids[id(o)] = len(self.ids) + 1
        self.i32(self.ids[id(o)])
        return False

    def obj(self, o):
        if o is None:
            self.i32(0)
        elif isinstance(o, bool):
            self.i32(5)
            self.i32(1 if o else 0)
        elif isinstance(o, (int, float)):
            self.i32(1)
            self.buf += struct.pack("<d", float(o))
        elif isinstance(o, str):
            self.i32(2)
            self.s(o)
        elif isinstance(o, dict):
            if self.ref(o, 3):
                return
            self.i32(len(o))
            for k, v in o.items():
                self.obj(k)
                self.obj(v)
        elif isinstance(o, Tensor):
            if self.ref(o, 4):
                return
            self.s("V 1")
            self.s(o.cls)
            self.i32(len(o.size))
            for d in o.size:
                self.i64(d)
            for d in o.stride:
                self.i64(d)
            self.i64(o.offset + 1)
            self.obj(o.storage)
        elif isinstance(o, Storage):
            if self.ref(o, 4):
                return
            self.s("V 1")
            self.s(o.cls)
            self.i64(o.data.size)
            self.buf += o.data.tobytes()
        elif isinstance(o, Obj):
            if self.ref(o, 4):
                return
            self.s("V 1")
            self.s(o.cls)
            self.obj(o.fields)
        else:
            raise TypeError(type(o))


def seq(*mods):
    return Obj("nn.Sequential", {"modules": {i + 1: m for i, m in enumerate(mods)}, "train": True,
                                 "output": Tensor(None, []), "gradInput": Tensor(None, [])})


def cuda_net(flat, layout, classes, tensor_cls="torch.CudaTensor", storage_cls="torch.CudaStorage", bn=None):
    """nn.Sequential{Copy, Sequential{layers...}, Copy}; every weight/bias is a view into the one flat storage."""
    st = Storage(flat, storage_cls)
    gst = Storage(np.zeros_like(flat), storage_cls)
    mods, items = [], list(layout.items())
    i = 0
    for cls, nparam in classes:
        fields = {"train": True}
        for j in range(nparam):
            name, (off, shape) = items[i]
            key = "weight" if j == 0 else "bias"
            fields[key] = Tensor(st, shape, offset=off, cls=tensor_cls)
            fields["grad" + key.capitalize()] = Tensor(gst, shape, offset=off, cls=tensor_cls)
            i += 1
        if "BatchNormalization" in cls and bn is not None:
            fields.update(bn.pop(0))
        mods.append(Obj(cls, fields))
    assert i == len(items)
    copy = lambda a, b: Obj("nn.Copy", {"intype": a, "outtype": b, "train": True})
    return seq(copy("torch.FloatTensor", "torch.CudaTensor"), seq(*mods), copy("torch.CudaTensor", "torch.FloatTensor"))


# create_G_d / create_D_c (models_c2f.lua:113-145, :237-278)
C2F_G_CLASSES = [("cudnn.SpatialConvolutionUpsample", 2), ("nn.PReLU", 1)] * 4 + [("cudnn.SpatialConvolutionUpsample", 2)]
C2F_D_CLASSES = ([("nn.CAddTable", 0)] + [("nn.SpatialConvolution", 2), ("nn.PReLU", 1)] * 2 + [("nn.SpatialMaxPooling", 0)] +
                 [("nn.SpatialConvolution", 2), ("nn.PReLU", 1)] * 2 + [("nn.SpatialMaxPooling", 0), ("nn.Dropout", 0),
                                                                       ("nn.View", 0), ("nn.Linear", 2), ("nn.PReLU", 1),
                                                                       ("nn.Dropout", 0), ("nn.Linear", 2), ("nn.Sigmoid", 0)])
# create_G_decoder_upsampling16 (models.lua:27-51) and a D16 whose modules hold create_D16_d's parameters in order
S16_G_CLASSES = [("nn.Linear", 2), ("nn.View", 0), ("nn.PReLU", 1), ("nn.SpatialUpSamplingNearest", 0),
                 ("cudnn.SpatialConvolution", 2), ("nn.SpatialBatchNormalization", 2), ("nn.PReLU", 1),
                 ("nn.SpatialUpSamplingNearest", 0), ("cudnn.SpatialConvolution", 2), ("nn.SpatialBatchNormalization", 2),
                 ("nn.PReLU", 1), ("cudnn.SpatialConvolution", 2), ("nn.Sigmoid", 0)]
S16_D_CLASSES = ([("nn.SpatialConvolution", 2), ("nn.PReLU", 1)] * 4 + [("nn.Linear", 2), ("nn.PReLU", 1)] * 3 +
                 [("nn.Linear", 2), ("nn.Sigmoid", 0)])


def write_c2f_like(path, C=3, S=64, seed=1):
    """adversarial_c2f.lua:216's torch.save(filename, {D, G, opt, epoch}) for nets of C channels at fine size S"""
    rng = np.random.default_rng(seed)
    (gl, ng), (dl, nd) = LY.c2f_G_layout(C), LY.c2f_D_layout(C, S)
    PG, PD = rng.standard_normal(ng).astype(np.float32), rng.standard_normal(nd).astype(np.float32)
    G = cuda_net(PG, gl, C2F_G_CLASSES)
    G = seq(Obj("nn.JoinTable", {"dimension": 2, "nInputDims": 2}), *G.fields["modules"].values())
    root = {"G": G, "D": cuda_net(PD, dl, C2F_D_CLASSES),
            "opt": {"coarseSize": S // 2, "fineSize": S, "grayscale": C == 1}, "epoch": 11}
    w = W()
    w.obj(root)
    open(path, "wb").write(bytes(w.buf))
    return PG, PD


def write_s16_like(path, C=3, seed=2, with_bn=True, with_D=True):
    """adversarial.lua:328's torch.save for the --scale 16 nets"""
    from oracle import oracle_s16 as O16
    rng = np.random.default_rng(seed)
    gl, dl = O16.G_layout(C), O16.D_layout(C)
    PG = rng.standard_normal(O16.G_param_count(C)).astype(np.float32)
    PD = rng.standard_normal(O16.D_param_count(C)).astype(np.float32)
    rm1, rv1 = rng.standard_normal(256).astype(np.float32), rng.uniform(0.5, 2, 256).astype(np.float32)
    rm2, rv2 = rng.standard_normal(128).astype(np.float32), rng.uniform(0.5, 2, 128).astype(np.float32)
    t1 = lambda a: Tensor(Storage(np.ascontiguousarray(a, np.float32)), [a.size], cls="torch.CudaTensor")
    bn = [{"running_mean": t1(rm1), "running_var": t1(rv1), "eps": 1e-5, "momentum": 0.1},
          {"running_mean": t1(rm2), "running_var": t1(rv2), "eps": 1e-5, "momentum": 0.1}] if with_bn else None
    root = {"G": cuda_net(PG, gl, S16_G_CLASSES, bn=bn), "opt": {"scale": 16}, "epoch": 4}
    if with_D:
        root["D"] = cuda_net(PD, dl, S16_D_CLASSES)
    w = W()
    w.obj(root)
    open(path, "wb").write(bytes(w.buf))
    return PG, PD, np.concatenate([rm1, rv1, rm2, rv2])


# ------------------------------------------------------------------ image.scale
@pytest.mark.parametrize("src,dst", [(16, 32), (32, 64), (16, 64)])
def test_scale_enlarge_is_bilinear_with_aligned_corners(src, dst):
    torch = pytest.importorskip("torch")
    x = np.random.default_rng(src + dst).random((3, 3, src, src))
    ref = torch.nn.functional.interpolate(torch.from_numpy(x), size=(dst, dst), mode="bilinear", align_corners=True)
    # image.scale forms the interpolation fraction in float32: di * scale is off by up to half an ulp of di (< 2^-18 for
    # di < 64), which moves a value in [0, 1) by as much; the exact rule agrees to 1e-6 almost everywhere
    d = np.abs(OD.scale(x, dst, dst) - ref.numpy())
    assert d.max() <= 2.0 ** -18 and np.mean(d > 1e-6) < 1e-3, (d.max(), np.mean(d > 1e-6))


@pytest.mark.parametrize("S", [16, 32, 64])
def test_scale_at_equal_size_is_the_identity(S):
    x = np.random.default_rng(S).random((2, 3, S, S))
    np.testing.assert_array_equal(OD.scale(x, S, S), x)


# ------------------------------------------------------------------ the pick rule
PICK_CASES = {
    "distinct": [0.1, 0.7, 0.3, 0.69],
    "tie_first_wins": [0.2, 0.9, 0.9, 0.1],
    "saturated_ties": [0.5, 1.0, 1.0, 1.0],
    "all_saturated": [1.0, 1.0, 1.0, 1.0],
    "nan_first": [np.nan, 0.9, 1.0, 0.5],
    "nan_later": [0.3, np.nan, 0.2, 0.4],
    "nan_after_max": [0.3, 0.8, np.nan, 0.4],
    "all_nan": [np.nan, np.nan, np.nan, np.nan],
    "single_try": [0.25],
}


@pytest.mark.parametrize("name", sorted(PICK_CASES))
def test_pick_rule_is_sample_lua_loop(name):
    pred = np.asarray(PICK_CASES[name], np.float32)[None]
    assert RR.pick_rule(pred)[0] == RR.lua_pick(list(pred[0]))


def test_pick_rule_on_random_rows_with_ties_and_nans():
    rng = np.random.default_rng(3)
    pred = rng.choice(np.array([0.1, 0.5, 1.0, np.nan], np.float32), size=(500, 10))
    np.testing.assert_array_equal(RR.pick_rule(pred), [RR.lua_pick(list(r)) for r in pred])


def test_refine_restatement_against_literal_loop():
    """the fp64 refine on a small case: out = up + diff[pick] with pick from the loop of sample.lua:199-207"""
    C, S, N, T = 3, 16, 2, 4
    rng = np.random.default_rng(5)
    PG = LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2)
    PD = LY.trained_like_init(LY.c2f_D_layout(C, S), rng, 1.0)
    images = rng.random((N, C, 8, 8))
    noise = rng.uniform(-1, 1, (N * T, 1, S, S))
    from oracle import oracle_c2f_sized as OS
    masks = (rng.random((N * T, OS.mask_per_sample(S))) < 0.5).astype(np.float64)
    for training in (0, 1):
        r = RR.refine(PG, PD, images, S, noise, masks, training)
        up = OD.scale(images, S, S)
        for i in range(N):
            j = RR.lua_pick(list(r["pred"][i].astype(np.float32)))
            assert j == r["pick"][i]
            np.testing.assert_array_equal(r["out"][i], up[i] + r["diff"][i * T + j])


# ------------------------------------------------------------------ checkpoints
@pytest.mark.parametrize("C,S", [(3, 64), (1, 32), (3, 16)])
def test_reads_c2f_checkpoint(tmp_path, C, S):
    from face_generator_b200 import checkpoint as CK
    p = tmp_path / ("adversarial_c2f_%d_to_%d.net" % (S // 2, S))
    PG, PD = write_c2f_like(p, C, S)
    ck = CK.read_c2f_checkpoint(p, C, S)
    np.testing.assert_array_equal(ck["PG"], PG)
    np.testing.assert_array_equal(ck["PD"], PD)
    assert ck["epoch"] == 11


def test_c2f_checkpoint_refuses_other_fine_size_and_channels(tmp_path):
    from face_generator_b200 import checkpoint as CK
    p = tmp_path / "adversarial_c2f_32_to_64.net"
    write_c2f_like(p, 3, 64)
    with pytest.raises(FGError, match="fine size 64.*nn.Sequential"):
        CK.read_c2f_checkpoint(p, 3, 32)
    with pytest.raises(FGError, match="c2f G with 1 channels"):
        CK.read_c2f_checkpoint(p, 1, 64)
    with pytest.raises(FGError):
        CK.read_c2f_checkpoint(p, 3, 48)


@pytest.mark.parametrize("C", [3, 1])
def test_reads_s16_checkpoint(tmp_path, C):
    from face_generator_b200 import checkpoint as CK
    p = tmp_path / "adversarial.net"
    PG, PD, bn = write_s16_like(p, C)
    ck = CK.read_s16_checkpoint(p, C)
    np.testing.assert_array_equal(ck["PG"], PG)
    np.testing.assert_array_equal(ck["PD"], PD)
    np.testing.assert_array_equal(ck["bn"], bn)
    assert ck["epoch"] == 4
    q = tmp_path / "g_only.net"
    write_s16_like(q, C, with_D=False)
    assert CK.read_s16_checkpoint(q, C)["PD"] is None


def test_s16_checkpoint_refuses_wrong_channels_and_missing_statistics(tmp_path):
    from face_generator_b200 import checkpoint as CK
    p = tmp_path / "adversarial.net"
    write_s16_like(p, 3)
    with pytest.raises(FGError, match="--scale 16 G with 1 channels"):
        CK.read_s16_checkpoint(p, 1)
    q = tmp_path / "no_bn.net"
    write_s16_like(q, 3, with_bn=False)
    with pytest.raises(FGError, match="768"):
        CK.read_s16_checkpoint(q, 3)
    # a 32x32 reference checkpoint is not a --scale 16 one
    r = tmp_path / "c2f.net"
    write_c2f_like(r, 3, 32)
    with pytest.raises(FGError):
        CK.read_s16_checkpoint(r, 3)
