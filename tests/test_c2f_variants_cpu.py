"""CPU: models_c2f.lua's coarse-to-fine generators and discriminators (create_G_a, _b, _c, _d; create_D_a, _b, _c).

 * tests/c2f_var_ref.py (the float64 restatement the GPU tests hold the CUDA path to) against torch.nn modules built
   independently from the same shapes, forward and every gradient, for every net at 1 and 3 channels; for the default
   pair it equals tests/torch_ref_c2f.py;
 * parameter counts and keep-flag widths written out by hand from models_c2f.lua's layer shapes, against the C ABI;
 * adversarial_c2f_*.net checkpoint trees of every G and D (with and without the CUDA-mode Copy layers) are recognised,
   read in getParameters() order and refused for a pair holding another net.
"""
import numpy as np
import pytest
import torch

import c2f_var_ref as V
from face_generator_b200.lib import FGError

nn = torch.nn


def _modules_G(name, C, P):
    """the generator as torch.nn modules, parameters copied from P in getParameters() order"""
    mods, o = [], 0
    convs = V.G_convs(name, C)
    for i, (cin, cout, k) in enumerate(convs):
        conv = nn.Conv2d(cin, cout, k, padding=k // 2).double()
        mods.append(conv)
        if i < len(convs) - 1:
            mods.append(nn.PReLU(1).double())
    return nn.Sequential(*mods), _load(mods, P)


def _modules_D(name, C, S, P):
    mods = []
    for cin, cout, _, pool in V.D_convs(name, C, S):
        mods += [nn.Conv2d(cin, cout, 3, padding=1).double(), nn.PReLU(1).double()]
        if pool:
            mods.append(nn.MaxPool2d(2))
    vc, vh = V.D_view(name, S)
    head = [nn.Linear(vc * vh * vh, 512).double(), nn.PReLU(1).double(), nn.Linear(512, 1).double()]
    _load(mods + head, P)
    return nn.Sequential(*mods), head


def _load(mods, P):
    o = 0
    with torch.no_grad():
        for m in mods:
            for t in m.parameters():  # weight, then bias
                t.copy_(torch.from_numpy(P[o:o + t.numel()]).view_as(t))
                o += t.numel()
    assert o == P.size
    return o


def _grads(mods):
    return np.concatenate([t.grad.numpy().ravel() for m in mods for t in m.parameters()])


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("name", V.GENERATORS)
def test_G_restatement_equals_torch_modules(name, C):
    S, B = 16, 3
    rng = np.random.default_rng(C + len(name))
    P = V.trained_like(V.G_layout(name, C), rng)
    noise, cond = rng.uniform(-1, 1, (B, 1, S, S)), rng.random((B, C, S, S))
    dout = rng.standard_normal((B, C, S, S))
    Pt = torch.from_numpy(P).requires_grad_(True)
    out = V.G_forward(Pt, torch.from_numpy(noise), torch.from_numpy(cond), name, C)
    out.backward(torch.from_numpy(dout))
    net, _ = _modules_G(name, C, P)
    ref = net(torch.cat([torch.from_numpy(noise), torch.from_numpy(cond)], 1))
    ref.backward(torch.from_numpy(dout))
    assert out.shape == (B, C, S, S)
    np.testing.assert_allclose(out.detach().numpy(), ref.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(Pt.grad.numpy(), _grads(list(net)), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("S", V.FINE_SIZES)
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("name", V.DISCRIMINATORS)
def test_D_restatement_equals_torch_modules(name, C, S):
    B = 3
    rng = np.random.default_rng(10 * C + S)
    P = V.trained_like(V.D_layout(name, C, S), rng, 1.0)
    diff, cond = rng.standard_normal((B, C, S, S)) * 0.1, rng.random((B, C, S, S))
    masks = (rng.random((B, V.mask_per_sample(name, S))) < 0.5).astype(np.float64)
    dout = rng.standard_normal(B)
    Pt = torch.from_numpy(P).requires_grad_(True)
    x = torch.from_numpy(diff).requires_grad_(True)
    out = V.D_forward(Pt, x, torch.from_numpy(cond), torch.from_numpy(masks), name, C, S)
    out.backward(torch.from_numpy(dout))
    convs, (L1, pr, L2) = _modules_D(name, C, S, P)
    xr = torch.from_numpy(diff).requires_grad_(True)
    m = torch.from_numpy(masks)
    h = convs(xr + torch.from_numpy(cond)).reshape(B, -1)
    n = h.shape[1]
    assert n + 512 == masks.shape[1]
    ref = torch.sigmoid(L2(pr(L1(h * m[:, :n] * 2.0)) * m[:, n:] * 2.0)).reshape(B)
    ref.backward(torch.from_numpy(dout))
    # the restatement's Sigmoid hands on a float32 output (torch_ref.d_sigmoid, as the reference's fp32 D): 1e-6
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()
    assert rel(out.detach().numpy(), ref.detach().numpy()) < 1e-6
    assert rel(x.grad.numpy(), xr.grad.numpy()) < 1e-6
    g, gr = Pt.grad.numpy(), _grads(list(convs) + [L1, pr, L2])
    for k, (o, s) in V.D_layout(name, C, S).items():
        n = int(np.prod(s))
        assert rel(g[o:o + n], gr[o:o + n]) < 1e-6, k


def test_default_pair_equals_torch_ref_c2f():
    import torch_ref_c2f as RC
    from oracle import oracle_c2f as OC
    C, B = 3, 2
    rng = np.random.default_rng(5)
    assert {k: s for k, (o, s) in V.G_layout("create_G_d", C).items()} == {k: s for k, (o, s) in OC.G_layout(C).items()}
    PG, PD = RC.trained_like_G(C, rng), RC.trained_like_D(C, rng)
    noise, cond = torch.from_numpy(rng.uniform(-1, 1, (B, 1, 32, 32))), torch.from_numpy(rng.random((B, C, 32, 32)))
    masks = torch.from_numpy(RC.make_masks(B, rng))
    a = V.G_forward(torch.from_numpy(PG), noise, cond, "create_G_d", C)
    b = RC.G_forward(torch.from_numpy(PG), noise, cond, C)
    assert torch.equal(a, b)
    a = V.D_forward(torch.from_numpy(PD), a, cond, masks, "create_D_c", C, 32)
    b = RC.D_forward(torch.from_numpy(PD), b, cond, masks, C)
    assert torch.equal(a, b)


# ---- counts: written out by hand from models_c2f.lua's layer shapes -------------------------------------------------
def _conv(cin, cout, k):
    return cout * cin * k * k + cout


def hand_G(name, C):
    J = C + 1  # JoinTable{noise, coarse}
    return {
        # :113-145  SCU(C+1,64,3) P SCU(64,64,3) P SCU(64,128,5) P SCU(128,256,5) P SCU(256,C,7)
        "create_G_d": _conv(J, 64, 3) + 1 + _conv(64, 64, 3) + 1 + _conv(64, 128, 5) + 1 + _conv(128, 256, 5) + 1
        + _conv(256, C, 7),
        # :16-45  SCU(C+1,64,3) P SCU(64,128,7) P SCU(128,C,5)
        "create_G_a": _conv(J, 64, 3) + 1 + _conv(64, 128, 7) + 1 + _conv(128, C, 5),
        # :47-78  SCU(C+1,64,3) P SCU(64,64,3) P SCU(64,256,5) P SCU(256,C,7)
        "create_G_b": _conv(J, 64, 3) + 1 + _conv(64, 64, 3) + 1 + _conv(64, 256, 5) + 1 + _conv(256, C, 7),
        # :80-111  SCU(C+1,64,3) P SCU(64,128,3) P SCU(128,256,5) P SCU(256,C,7)
        "create_G_c": _conv(J, 64, 3) + 1 + _conv(64, 128, 3) + 1 + _conv(128, 256, 5) + 1 + _conv(256, C, 7),
    }[name]


def hand_D(name, C, S):
    head = lambda n_in: n_in * 512 + 512 + 1 + 512 + 1  # Linear(n_in, 512) PReLU Linear(512, 1)
    return {
        # :156-192  conv(C,64) P conv(64,64) P pool | View(64*S/2*S/2)
        "create_D_a": _conv(C, 64, 3) + 1 + _conv(64, 64, 3) + 1 + head(64 * (S // 2) ** 2),
        # :194-235  conv(C,64) P conv(64,64) P pool conv(64,128) P conv(128,128) P pool | View(128*S/4*S/4)
        "create_D_b": _conv(C, 64, 3) + 1 + _conv(64, 64, 3) + 1 + _conv(64, 128, 3) + 1 + _conv(128, 128, 3) + 1
        + head(128 * (S // 4) ** 2),
        # :237-278  conv(C,64) P conv(64,64) P pool conv(64,128) P conv(128,256) P pool | View(256*S/4*S/4)
        "create_D_c": _conv(C, 64, 3) + 1 + _conv(64, 64, 3) + 1 + _conv(64, 128, 3) + 1 + _conv(128, 256, 3) + 1
        + head(256 * (S // 4) ** 2),
    }[name]


def hand_mask(name, S):
    return {"create_D_a": 64 * (S // 2) ** 2, "create_D_b": 128 * (S // 4) ** 2, "create_D_c": 256 * (S // 4) ** 2}[name] + 512


def test_counts_and_widths_match_the_c_abi():
    from face_generator_b200.lib import (C2F_DISCRIMINATORS, C2F_GENERATORS, c2f_disc_param_count, c2f_gen_param_count,
                                         c2f_mask_per_sample, load_library)
    lib = load_library()
    for name, gid in C2F_GENERATORS.items():
        for C in (1, 3):
            n = hand_G(name, C)
            assert c2f_gen_param_count(name, C) == lib.fg_c2f_gen_param_count(gid, C) == n == V.count(V.G_layout(name, C))
    for name, did in C2F_DISCRIMINATORS.items():
        for S in (16, 32, 64):
            for C in (1, 3):
                n = hand_D(name, C, S)
                assert c2f_disc_param_count(name, C, S) == lib.fg_c2f_disc_param_count(did, C, S) == n
                assert n == V.count(V.D_layout(name, C, S))
            assert hand_D(name, 1, S) == hand_D(name, 3, S) - 1152
            assert c2f_mask_per_sample(S, name) == lib.fg_c2f_disc_mask_per_sample(did, S) == hand_mask(name, S)
            assert hand_mask(name, S) == V.mask_per_sample(name, S)
    # the defaults: DEFAULT (0) and the named entries agree with the existing entry points
    for C in (1, 3):
        assert lib.fg_c2f_gen_param_count(0, C) == lib.fg_c2f_gen_param_count(1, C) == lib.fg_c2f_param_count(0, C)
        for S in (16, 32, 64):
            assert lib.fg_c2f_disc_param_count(0, C, S) == lib.fg_c2f_param_count_sized(1, C, S) == hand_D("create_D_c", C, S)
    for S in (16, 32, 64):
        assert lib.fg_c2f_disc_mask_per_sample(0, S) == lib.fg_c2f_mask_per_sample_sized(S)
    # create_D_a and create_D_c keep as many flags at every size
    assert all(hand_mask("create_D_a", S) == hand_mask("create_D_c", S) for S in (16, 32, 64))


def test_unknown_nets_and_sizes_return_minus_one():
    from face_generator_b200.lib import c2f_disc_id, c2f_gen_id, load_library
    lib = load_library()
    for g in (-1, 5, 99):
        assert lib.fg_c2f_gen_param_count(g, 3) == -1
    for d in (-1, 4, 99):
        assert lib.fg_c2f_disc_param_count(d, 3, 32) == -1
        assert lib.fg_c2f_disc_mask_per_sample(d, 32) == -1
    for S in (0, 8, 48, 128):
        assert lib.fg_c2f_disc_param_count(1, 3, S) == -1
        assert lib.fg_c2f_disc_mask_per_sample(2, S) == -1
    assert lib.fg_c2f_gen_param_count(2, 0) == -1 and lib.fg_c2f_disc_param_count(2, 0, 32) == -1
    with pytest.raises(FGError, match="unknown c2f generator"):
        c2f_gen_id("create_G_e")
    with pytest.raises(FGError, match="unknown c2f discriminator"):
        c2f_disc_id("create_D32b")


def test_python_counts_refuse_unsupported_sizes():
    from face_generator_b200.lib import c2f_disc_param_count, c2f_gen_param_count, c2f_mask_per_sample
    for S in (0, 8, 48):
        with pytest.raises(FGError, match="fine size %d" % S):
            c2f_mask_per_sample(S)
        with pytest.raises(FGError, match="fine size %d" % S):
            c2f_disc_param_count("create_D_a", 3, S)
    with pytest.raises(FGError, match="0 channels"):
        c2f_gen_param_count("create_G_b", 0)
    assert c2f_mask_per_sample(32) == 256 * 8 * 8 + 512


def test_create_nets_refuses_null_arguments():
    from face_generator_b200.lib import load_library
    import ctypes as C
    lib = load_library()
    h = C.c_void_p()
    assert lib.fg_c2f_create_nets(None, 32, 2, 2, C.byref(h)) != 0
    assert lib.fg_c2f_get_gen(None) < 0 and lib.fg_c2f_get_disc(None) < 0


# ---- checkpoints: adversarial_c2f.lua:216's {D, G, opt, epoch} with models_c2f.lua's trees --------------------------
def c2f_tree(kind, name, C, S, P, cuda):
    """models_c2f.lua's net as saved: Sequential{JoinTable | CAddTable, [Copy], Sequential{layers}, [Copy]}, every
    weight / bias a view into one flat storage P"""
    import test_t7 as T
    st_cls, t_cls = ("torch.CudaStorage", "torch.CudaTensor") if cuda else ("torch.FloatStorage", "torch.FloatTensor")
    st = T.Storage(P, st_cls)
    o = [0]

    def param(shape):
        t = T.Tensor(st, shape, offset=o[0], cls=t_cls)
        o[0] += int(np.prod(shape))
        return t

    def conv(cls, cin, cout, k):
        w = param((cout, cin, k, k))
        return T.Obj(cls, {"weight": w, "bias": param((cout,)), "nInputPlane": cin, "nOutputPlane": cout, "kW": k,
                           "kH": k, "train": True})

    prelu = lambda: T.Obj("nn.PReLU", {"weight": param((1,)), "train": True})
    leaf = lambda cls: T.Obj(cls, {"train": True})
    mods = []
    if kind == "G":
        convs = V.G_convs(name, C)
        for i, (cin, cout, k) in enumerate(convs):
            mods.append(conv("cudnn.SpatialConvolutionUpsample", cin, cout, k))
            if i < len(convs) - 1:
                mods.append(prelu())
        mods.append(leaf("nn.View"))
        first = T.Obj("nn.JoinTable", {"dimension": 2, "nInputDims": 2})
    else:
        for cin, cout, _, pool in V.D_convs(name, C, S):
            mods += [conv("nn.SpatialConvolution", cin, cout, 3), prelu()] + ([leaf("nn.SpatialMaxPooling")] if pool else [])
        vc, vh = V.D_view(name, S)
        mods += [leaf("nn.Dropout"), leaf("nn.View")]
        mods.append(T.Obj("nn.Linear", {"weight": param((512, vc * vh * vh)), "bias": param((512,)), "train": True}))
        mods += [prelu(), leaf("nn.Dropout")]
        mods.append(T.Obj("nn.Linear", {"weight": param((1, 512)), "bias": param((1,)), "train": True}))
        mods.append(leaf("nn.Sigmoid"))
        first = leaf("nn.CAddTable")
    assert o[0] == P.size
    copy = lambda a, b: T.Obj("nn.Copy", {"intype": a, "outtype": b, "train": True})
    if cuda:
        return T.seq(first, copy("torch.FloatTensor", "torch.CudaTensor"), T.seq(*mods),
                     copy("torch.CudaTensor", "torch.FloatTensor"))
    return T.seq(first, T.seq(*mods))


def write_c2f(path, gen, disc, C, S, cuda, seed=3):
    import test_t7 as T
    rng = np.random.default_rng(seed)
    PG = rng.standard_normal(V.count(V.G_layout(gen, C))).astype(np.float32)
    PD = rng.standard_normal(V.count(V.D_layout(disc, C, S))).astype(np.float32)
    w = T.W()
    w.obj({"G": c2f_tree("G", gen, C, S, PG, cuda), "D": c2f_tree("D", disc, C, S, PD, cuda),
           "opt": {"fineSize": S, "coarseSize": S // 2}, "epoch": 7})
    open(path, "wb").write(bytes(w.buf))
    return PG, PD


@pytest.mark.parametrize("cuda", [True, False], ids=["copy", "plain"])
@pytest.mark.parametrize("gen,disc", [(g, "create_D_c") for g in V.GENERATORS] +
                         [("create_G_d", d) for d in V.DISCRIMINATORS if d != "create_D_c"])
def test_checkpoint_trees_are_recognised_and_loaded(tmp_path, gen, disc, cuda):
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200.checkpoint import T7File
    C, S = 3, 32
    p = tmp_path / "adversarial_c2f_16_to_32.net"
    PG, PD = write_c2f(p, gen, disc, C, S, cuda)
    with T7File(p) as f:
        assert CK.recognise_c2f_G(f.net_describe("G"), CK.conv_weight_shapes(f, "G")) == gen
        assert CK.recognise_c2f_D(f.net_describe("D"), CK.conv_weight_shapes(f, "D")) == disc
    ck = CK.read_c2f_checkpoint(p, C, S, gen, disc)
    np.testing.assert_array_equal(ck["PG"], PG)  # getParameters() order
    np.testing.assert_array_equal(ck["PD"], PD)
    assert ck["epoch"] == 7
    for other in V.GENERATORS:
        if other != gen:
            with pytest.raises(FGError, match="checkpoint G is %s; the c2f net has %s" % (gen, other)):
                CK.read_c2f_checkpoint(p, C, S, other, disc)
    for other in V.DISCRIMINATORS:
        if other != disc:
            with pytest.raises(FGError, match="checkpoint D is %s; the c2f net has %s" % (disc, other)):
                CK.read_c2f_checkpoint(p, C, S, gen, other)
    with pytest.raises(FGError, match="parameters"):  # the same nets at another fine size
        CK.read_c2f_checkpoint(p, C, 64, gen, disc)


@pytest.mark.parametrize("name", V.DISCRIMINATORS)
def test_every_discriminator_is_recognised_at_every_size_and_channel_count(tmp_path, name):
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200.checkpoint import T7File
    for S in V.FINE_SIZES:
        for C in (1, 3):
            p = tmp_path / ("n%d_%d.net" % (S, C))
            write_c2f(p, "create_G_a", name, C, S, cuda=C == 3)
            with T7File(p) as f:
                assert CK.recognise_c2f_D(f.net_describe("D"), CK.conv_weight_shapes(f, "D")) == name
                assert CK.recognise_c2f_G(f.net_describe("G"), CK.conv_weight_shapes(f, "G")) == "create_G_a"
            assert CK.read_c2f_checkpoint(p, C, S, "create_G_a", name)["PD"].size == hand_D(name, C, S)


def test_the_32x32_discriminator_is_not_a_c2f_net(tmp_path):
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200.checkpoint import T7File
    from test_t7 import write_reference_like
    p = tmp_path / "adversarial.net"
    write_reference_like(p, C=3)
    with T7File(p) as f:
        assert CK.recognise_c2f_D(f.net_describe("D"), CK.conv_weight_shapes(f, "D")) is None
        assert CK.recognise_c2f_G(f.net_describe("G"), CK.conv_weight_shapes(f, "G")) is None
