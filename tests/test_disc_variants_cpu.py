"""CPU: the float64 restatement of create_D32 / create_D16 / create_D16_b / create_D16_c (tests/dbr_ref.py) against
torch.autograd, and the C ABI's parameter counts, keep-flag widths and side checks for them (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

import dbr_ref as R
from face_generator_b200.lib import FGError

NAMES = ["create_D32", "create_D16", "create_D16_b", "create_D16_c"]


def shapes_count(name, C_):
    """the parameter count from the layer shapes alone (every PReLU() has one slope)"""
    side, branches, (hout, _) = R.NETS[name]
    n, joint = 0, 0
    for _, convs, lins in branches:
        cin, s = C_, side
        for cout, k, stride, pool in convs:
            n += cout * cin * k * k + cout + 1
            s = s // stride // (2 if pool else 1)
            cin = cout
        fin = cin * s * s
        for fout, _ in lins:
            n += fout * fin + fout + 1
            fin = fout
        joint += fin
    return n + hout * joint + hout + 1 + hout + 1


def mask_width(name):
    _, branches, (hout, hdrop) = R.NETS[name]
    m = 0
    for _, convs, lins in branches:
        m += convs[-1][0] if convs else 0
        m += sum(f for f, d in lins if d)
    return m + (hout if hdrop else 0)


@pytest.mark.parametrize("name", NAMES)
def test_param_counts_and_mask_widths_match_the_c_abi(name):
    from face_generator_b200.lib import disc_mask_per_sample, disc_param_count, disc_id, load_library
    lib = load_library()
    for C_ in (1, 3):
        net = R.Net(name, C_)
        assert net.n_params == shapes_count(name, C_)
        assert disc_param_count(name, C_) == net.n_params
    assert disc_mask_per_sample(name) == R.Net(name, 3).mask == mask_width(name)
    assert lib.fg_disc_side(disc_id(name)) == R.NETS[name][0]


def test_the_defaults_keep_their_counts():
    from face_generator_b200.lib import disc_mask_per_sample, disc_param_count, load_library
    lib = load_library()
    for C_ in (1, 3):
        assert disc_param_count("create_D32b", C_) == lib.fg_param_count(1, C_)
        assert disc_param_count("create_D16_d", C_) == lib.fg_s16_param_count(1, C_)
    assert disc_mask_per_sample("create_D32b") == 1984
    assert disc_mask_per_sample("create_D16_d") == lib.fg_s16_mask_per_sample() == 1152
    assert lib.fg_disc_param_count(0, 3) == -1 and lib.fg_disc_mask_per_sample(99) == -1 and lib.fg_disc_side(99) == 0
    assert lib.fg_disc_param_count(3, 2) == -1


def test_a_discriminator_of_the_other_side_is_refused_before_any_allocation():
    from face_generator_b200.lib import load_library, disc_id, FGError, disc_param_count
    lib = load_library()
    h = C.c_void_p()
    for name in ("create_D16", "create_D16_b", "create_D16_c", "create_D16_d"):
        assert lib.fg_create_disc(C.byref(h), 0, 8, 3, disc_id(name)) == -4  # FG_ERR_UNSUPPORTED
        assert b"16x16" in lib.fg_last_error()
        assert not h.value
    assert lib.fg_create_disc(C.byref(h), 0, 8, 3, 42) == -1
    with pytest.raises(FGError):
        disc_param_count("create_D64", 3)


def _case(name, C_, B, seed):
    net = R.Net(name, C_)
    rng = np.random.default_rng(seed)
    P = R.make_params(net, seed, near=False)
    x = rng.uniform(0, 1, (B, C_, net.side, net.side))
    keep = (rng.uniform(0, 1, (B, net.mask)) >= 0.5).astype(np.float64)
    dout = rng.standard_normal(B)
    return net, P, x, keep, dout


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("training", [True, False])
def test_restatement_backward_equals_autograd(name, training):
    C_ = 3 if name != "create_D16_b" else 1
    net, P, x, keep, dout = _case(name, C_, 3, seed=7)
    keep = keep if training else None
    out, dx, gP, _ = R.run(net, P, x, keep, dout)
    Pt = torch.tensor(P, requires_grad=True)
    xt = torch.tensor(x, requires_grad=True)
    c = R.Ctx(Pt, None if keep is None else torch.tensor(keep))
    o = torch.sigmoid(net.forward(c, xt))
    (o * torch.tensor(dout)).sum().backward()
    np.testing.assert_allclose(out, o.detach().numpy(), rtol=0, atol=0)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(gP, Pt.grad.numpy(), rtol=1e-10, atol=1e-14)
    # every parameter tensor gets a gradient (the dropout flags leave most of each tensor live)
    for pname, off, n in net.param_tensors():
        assert np.abs(gP[off:off + n]).max() > 0, pname


def test_keep_flags_are_in_module_order():
    """create_D16: fine SpatialDropout (64 planes), fine Dropout (1024), coarse SpatialDropout (64), coarse Dropout
    (1024), dense Dropout (1024), head Dropout (1024)"""
    net = R.Net("create_D16", 3)
    drops = [(m.moff, m.width, m.spatial) for _, mods, _ in net.branches for m in mods if isinstance(m, R.Dropout)]
    drops += [(m.moff, m.width, m.spatial) for m in net.head if isinstance(m, R.Dropout)]
    assert drops == [(0, 64, True), (64, 1024, False), (1088, 64, True), (1152, 1024, False), (2176, 1024, False),
                     (3200, 1024, False)]


def test_maxpool_takes_the_first_strict_maximum():
    win = torch.tensor([[1.0, 1.0, 0.5, 1.0], [0.0, 2.0, 2.0, 1.0], [-1.0, -1.0, -1.0, -1.0], [3.0, 1.0, 3.0, 3.0]])
    assert R.first_max(win).tolist() == [0, 1, 0, 0]
    x = torch.tensor([[[[1.0, 1.0], [1.0, 1.0]]]])
    m = R.MaxPool("t")
    c = R.Ctx(torch.zeros(1, dtype=torch.float64), None)
    assert m.fwd(c, x).item() == 1.0 and m.idx.item() == 0
    dx = m.bwd(c, torch.tensor([[[[5.0]]]]))
    assert dx.flatten().tolist() == [5.0, 0.0, 0.0, 0.0]


# ---- the counts of the models.lua layer shapes, written out by hand (weights + biases + one slope per PReLU) --------
def test_param_counts_from_the_layer_shapes_written_out():
    from face_generator_b200.lib import disc_param_count
    lin = lambda i, o: i * o + o + 1  # Linear + PReLU
    conv = lambda i, o, k: o * i * k * k + o + 1  # SpatialConvolution + PReLU
    for C in (1, 3):
        d32 = (conv(C, 64, 3) + conv(64, 64, 3) + lin(64 * 16 * 16, 1024)
               + conv(C, 32, 5) + conv(32, 32, 5) + conv(32, 54, 5) + conv(54, 54, 5) + lin(54 * 8 * 8, 1024)
               + lin(1024, 1024) + lin(C * 32 * 32, 1024) + lin(1024, 1024) + lin(3072, 1024) + 1024 + 1)
        d16 = (conv(C, 64, 3) + conv(64, 64, 3) + lin(64 * 8 * 8, 1024) + conv(C, 32, 5) + conv(32, 64, 5)
               + lin(64 * 8 * 8, 1024) + lin(C * 256, 1024) + lin(1024, 1024) + lin(3072, 1024) + 1024 + 1)
        d16b = (conv(C, 64, 3) + conv(64, 64, 3) + conv(64, 128, 3) + conv(128, 128, 3) + lin(128 * 8 * 8, 512)
                + conv(C, 64, 5) + conv(64, 64, 5) + conv(64, 128, 5) + conv(128, 128, 5) + lin(128 * 8 * 8, 512)
                + lin(C * 256, 1024) + lin(1024, 1024) + lin(2048, 1024) + 1024 + 1)
        d16c = (conv(C, 64, 3) + conv(64, 64, 3) + conv(64, 128, 3) + conv(128, 128, 3) + conv(128, 512, 3)
                + lin(512 * 4 * 4, 1024) + conv(C, 64, 5) + conv(64, 64, 5) + conv(64, 128, 5) + conv(128, 128, 5)
                + conv(128, 512, 5) + lin(512 * 4 * 4, 1024) + lin(C * 256, 1024) + lin(1024, 1024) + lin(3072, 1024)
                + 1024 + 1)
        for name, n in (("create_D32", d32), ("create_D16", d16), ("create_D16_b", d16b), ("create_D16_c", d16c)):
            assert disc_param_count(name, C) == n, (name, C)
    # the figures models.lua's shapes give for colour / grayscale
    assert [disc_param_count(n, 3) for n in NAMES] == [28894941, 13467914, 13308046, 24975504]
    assert [disc_param_count(n, 1) for n in NAMES] == [26795037, 12940874, 12779406, 24446864]


# ---- checkpoints: adversarial.net trees of each discriminator (independent Torch7 writer of tests/test_t7.py) -------
def disc_tree(name, C, P, T=None):
    """nn.Sequential{nn.Copy, nn.Sequential{nn.ConcatTable{branches}, nn.JoinTable, head}, nn.Copy} as the reference's
    CUDA-mode D is saved, every weight / bias a view into one flat storage P; T: the writer module (test_t7's)"""
    if T is None:
        import test_t7 as T
    Obj, Storage, Tensor, seq = T.Obj, T.Storage, T.Tensor, T.seq
    net = R.Net(name, C)
    st, gst = Storage(P, "torch.CudaStorage"), Storage(np.zeros_like(P), "torch.CudaStorage")
    view = lambda off, shape: Tensor(st, shape, offset=off, cls="torch.CudaTensor")

    def leaf(m):
        if isinstance(m, R.Conv):
            shape = (m.cout, m.cin, m.k, m.k)
            return Obj("nn.SpatialConvolution", {"weight": view(m.off, shape), "bias": view(m.off + m.n - m.cout, (m.cout,)),
                                                 "gradWeight": Tensor(gst, shape, offset=m.off), "train": True})
        if isinstance(m, R.Linear):
            return Obj("nn.Linear", {"weight": view(m.off, (m.fout, m.fin)), "bias": view(m.off + m.fout * m.fin, (m.fout,)),
                                     "train": True})
        if isinstance(m, R.PReLU):
            return Obj("nn.PReLU", {"weight": view(m.off, (1,)), "train": True})
        cls = {R.MaxPool: "nn.SpatialMaxPooling", R.View: "nn.View"}.get(type(m))
        if cls is None:
            cls = "nn.SpatialDropout" if m.spatial else "nn.Dropout"
        return Obj(cls, {"train": True})

    branches = [seq(*[leaf(m) for m in mods]) for _, mods, _ in net.branches]
    concat = Obj("nn.ConcatTable", {"modules": {i + 1: b for i, b in enumerate(branches)}, "train": True})
    inner = seq(concat, Obj("nn.JoinTable", {"dimension": 2}), *[leaf(m) for m in net.head], Obj("nn.Sigmoid", {}))
    copy = lambda a, b: Obj("nn.Copy", {"intype": a, "outtype": b, "train": True})
    return seq(copy("torch.FloatTensor", "torch.CudaTensor"), inner, copy("torch.CudaTensor", "torch.FloatTensor"))


def write_root(path, root, T=None):
    if T is None:
        import test_t7 as T
    w = T.W()
    w.obj(root)
    open(path, "wb").write(bytes(w.buf))


@pytest.mark.parametrize("name", NAMES)
def test_checkpoint_trees_are_recognised(tmp_path, name):
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200.checkpoint import T7File
    C_ = 3
    P = np.random.default_rng(4).standard_normal(R.Net(name, C_).n_params).astype(np.float32)
    p = tmp_path / "adversarial.net"
    write_root(p, {"D": disc_tree(name, C_, P), "epoch": 2})
    with T7File(p) as f:
        assert CK.recognise_disc(f.net_describe("D")) == name
        np.testing.assert_array_equal(f.net_params("D"), P)  # getParameters() order through the ConcatTable
        np.testing.assert_array_equal(CK._check_disc(f, name, C_, "this net"), P)
        for other in NAMES + ["create_D32b", "create_D16_d"]:
            if other != name:
                with pytest.raises(FGError, match="checkpoint D is %s; this net has %s" % (name, other)):
                    CK._check_disc(f, other, C_, "this net")
        with pytest.raises(FGError, match="parameters"):  # the right tree with the other channel count
            CK._check_disc(f, name, 1, "this net")


def test_default_trees_are_recognised(tmp_path):
    from face_generator_b200 import checkpoint as CK
    from face_generator_b200.checkpoint import T7File
    from test_t7 import write_reference_like
    p = tmp_path / "adversarial.net"
    write_reference_like(p, C=3)
    with T7File(p) as f:
        assert CK.recognise_disc(f.net_describe("D")) == "create_D32b"
        with pytest.raises(FGError, match="checkpoint D is create_D32b; this 32x32 net has create_D32"):
            CK._check_disc(f, "create_D32", 3, "this 32x32 net")


@pytest.mark.parametrize("name", ["create_D16", "create_D16_b", "create_D16_c"])
def test_s16_checkpoint_with_a_branched_D_loads_into_its_net_only(tmp_path, name):
    from face_generator_b200 import checkpoint as CK
    from oracle import oracle_s16 as O16
    import test_c2f_refine_cpu as T
    C_ = 1
    rng = np.random.default_rng(9)
    PG = rng.standard_normal(O16.G_param_count(C_)).astype(np.float32)
    PD = rng.standard_normal(R.Net(name, C_).n_params).astype(np.float32)
    t1 = lambda a: T.Tensor(T.Storage(np.ascontiguousarray(a, np.float32)), [a.size], cls="torch.CudaTensor")
    bn = [{"running_mean": t1(np.zeros(256)), "running_var": t1(np.ones(256))},
          {"running_mean": t1(np.zeros(128)), "running_var": t1(np.ones(128))}]
    p = tmp_path / "adversarial.net"
    write_root(p, {"G": T.cuda_net(PG, O16.G_layout(C_), T.S16_G_CLASSES, bn=bn), "D": disc_tree(name, C_, PD, T),
                   "epoch": 5}, T)
    ck = CK.read_s16_checkpoint(p, C_, name)
    np.testing.assert_array_equal(ck["PG"], PG)
    np.testing.assert_array_equal(ck["PD"], PD)
    assert ck["epoch"] == 5
    with pytest.raises(FGError, match="checkpoint D is %s; the --scale 16 D with 1 channels has create_D16_d" % name):
        CK.read_s16_checkpoint(p, C_)
