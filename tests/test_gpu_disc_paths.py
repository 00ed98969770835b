"""GPU: the serial step off the default numeric path against float64.

test_gpu_disc_variants.py holds create_D32, create_D16, create_D16_b and create_D16_c to the float64 restatement
(tests/dbr_ref.py) on the default 3xFP16 tensor-core operands, and test_gpu_headline.py the 32x32 G at the headline
batch.  The same checks run here on contexts switched to
  mma_f16 = 0    3xTF32 operands: the producer kernels write the operand split themselves (the BatchNorm-backward
                 kernels into G's dz split, k_bn_prelu_bwd_apply),
  conv_impl = 0  the fp32 FFMA kernels, whose weight gradients reduce split-K partials in splitk_ws / small_ws.
The discriminators' forward and backward check also takes the GPU's branch at every PReLU pre-activation within
rounding of 0 (KinkPReLU), as test_gpu_headline.py does for G: another operand rounding flips other kinks.
conv_impl = 1 (dense forward pack) differs from the default only in G's upsampled layers (upsl_pack / upsl_fwd,
convl.cu); a discriminator's layers see it only as "not the 3xFP16 split" (tc_f16), which is the mma_f16 = 0 path.
"""
import numpy as np
import pytest
import torch

import dbr_ref as R
import parity_utils as PU

pytestmark = pytest.mark.gpu

NAMES = ["create_D32", "create_D16", "create_D16_b", "create_D16_c"]
PATHS = [("mma_f16", 0), ("conv_impl", 0)]


@pytest.fixture
def disc_checks(monkeypatch):
    """disc_checks(opt, val): test_gpu_disc_variants, its contexts made with option opt = val"""
    import test_gpu_disc_variants as DV

    def on_path(opt, val):
        make = DV.make

        def make_on_path(name, C_, max_batch):
            ctx, net = make(name, C_, max_batch)
            ctx.set_option(opt, val)
            assert ctx.get_option(opt) == val
            return ctx, net
        monkeypatch.setattr(DV, "make", make_on_path)
        return DV
    return on_path


class KinkPReLU(R.PReLU):
    """R.PReLU that takes the GPU's branch where the float64 pre-activation lies within PU.KINK_MARGIN of 0 (relative
    to the layer's largest): there the two decisions differ by rounding alone.  With the slopes of R.make_params
    (1 - k 1e-3) a flip moves one dz by about 1e-3 |dY|; a Linear whose dY is a slice of the joint gradient adds a few
    such moves into one bias entry and one weight row, up to a few 1e-4 of the gradient's largest entry at batch 256.
    zget(name): the GPU's pre-activation, flat NHWC (the "D.*" debug tensor of the last D forward)."""

    def __init__(self, m, zname, zget, counts):
        self.off, self.n = m.off, m.n
        self.zname, self.zget, self.counts = zname, zget, counts

    def fwd(self, c, x):
        self.x = x
        z = x.detach()
        amb = z.abs() < PU.KINK_MARGIN * z.abs().max()
        self.pos = z > 0
        n = int(amb.sum())
        self.counts[self.zname] = n
        assert n <= max(8, PU.KINK_MAX_FRAC * z.numel()), (self.zname, n, z.numel())
        if n:
            g = torch.from_numpy(self.zget(self.zname)[:z.numel()].astype(np.float64))
            g = g.reshape(z.shape[0], *z.shape[2:], z.shape[1]).permute(0, 3, 1, 2) if z.dim() == 4 else g.reshape(z.shape)
            self.pos = torch.where(amb, g > 0, self.pos)
        return torch.where(self.pos, x, c.P[self.off] * x)

    def bwd(self, c, dy):
        x, a = self.x.detach(), c.P[self.off].detach()
        t = (dy * x)[~self.pos]
        c.acc(self.off, t.sum().reshape(1))
        c.gabs[self.off] = c.gabs.get(self.off, 0.0) + float(t.abs().sum())
        return torch.where(self.pos, dy, a * dy)


def kink_net(name, C_, zget, counts):
    """R.Net with every PReLU a KinkPReLU reading the GPU pre-activation of the same layer: "D.<branch>.z<i>" behind
    conv i, "D.<branch>.zl<j>" behind Linear j, "D.head.z" in the head"""
    ref = R.Net(name, C_)
    for bname, mods in [(b, m) for b, m, _ in ref.branches] + [("head", ref.head)]:
        nc = nl = 0
        for k, m in enumerate(mods):
            nc += isinstance(m, R.Conv)
            nl += isinstance(m, R.Linear)
            if isinstance(m, R.PReLU):
                zn = "D.head.z" if bname == "head" else \
                    "D.%s.%s" % (bname, "z%d" % nc if isinstance(mods[k - 1], R.Conv) else "zl%d" % nl)
                mods[k] = KinkPReLU(m, zn, zget, counts)
    return ref


@pytest.mark.parametrize("opt,val", PATHS)
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("C_", [1, 3])
@pytest.mark.parametrize("B", [6, 256])
def test_disc_forward_backward_off_the_default_path_against_float64(opt, val, name, C_, B):
    """forward (eval and training), input gradient and every parameter gradient at the 1e-4 bar of
    test_gpu_disc_forward_backward_against_float64, with the GPU's own decisions where the float64 ones differ by
    rounding alone: max-pool windows whose top two candidates tie, and PReLU pre-activations at 0"""
    import test_gpu_disc_variants as DV
    ctx, net = DV.make(name, C_, 256)
    try:
        ctx.set_option(opt, val)
        assert ctx.get_option(opt) == val
        counts = {}
        ref = kink_net(name, C_, lambda n: net.debug_tensor(n), counts)
        assert net.nD == ref.n_params and net.mask_per_sample == ref.mask
        rng = np.random.default_rng(B * 10 + C_)
        P = R.make_params(ref, 11 + C_)
        net.set_params(1, P.astype(np.float32))
        net.set_params(0, rng.uniform(-0.05, 0.05, net.nG).astype(np.float32))
        x = rng.uniform(0, 1, (B, C_, ref.side, ref.side)).astype(np.float32)
        keep = (rng.uniform(0, 1, (B, ref.mask)) >= 0.5).astype(np.float32)
        dout = rng.standard_normal(B).astype(np.float32)

        def routed():
            route, offs = DV.gpu_route(net, P)
            offs.update(DV.pool_slopes(ref))
            return route
        out_e = net.D_forward(x, training=False)
        ref_e = R.run(ref, P, x, None, route=routed())[0]
        assert DV.relerr(out_e, ref_e) < DV.BAR
        net.zero_grads(1)
        out = net.D_forward(x, masks=keep, training=True)
        dx = net.D_backward(dout, want_wgrad=True, want_dimages=True) if net is ctx else \
            net.D_backward(dout, want_wgrad=True, want_dimg=True)
        g = net.get_grads(1)
        route = routed()
        ref_out, ref_dx, ref_g, rc = R.run(ref, P, x, keep, dout, route=route)
    finally:
        DV.close(ctx, net)
    errs = {"out": DV.relerr(out, ref_out), "dx": DV.relerr(dx, ref_dx)}
    for pname, off, n in ref.param_tensors():
        if pname.endswith(".a"):  # one sum of signed terms, whose rounding scales with the sum of their sizes
            errs[pname] = abs(float(g[off]) - ref_g[off]) / max(abs(ref_g[off]), rc.gabs[off], 1e-30)
        else:
            errs[pname] = DV.relerr(g[off:off + n], ref_g[off:off + n])
    bad = {k: v for k, v in errs.items() if not v < DV.BAR}
    assert not bad, (bad, route.count, {k: v for k, v in counts.items() if v})


@pytest.mark.parametrize("name", NAMES)
def test_disc_train_step_on_tf32_against_float64(disc_checks, name):
    """one fused train_step_iters (1, 1) on 3xTF32 operands against the float64 loop body: confusion counts, both
    nets' Adam moments and parameters"""
    disc_checks("mma_f16", 0).test_gpu_disc_train_step_iters_against_float64(name, 1, 1)


class _TF32:
    """the package, with every Context made on 3xTF32 operands"""

    def __init__(self, fg):
        self.fg = fg

    def Context(self, *args, **kw):
        ctx = self.fg.Context(*args, **kw)
        ctx.set_option("mma_f16", 0)
        assert ctx.get_option("mma_f16") == 0
        return ctx


@pytest.mark.parametrize("B", [256, 130])
def test_G_on_tf32_at_headline_batch(B):
    """the 32x32 G's forward and backward on 3xTF32 operands: every forward launch on its own input at 1e-5, outputs,
    noise and parameter gradients at 1e-4, and the backward's tensor-core launches on the split dz that the
    BatchNorm-backward kernels wrote"""
    import face_generator_b200 as fg
    import test_gpu_headline as TH
    TH._G_at_headline_batch(_TF32(fg), B, 2)
