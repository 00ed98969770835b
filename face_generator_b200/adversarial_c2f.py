"""Host-side mirror of adversarial_c2f.lua's loop body (adversarial_c2f.lua:121-187).

train_batch()          the fused call (fg_c2f_train_step): what lua/adversarial_c2f_b200.lua uses.
train_batch_modules()  the same iteration composed from MODEL_G / MODEL_D forward/backward calls in the order of
                       the reference's fevalD / fevalG_on_D closures (:40-116), to show the two levels agree.
train_batch_iters()    --D_iterations / --G_iterations: several D and G iterations in one fused call
train_batch_iters_modules()  the same iterations composed from the L-net calls and optim.adam steps
"""
import numpy as np

from .lib import C2f, NET_D, NET_G, _check


def create_noise_inputs(n, rng, fine_size=32):
    """noiseInputs:uniform(-1, 1) over NOISE_DIM = {1, fineSize, fineSize} (train_c2f.lua:80, adversarial_c2f.lua:135)."""
    return rng.uniform(-1.0, 1.0, (n, 1, fine_size, fine_size)).astype(np.float32)


def train_batch(net: C2f, hyper, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D=None, masks_G=None, seed=0,
                want_stats=True):
    B = cond_D.shape[0]
    return net.train_step(hyper, B, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D, masks_G, seed, want_stats)


def train_batch_iters(net: C2f, hyper, real_diffs, cond_Ds, noise_Ds, cond_Gs, noise_Gs, masks_D=None, masks_G=None,
                      seed=0, want_stats=True):
    """train_c2f.lua --D_iterations d / --G_iterations g: the train_batch inputs of every iteration stacked along a
    leading axis (real_diffs, cond_Ds, noise_Ds: d entries; cond_Gs, noise_Gs: g entries), one fused call
    (fg_c2f_train_step_iters)."""
    real_diffs, cond_Ds, noise_Ds, cond_Gs, noise_Gs = (np.ascontiguousarray(a, np.float32) for a in
                                                        (real_diffs, cond_Ds, noise_Ds, cond_Gs, noise_Gs))
    d, g, B = cond_Ds.shape[0], cond_Gs.shape[0], cond_Ds.shape[1]
    return net.train_step_iters(hyper, B, d, g, real_diffs, cond_Ds, noise_Ds, cond_Gs, noise_Gs, masks_D, masks_G, seed,
                                want_stats)


def _bce(ctx, outputs, targets):
    return ctx.bce_forward(outputs, targets), ctx.bce_backward(outputs, targets)


def train_batch_modules(net: C2f, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D, masks_G):
    """Gradients of one iteration WITHOUT the optimizer updates of G (D is not updated either): returns the raw
    accumulated gradients of the D step and of a G step taken against the *same* D parameters."""
    ctx = net.ctx
    Bh = real_diff.shape[0]
    B = 2 * Bh
    out = {}
    # ---- fevalD (:40-81) on [real | generated] ----
    fake = net.G_forward(noise_D, cond_D[Bh:])
    inputs = np.concatenate([real_diff, fake]).astype(np.float32)
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)]).astype(np.float32)
    net.zero_grads(NET_D)
    outputs = net.D_forward(inputs, cond_D, masks=masks_D)
    out["loss_D_bce"], df = _bce(ctx, outputs, targets)
    net.D_backward(df, want_wgrad=True, want_ddiff=False)
    out["grad_D"] = net.get_grads(NET_D)
    out["outputs_D"] = outputs
    # ---- fevalG_on_D (:85-116) ----
    net.zero_grads(NET_G)
    samples = net.G_forward(noise_G, cond_G)
    outputs = net.D_forward(samples, cond_G, masks=masks_G)
    out["loss_G"], df = _bce(ctx, outputs, np.ones(B, np.float32))
    ddiff = net.D_backward(df, want_wgrad=False, want_ddiff=True)
    net.G_backward(ddiff)
    out["grad_G"] = net.get_grads(NET_G)
    return out


class AdamState:
    """optim.adam's state for one net of a C2f / S16 pair in device memory (m, v, t), stepped with fg_adam_step on the
    net's own parameter and gradient buffers: the optimizer of the L-net compositions below.  penalty -> clamp -> Adam
    take the arguments the fused step gives them (adversarial_c2f.lua:95-110, incl. the G_L2 quirk)."""

    def __init__(self, pair, net):
        self.pair, self.net, self.n, self.t = pair, net, pair.count(net), 0
        ctx = pair.ctx
        self.m, self.v = ctx.dev_array(np.zeros(self.n, np.float32)), ctx.dev_array(np.zeros(self.n, np.float32))

    def step(self, hyper):
        isD = self.net == NET_D
        l1, l2 = (hyper.D_L1, hyper.D_L2) if isD else (hyper.G_L1, hyper.G_L2)
        pen = l1 != 0 or l2 != 0
        l1_grad = 0.0 if not pen else (l1 if isD else l2)
        self.t += 1
        lib, pre = self.pair.lib, self.pair._prefix
        p, g = getattr(lib, pre + "params_ptr")(self.pair.h, self.net), getattr(lib, pre + "grads_ptr")(self.pair.h, self.net)
        _check(lib.fg_adam_step(self.pair.ctx.h, p, g, self.m, self.v, self.n, hyper.lr_D if isD else hyper.lr_G, hyper.beta1,
                                hyper.beta2, hyper.eps, self.t, l1_grad, l2 if pen else 0.0,
                                hyper.D_clamp if isD else hyper.G_clamp, 1.0), "fg_adam_step")
        # fg_adam_step wrote the parameters behind the library's back: hand them over again, which marks the net's
        # weight packs stale, or the next forward would run on the packs of the old parameters
        self.pair.set_params(self.net, self.pair.get_params(self.net))

    def close(self):
        self.pair.ctx.dev_free(self.m)
        self.pair.ctx.dev_free(self.v)


def train_batch_iters_modules(net: C2f, hyper, real_diffs, cond_Ds, noise_Ds, cond_Gs, noise_Gs, masks_D, masks_G):
    """train_batch_iters composed from MODEL_G / MODEL_D forward/backward calls and optim.adam steps: len(cond_Ds) D
    iterations (:121-163), then len(cond_Gs) G iterations (:167-187), each with its own inputs and masks, each
    followed by its optimizer step.  The c2f loop has no accuracy gate.  Returns the per-iteration losses."""
    ctx = net.ctx
    Bh = real_diffs.shape[1]
    B = 2 * Bh
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)]).astype(np.float32)
    opt = {k: AdamState(net, k) for k in (NET_D, NET_G)}
    out = {"loss_D": [], "loss_G": []}
    for j in range(len(cond_Ds)):
        fake = net.G_forward(noise_Ds[j], cond_Ds[j][Bh:])
        net.zero_grads(NET_D)
        outputs = net.D_forward(np.concatenate([real_diffs[j], fake]), cond_Ds[j], masks=masks_D[j])
        f, df = _bce(ctx, outputs, targets)
        net.D_backward(df, want_wgrad=True, want_ddiff=False)
        opt[NET_D].step(hyper)
        out["loss_D"].append(f)
    for j in range(len(cond_Gs)):
        net.zero_grads(NET_G)
        samples = net.G_forward(noise_Gs[j], cond_Gs[j])
        outputs = net.D_forward(samples, cond_Gs[j], masks=masks_G[j])
        f, df = _bce(ctx, outputs, np.ones(B, np.float32))
        net.G_backward(net.D_backward(df, want_wgrad=False, want_ddiff=True))
        opt[NET_G].step(hyper)
        out["loss_G"].append(f)
    for o in opt.values():
        o.close()
    return out
