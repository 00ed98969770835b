"""Host-side mirror of adversarial_c2f.lua's loop body (adversarial_c2f.lua:121-187).

train_batch()          the fused call (fg_c2f_train_step): what lua/adversarial_c2f_b200.lua uses.
train_batch_modules()  the same iteration composed from MODEL_G / MODEL_D forward/backward calls in the order of
                       the reference's fevalD / fevalG_on_D closures (:40-116), to show the two levels agree.
"""
import numpy as np

from .lib import C2f, NET_D, NET_G


def create_noise_inputs(n, rng, fine_size=32):
    """noiseInputs:uniform(-1, 1) over NOISE_DIM = {1, fineSize, fineSize} (train_c2f.lua:80, adversarial_c2f.lua:135)."""
    return rng.uniform(-1.0, 1.0, (n, 1, fine_size, fine_size)).astype(np.float32)


def train_batch(net: C2f, hyper, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D=None, masks_G=None, seed=0,
                want_stats=True):
    B = cond_D.shape[0]
    return net.train_step(hyper, B, real_diff, cond_D, noise_D, cond_G, noise_G, masks_D, masks_G, seed, want_stats)


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
