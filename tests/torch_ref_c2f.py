"""Independent (test-only) PyTorch fp64 restatement of the coarse-to-fine nets
(models_c2f.lua:113-145 create_G_d, :237-278 create_D_c).  tests/test_oracle_c2f_vs_torch.py pins it to
oracle/fg_oracle_c2f.h on the CPU; tests/test_gpu_c2f_s16_headline.py holds the CUDA path to it on the GPU.

Hooks for the comparison at the BASELINE batch size: branch is torch_ref.prelu's PReLU branch hook (names "z1".."z4" in
G and D, "zl1" for D's Linear); route(name, win) picks the element of every 2x2 max-pool window (names "p2", "p4"):
win [B][C][H/2][W/2][4] holds the window in row-major order, the hook returns the index (int64, same shape minus the
last axis) of the element taken."""
import numpy as np
import torch
import torch.nn.functional as F

from torch_ref import d_sigmoid

from oracle import oracle_c2f as OC
from torch_ref import _split, prelu


def maxpool2(x, route=None, name=None):
    if route is None:
        return F.max_pool2d(x, 2, 2)
    B, Cc, H, W = x.shape
    win = x.reshape(B, Cc, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, Cc, H // 2, W // 2, 4)
    return win.gather(-1, route(name, win.detach()).unsqueeze(-1)).squeeze(-1)


def G_forward(P, noise, cond, C=3, branch=None):
    p = _split(P, OC.G_layout(C))
    x = torch.cat([noise, cond], dim=1)  # JoinTable(2,2): noise plane first
    pads = [1, 1, 2, 2, 3]
    for i in range(5):
        x = F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=pads[i])
        if i < 4:
            x = prelu(x, p["a%d" % (i + 1)], branch, "z%d" % (i + 1))
    return x


def D_forward(P, diff, cond, masks, C=3, branch=None, route=None):
    p = _split(P, OC.D_layout(C))
    B = diff.shape[0]
    x = diff + cond  # CAddTable
    for i in range(4):
        x = prelu(F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=1), p["a%d" % (i + 1)], branch,
                  "z%d" % (i + 1))
        if i in (1, 3):
            x = maxpool2(x, route, "p%d" % (i + 1))
    x = x.reshape(B, 16384) * masks[:, :16384] * 2.0  # nn.Dropout p=0.5 (v2), then View in (c,h,w) order
    h = prelu(F.linear(x, p["L1W"], p["L1b"]), p["a5"], branch, "zl1") * masks[:, 16384:] * 2.0
    return d_sigmoid(F.linear(h, p["L2W"], p["L2b"])).reshape(B)


def trained_like(layout, count, rng, gain=1.4):
    """He-style weights (activations stay O(1) through the PReLU stacks), slopes 0.25, small biases."""
    P = np.zeros(count)
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        if k.startswith("a"):
            P[o] = 0.25
        elif k.endswith("W"):
            P[o:o + n] = rng.standard_normal(n) * (gain / np.sqrt(int(np.prod(s[1:]))))
        else:
            P[o:o + n] = rng.standard_normal(n) * 0.05
    return P


def trained_like_G(C, rng):
    return trained_like(OC.G_layout(C), OC.G_param_count(C), rng)


def trained_like_D(C, rng):
    return trained_like(OC.D_layout(C), OC.D_param_count(C), rng)


def make_masks(B, rng):
    return (rng.random((B, OC.MASK_PER_SAMPLE)) < 0.5).astype(np.float64)


def make_pairs(B, C, rng):
    """Stand-in for dataset_c2f.lua:54-60: fine ~ U[0,1), coarse = 2x avg-down then 2x nearest-up, diff = fine - coarse."""
    fine = rng.random((B, C, 32, 32))
    small = fine.reshape(B, C, 16, 2, 16, 2).mean(axis=(3, 5))
    coarse = np.repeat(np.repeat(small, 2, axis=2), 2, axis=3)
    return fine - coarse, coarse
