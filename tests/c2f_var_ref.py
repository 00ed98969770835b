"""Independent (test-only) float64 restatement of every coarse-to-fine net of models_c2f.lua, built from the layer
shapes written out below (not from the library's descriptor tables):

  G = JoinTable(2,2){noise[1][S][S], coarse[C][S][S]} -> "same" SpatialConvolutionUpsample(factor 1) layers, a one-slope
      PReLU after each but the last, which outputs C channels (View, no Sigmoid)
  D = CAddTable{diff, coarse} -> 3x3 "same" convolutions, each followed by a one-slope PReLU and some by a 2x2 max pool,
      then Dropout, View, Linear(512), PReLU, Dropout, Linear(1), Sigmoid

Parameters in getParameters() order: G [c1W c1b a1 ... cnW cnb], D [c1W c1b a1 ... L1W L1b a5 L2W L2b].  Keep flags
per sample: the last pooled map in NCHW order, then the 512 flags of the second Dropout.

Hooks as tests/torch_ref_c2f.py: branch(name, x) is torch_ref.prelu's PReLU branch hook ("z1".. for the convolutions,
"zl1" for the Linear), route(name, win) picks the element of every 2x2 max-pool window ("p<i>" after convolution i).
"""
import numpy as np
import torch
import torch.nn.functional as F

from torch_ref import _split, d_sigmoid, prelu
from torch_ref_c2f import maxpool2

# (Cout, k) after the C+1 joined planes; Cout 0 = the C image channels
G_LAYERS = {
    "create_G_d": [(64, 3), (64, 3), (128, 5), (256, 5), (0, 7)],  # models_c2f.lua:113-145
    "create_G_a": [(64, 3), (128, 7), (0, 5)],                      # models_c2f.lua:16-45
    "create_G_b": [(64, 3), (64, 3), (256, 5), (0, 7)],             # models_c2f.lua:47-78
    "create_G_c": [(64, 3), (128, 3), (256, 5), (0, 7)],            # models_c2f.lua:80-111
}
# 3x3 convolutions (Cout, 2x2 max pool after)
D_LAYERS = {
    "create_D_c": [(64, False), (64, True), (128, False), (256, True)],  # models_c2f.lua:237-278
    "create_D_a": [(64, False), (64, True)],                             # models_c2f.lua:156-192
    "create_D_b": [(64, False), (64, True), (128, False), (128, True)],  # models_c2f.lua:194-235
}
GENERATORS = list(G_LAYERS)
DISCRIMINATORS = list(D_LAYERS)
FINE_SIZES = (16, 32, 64)


def G_convs(name, C):
    """[(Cin, Cout, k)] of the generator's layers"""
    out, cin = [], C + 1
    for cout, k in G_LAYERS[name]:
        cout = cout or C
        out.append((cin, cout, k))
        cin = cout
    return out


def D_convs(name, C, S):
    """[(Cin, Cout, H, pool)] of the discriminator's convolutions, H = the side they run at"""
    out, cin, H = [], C, S
    for cout, pool in D_LAYERS[name]:
        out.append((cin, cout, H, pool))
        cin = cout
        H = H // 2 if pool else H
    return out


def D_view(name, S):
    """(channels, side) of the pooled map View flattens"""
    cin, cout, H, pool = D_convs(name, 1, S)[-1]
    return cout, H // 2


def G_layout(name, C):
    out, o = {}, 0
    convs = G_convs(name, C)
    for i, (cin, cout, k) in enumerate(convs):
        items = [("c%dW" % (i + 1), (cout, cin, k, k)), ("c%db" % (i + 1), (cout,))]
        if i < len(convs) - 1:
            items.append(("a%d" % (i + 1), (1,)))
        for key, shape in items:
            out[key] = (o, shape)
            o += int(np.prod(shape))
    return out


def D_layout(name, C, S):
    items = []
    for i, (cin, cout, _, _) in enumerate(D_convs(name, C, S)):
        items += [("c%dW" % (i + 1), (cout, cin, 3, 3)), ("c%db" % (i + 1), (cout,)), ("a%d" % (i + 1), (1,))]
    vc, vh = D_view(name, S)
    items += [("L1W", (512, vc * vh * vh)), ("L1b", (512,)), ("a%d" % (len(D_LAYERS[name]) + 1), (1,)),
              ("L2W", (1, 512)), ("L2b", (1,))]
    out, o = {}, 0
    for key, shape in items:
        out[key] = (o, shape)
        o += int(np.prod(shape))
    return out


def count(layout):
    return sum(int(np.prod(s)) for _, s in layout.values())


def mask_per_sample(name, S):
    vc, vh = D_view(name, S)
    return vc * vh * vh + 512


def G_forward(P, noise, cond, name, C=3, branch=None):
    p = _split(P, G_layout(name, C))
    x = torch.cat([noise, cond], dim=1)  # JoinTable(2,2): noise plane first
    convs = G_convs(name, C)
    for i, (_, _, k) in enumerate(convs):
        x = F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=k // 2)
        if i < len(convs) - 1:
            x = prelu(x, p["a%d" % (i + 1)], branch, "z%d" % (i + 1))
    return x


def D_forward(P, diff, cond, masks, name, C=3, S=32, branch=None, route=None):
    p = _split(P, D_layout(name, C, S))
    B = diff.shape[0]
    x = diff + cond  # CAddTable
    convs = D_convs(name, C, S)
    for i, (_, _, _, pool) in enumerate(convs):
        x = prelu(F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=1), p["a%d" % (i + 1)], branch,
                  "z%d" % (i + 1))
        if pool:
            x = maxpool2(x, route, "p%d" % (i + 1))
    n = x[0].numel()
    x = x.reshape(B, n) * masks[:, :n] * 2.0  # nn.Dropout p = 0.5 (v2), then View in (c,h,w) order
    a = p["a%d" % (len(convs) + 1)]
    h = prelu(F.linear(x, p["L1W"], p["L1b"]), a, branch, "zl1") * masks[:, n:] * 2.0
    return d_sigmoid(F.linear(h, p["L2W"], p["L2b"])).reshape(B)


def trained_like(layout, rng, gain=1.4):
    """He-style weights (activations stay O(1) through the PReLU stacks), slopes 0.25, small biases"""
    P = np.zeros(count(layout))
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        if k.startswith("a"):
            P[o] = 0.25
        elif k.endswith("W"):
            P[o:o + n] = rng.standard_normal(n) * (gain / np.sqrt(int(np.prod(s[1:]))))
        else:
            P[o:o + n] = rng.standard_normal(n) * 0.05
    return P


def make_case(B, C, S, generator, discriminator, seed):
    """one loop body's inputs for the pair: float32 arrays, D's inputs for B samples (B/2 real pairs)"""
    rng = np.random.default_rng(seed)
    Bh = B // 2
    fine = rng.random((2 * B, C, S, S))  # rows [0, B/2): real pairs, [B/2, B): the fakes' condition, [B, 2B): G's
    small = fine.reshape(-1, C, S // 2, 2, S // 2, 2).mean(axis=(3, 5))
    coarse = np.repeat(np.repeat(small, 2, axis=2), 2, axis=3)
    diff = fine - coarse
    m = mask_per_sample(discriminator, S)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(
        PG=f(trained_like(G_layout(generator, C), rng)), PD=f(trained_like(D_layout(discriminator, C, S), rng, 1.0)),
        real_diff=f(diff[:Bh]), cond_D=f(coarse[:B]),
        noise_D=f(rng.uniform(-1, 1, (Bh, 1, S, S))), cond_G=f(coarse[B:]),
        noise_G=f(rng.uniform(-1, 1, (B, 1, S, S))),
        masks_D=f(rng.random((B, m)) < 0.5), masks_G=f(rng.random((B, m)) < 0.5))
