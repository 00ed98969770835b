"""Flat parameter layouts (getParameters() order) and synthetic initialisations, numpy only.

G: models.lua:57-81, D: models.lua:382-416; init: utils/nn_utils.lua:17-29 via train.lua:137-138."""
import numpy as np


def G_layout(c):
    out, o = {}, 0
    for name, shape in [("L1W", (8192, 100)), ("L1b", (8192,)), ("a1", (1,)), ("C1W", (256, 128, 5, 5)),
                        ("C1b", (256,)), ("g1", (256,)), ("be1", (256,)), ("a2", (1,)), ("C2W", (128, 256, 5, 5)),
                        ("C2b", (128,)), ("g2", (128,)), ("be2", (128,)), ("a3", (1,)), ("C3W", (c, 128, 3, 3)),
                        ("C3b", (c,))]:
        out[name] = (o, shape)
        o += int(np.prod(shape))
    return out, o


def D_layout(c):
    out, o = {}, 0
    cin, cout = [c, 64, 128, 256], [64, 128, 256, 512]
    items = []
    for i in range(4):
        items += [("c%dW" % (i + 1), (cout[i], cin[i], 3, 3)), ("c%db" % (i + 1), (cout[i],)), ("a%d" % (i + 1), (1,))]
    items += [("L1W", (512, 2048)), ("L1b", (512,)), ("a5", (1,)), ("L2W", (512, 512)), ("L2b", (512,)),
              ("a6", (1,)), ("L3W", (1, 512)), ("L3b", (1,))]
    for name, shape in items:
        out[name] = (o, shape)
        o += int(np.prod(shape))
    return out, o


def reference_init(layout_total, rng):
    """NN_UTILS.initializeWeights: every `.weight` ~ N(0, 0.005^2), every `.bias` ~ N(0, 0.001^2) --
    including BN gamma (a weight), BN beta (a bias) and the PReLU slopes (weights)."""
    layout, total = layout_total
    P = np.empty(total, np.float32)
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        is_bias = k.endswith("b") or k.startswith("be")
        P[o:o + n] = rng.standard_normal(n) * (0.001 if is_bias else 0.005)
    return P


def trained_like_init(layout_total, rng, gain=1.0, slope=0.25):
    """Non-degenerate synthetic weights (fan-in scaled, gamma~U(0.5,1.5), slopes 0.25) so activations,
    BatchNorm statistics and gradients look like a network in training (SURVEY.md 8d, config 2)."""
    layout, total = layout_total
    P = np.empty(total, np.float32)
    for k, (o, s) in layout.items():
        n = int(np.prod(s))
        if k[0] == "a":
            P[o:o + n] = slope
        elif k in ("g1", "g2"):
            P[o:o + n] = rng.uniform(0.5, 1.5, n)
        elif k.endswith("W"):
            P[o:o + n] = rng.standard_normal(n) * (gain / np.sqrt(np.prod(s[1:])))
        else:
            P[o:o + n] = rng.standard_normal(n) * 0.05
    return P


def c2f_G_layout(c):
    """create_G_d (models_c2f.lua:113-145): 5 SpatialConvolutionUpsample(factor 1) with 4 shared-slope PReLUs."""
    cin, cout, k = [c + 1, 64, 64, 128, 256], [64, 64, 128, 256, c], [3, 3, 5, 5, 7]
    out, o = {}, 0
    for i in range(5):
        items = [("c%dW" % (i + 1), (cout[i], cin[i], k[i], k[i])), ("c%db" % (i + 1), (cout[i],))]
        if i < 4:
            items.append(("a%d" % (i + 1), (1,)))
        for name, shape in items:
            out[name] = (o, shape)
            o += int(np.prod(shape))
    return out, o


def c2f_D_layout(c, fine_size=32):
    """create_D_c (models_c2f.lua:237-278) at fine size S: the Linear reads View(256*(S/4)^2)."""
    cin, cout = [c, 64, 64, 128], [64, 64, 128, 256]
    items = []
    for i in range(4):
        items += [("c%dW" % (i + 1), (cout[i], cin[i], 3, 3)), ("c%db" % (i + 1), (cout[i],)), ("a%d" % (i + 1), (1,))]
    items += [("L1W", (512, 256 * (fine_size // 4) ** 2)), ("L1b", (512,)), ("a5", (1,)), ("L2W", (1, 512)), ("L2b", (1,))]
    out, o = {}, 0
    for name, shape in items:
        out[name] = (o, shape)
        o += int(np.prod(shape))
    return out, o


def c2f_pairs(B, c, rng, fine_size=32):
    """Synthetic stand-in for dataset_c2f.lua:54-60: fine ~ U[0,1), coarse = 2x average-down then 2x nearest-up,
    diff = fine - coarse.  Returns (diff, coarse), both [B][c][S][S] float32 (S = fine_size)."""
    S = fine_size
    fine = rng.random((B, c, S, S))
    small = fine.reshape(B, c, S // 2, 2, S // 2, 2).mean(axis=(3, 5))
    coarse = np.repeat(np.repeat(small, 2, axis=2), 2, axis=3)
    return (fine - coarse).astype(np.float32), coarse.astype(np.float32)
