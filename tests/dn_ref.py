"""float64 restatement of train_denoiser.lua's decoders and batch step (numpy, forward and hand-written backward), the
reference the GPU denoiser is checked against.  Layouts: images NCHW [B][C][S][S]; keep flags [B][mps] with the conv
block's 8(S-4)^2 flags first ([8][S-4][S-4] order), then 2048; flat parameters in getParameters() order; BatchNorm
state [mean1 8][var1 8][mean2 8][var2 8][mean3 2048][var3 2048]."""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

SLOPE = 0.333
HIDDEN = 2048
BN_EPS = 1e-5
BCE_EPS = 1e-12


def shapes(C, S):
    A, O = 8 * (S - 4) ** 2, C * S * S
    return [("c1W", (8, C, 3, 3)), ("c1b", (8,)), ("g1", (8,)), ("b1", (8,)), ("c2W", (8, 8, 3, 3)), ("c2b", (8,)),
            ("g2", (8,)), ("b2", (8,)), ("L1W", (HIDDEN, A)), ("L1b", (HIDDEN,)), ("g3", (HIDDEN,)), ("b3", (HIDDEN,)),
            ("L2W", (O, HIDDEN)), ("L2b", (O,))]


def param_count(C, S):
    return sum(int(np.prod(s)) for _, s in shapes(C, S))


def mask_per_sample(S):
    return 8 * (S - 4) ** 2 + HIDDEN


def unflat(P, C, S):
    out, o = {}, 0
    for name, shape in shapes(C, S):
        n = int(np.prod(shape))
        out[name] = np.asarray(P[o:o + n], np.float64).reshape(shape)
        o += n
    return out


def flat(d, C, S):
    return np.concatenate([d[name].ravel() for name, _ in shapes(C, S)])


def bn_init():
    s = np.zeros(2 * (16 + HIDDEN))
    s[8:16] = 1
    s[24:32] = 1
    s[32 + HIDDEN:] = 1
    return s


def _bn_slices(l):
    if l < 2:
        return slice(16 * l, 16 * l + 8), slice(16 * l + 8, 16 * l + 16)
    return slice(32, 32 + HIDDEN), slice(32 + HIDDEN, 32 + 2 * HIDDEN)


def conv_valid(x, W, b):  # x [B][Ci][H][H], W [8][Ci][3][3] -> [B][8][H-2][H-2]
    win = sliding_window_view(x, (3, 3), axis=(2, 3))  # [B][Ci][Ho][Ho][3][3]
    return np.einsum("bcyxkl,ockl->boyx", win, W, optimize=True) + b[None, :, None, None]


def conv_wgrad(x, dz):
    win = sliding_window_view(x, (3, 3), axis=(2, 3))
    return np.einsum("bcyxkl,boyx->ockl", win, dz, optimize=True), dz.sum(axis=(0, 2, 3))


def conv_dgrad(dz, W):  # the transposed valid convolution
    B, O, Ho, _ = dz.shape
    pad = np.pad(dz, ((0, 0), (0, 0), (2, 2), (2, 2)))
    win = sliding_window_view(pad, (3, 3), axis=(2, 3))  # [B][O][Ho+2][Ho+2][3][3]
    return np.einsum("boyxkl,ockl->bcyx", win, W[:, :, ::-1, ::-1], optimize=True)


def _stat_axes(z):
    return (0, 2, 3) if z.ndim == 4 else (0,)


def _bc(v, z):
    return v[None, :, None, None] if z.ndim == 4 else v[None, :]


def bn_act_fwd(z, g, b, state, l, training, mask, scale, kinks=None):
    """BatchNorm (nn.(Spatial)BatchNormalization, eps 1e-5, momentum 0.1) -> LeakyReLU(0.333) -> Dropout (mask: keep
    flags shaped like z, None = none).  Updates `state` in training.  kinks (optional): callable(l, u) -> (flat indices,
    branches) forcing LeakyReLU's gradient branch (u >= 0) of those elements in the backward -- the elements within
    rounding of the kink, where another correct implementation may take the other branch."""
    sm, sv = _bn_slices(l)
    ax = _stat_axes(z)
    if training:
        n = z.size // z.shape[1]
        mean, var = z.mean(axis=ax), z.var(axis=ax)
        state[sm] = 0.9 * state[sm] + 0.1 * mean
        state[sv] = 0.9 * state[sv] + 0.1 * var * n / (n - 1)
    else:
        mean, var = state[sm].copy(), state[sv].copy()
    istd = 1.0 / np.sqrt(var + BN_EPS)
    xh = (z - _bc(mean, z)) * _bc(istd, z)
    u = _bc(g, z) * xh + _bc(b, z)
    h = np.where(u > 0, u, SLOPE * u)
    if mask is not None:
        h = h * mask * scale
    pos = u >= 0
    if kinks is not None:
        idx, branch = kinks(l, u)
        pos.flat[idx] = branch
    return h, dict(xh=xh, u=u, pos=pos, istd=istd, mask=mask, training=training)


def bn_act_bwd(dh, g, cache, scale):
    """-> dz, dgamma, dbeta.  LeakyReLU's gradient is the waifu2x rule: slope 1 at u >= 0."""
    d = dh * cache["mask"] * scale if cache["mask"] is not None else dh
    gg = np.where(cache["pos"], d, SLOPE * d)
    xh, ax = cache["xh"], _stat_axes(dh)
    dgamma, dbeta = (gg * xh).sum(axis=ax), gg.sum(axis=ax)
    k = _bc(g * cache["istd"], dh)
    if cache["training"]:
        n = dh.size // dh.shape[1]
        dz = k * (gg - _bc(dbeta / n, dh) - xh * _bc(dgamma / n, dh))
    else:
        dz = k * gg
    return dz, dgamma, dbeta


def decoder_forward(P, x, state, training, masks, C, S, p_drop=0.2, kinks=None):
    """x [B][C][S][S] (after WhiteNoise) -> logits [B][C S S] and the cache of the backward.  masks [B][mps] or None."""
    W = unflat(P, C, S)
    B, A2 = x.shape[0], (S - 4) ** 2
    scale = 1.0 / (1.0 - p_drop)
    m2 = m3 = None
    if training and masks is not None:
        masks = np.asarray(masks, np.float64)
        m2 = masks[:, :8 * A2].reshape(B, 8, S - 4, S - 4)
        m3 = masks[:, 8 * A2:]
    z1 = conv_valid(x, W["c1W"], W["c1b"])
    h1, k1 = bn_act_fwd(z1, W["g1"], W["b1"], state, 0, training, None, 1.0, kinks)
    z2 = conv_valid(h1, W["c2W"], W["c2b"])
    h2, k2 = bn_act_fwd(z2, W["g2"], W["b2"], state, 1, training, m2, scale, kinks)
    h2f = h2.reshape(B, -1)
    z3 = h2f @ W["L1W"].T + W["L1b"]
    h3, k3 = bn_act_fwd(z3, W["g3"], W["b3"], state, 2, training, m3, scale, kinks)
    z4 = h3 @ W["L2W"].T + W["L2b"]
    return z4, dict(W=W, x=x, h1=h1, h2=h2, h2f=h2f, h3=h3, k=(k1, k2, k3), scale=scale)


def decoder_backward(cache, dz4, C, S):
    """dz4: gradient at the logits [B][C S S] -> flat parameter gradient"""
    W, sc = cache["W"], cache["scale"]
    k1, k2, k3 = cache["k"]
    G = {}
    G["L2W"], G["L2b"] = dz4.T @ cache["h3"], dz4.sum(0)
    dh3 = dz4 @ W["L2W"]
    dz3, G["g3"], G["b3"] = bn_act_bwd(dh3, W["g3"], k3, sc)
    G["L1W"], G["L1b"] = dz3.T @ cache["h2f"], dz3.sum(0)
    dh2 = (dz3 @ W["L1W"]).reshape(cache["h2"].shape)
    dz2, G["g2"], G["b2"] = bn_act_bwd(dh2, W["g2"], k2, sc)
    G["c2W"], G["c2b"] = conv_wgrad(cache["h1"], dz2)
    dh1 = conv_dgrad(dz2, W["c2W"])
    dz1, G["g1"], G["b1"] = bn_act_bwd(dh1, W["g1"], k1, 1.0)
    G["c1W"], G["c1b"] = conv_wgrad(cache["x"], dz1)
    return flat(G, C, S)


def sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def bce(y, t):
    """the 2015 Lua nn.BCECriterion (size-averaged) and its gradient, composed with Sigmoid.backward"""
    n = y.size
    loss = -np.mean(t * np.log(y + BCE_EPS) + (1 - t) * np.log(1 - y + BCE_EPS))
    dy = -(t - y) / (y * (1 - y + BCE_EPS) + BCE_EPS) / n
    return loss, dy * y * (1 - y)


def to_flat_img(x):  # [B][C][S][S] -> [B][C S S] (View order)
    return x.reshape(x.shape[0], -1)


def adam(P, g, m, v, t, h):
    """penalty -> clamp -> optim.adam on the shared (m, v, t); returns the new (P, m, v, t)"""
    g = g + h["L1"] * np.sign(P) + h["L2"] * P
    if h["clamp"] != 0:
        g = np.clip(g, -h["clamp"], h["clamp"])
    t += 1
    m = h["beta1"] * m + (1 - h["beta1"]) * g
    v = h["beta2"] * v + (1 - h["beta2"]) * g * g
    step = h["lr"] * np.sqrt(1 - h["beta2"] ** t) / (1 - h["beta1"] ** t)
    return P - step * m / (np.sqrt(v) + h["eps"]), m, v, t


HYPER = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, L1=0.0, L2=0.0, clamp=1.0, p_drop=0.2, noise_std=0.1)


def train_step(st, images, noise, masks, C, S, h=HYPER, ae2_input=None, ae2_kinks=None):
    """train_denoiser.lua:247-341 on st = dict(P1, P2, m, v, t, bn1, bn2) (updated in place); noise [2][B][C][S][S],
    masks [3][B][mps].  Returns (loss_AE1, loss_AE2) and the two gradients (after penalty / clamp they are not).
    ae2_input (optional, [B][C][S][S]): AE2's input as another implementation computed it, in place of AE's output
    here; AE's second forward still runs (it updates AE's running statistics).  ae2_kinks: the `kinks` of AE2's forward."""
    x = np.asarray(images, np.float64)
    t = to_flat_img(x)
    # fevalAE + adam
    z4, cache = decoder_forward(st["P1"], x + noise[0], st["bn1"], True, masks[0], C, S, h["p_drop"])
    loss1, dz4 = bce(sigmoid(z4), t)
    g1 = decoder_backward(cache, dz4, C, S)
    st["P1"], st["m"], st["v"], st["t"] = adam(st["P1"], g1, st["m"], st["v"], st["t"], h)
    # fevalAE2 + adam: AE forward again with fresh noise / masks and its updated parameters
    z4a, _ = decoder_forward(st["P1"], x + noise[1], st["bn1"], True, masks[1], C, S, h["p_drop"])
    y1 = sigmoid(z4a).reshape(x.shape) if ae2_input is None else np.asarray(ae2_input, np.float64)
    z4b, cache2 = decoder_forward(st["P2"], y1, st["bn2"], True, masks[2], C, S, h["p_drop"], ae2_kinks)
    loss2, dz4b = bce(sigmoid(z4b), t)
    g2 = decoder_backward(cache2, dz4b, C, S)
    st["P2"], st["m"], st["v"], st["t"] = adam(st["P2"], g2, st["m"], st["v"], st["t"], h)
    return (loss1, loss2), (g1, g2)


def evaluate(P, bn, x, C, S):
    """AE1_DECODER:evaluate():forward(x) (train.lua --denoise)"""
    z4, _ = decoder_forward(P, np.asarray(x, np.float64), bn.copy(), False, None, C, S)
    return sigmoid(z4).reshape(x.shape)


def make_params(C, S, rng):
    """test parameters: weights ~ U(+-1/sqrt(fan_in)) (torch's reset), gamma ~ U(0.5, 1.5), beta ~ U(-0.1, 0.1)"""
    parts = []
    for name, shape in shapes(C, S):
        n = int(np.prod(shape))
        if name[0] == "g":
            parts.append(rng.uniform(0.5, 1.5, n))
        elif name[0] == "b" and len(name) == 2:
            parts.append(rng.uniform(-0.1, 0.1, n))
        else:
            wshape = dict(shapes(C, S))[name[:-1] + "W"]
            fan = int(np.prod(wshape[1:]))
            parts.append(rng.uniform(-1, 1, n) / np.sqrt(fan))
    return np.concatenate(parts)


def make_case(C, S, B, seed):
    """images, noise [2], masks [3] and both decoders' parameters, all float32-representable"""
    rng = np.random.default_rng(seed)
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    mps = mask_per_sample(S)
    return dict(images=f(rng.uniform(0, 1, (B, C, S, S))), noise=f(rng.normal(0, 0.1, (2, B, C, S, S))),
                masks=f(rng.uniform(0, 1, (3, B, mps)) >= 0.2), P1=f(make_params(C, S, rng)), P2=f(make_params(C, S, rng)))


def zero_grad_biases(C, S):
    """boolean mask of the analytically zero-gradient entries: the conv biases and Linear1's bias, each in front of a
    BatchNorm"""
    out, o = [], 0
    for name, shape in shapes(C, S):
        n = int(np.prod(shape))
        out.append(np.full(n, name in ("c1b", "c2b", "L1b")))
        o += n
    return np.concatenate(out)


def relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
