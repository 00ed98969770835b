"""float64 numpy restatement of train_autoencoder.lua's net and batch step, the reference of the fg_ae_* tests.

    MODEL_AE = View(I) Linear(I,512) ReLU Linear(512,d) Tanh Dropout(p) Linear(d,256) ReLU Linear(256,I) Sigmoid   (:80-92)
    step     = zero gradients, forward, nn.AbsCriterion(outputs, inputs), backward, g += L1 sign(P) + L2 P, optim.adam  (:178-209)

Written from those semantics, not from the library.  Keep flags are inputs.  nn.ReLU and nn.AbsCriterion are not
differentiable at their kinks; `kinks` lets a caller fix the side of chosen elements (to the side another
implementation took for elements within rounding of the kink), everything else follows the rules here:
ReLU passes the gradient where z > 0; the criterion's gradient is +1/n where y >= t (a tie is positive), else -1/n.
"""
import numpy as np

H1, H3 = 512, 256
HYPER = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, L1=0.0, L2=0.0, p_drop=0.5)


def shapes(S, d):
    I = S * S
    return [("L1W", (H1, I)), ("L1b", (H1,)), ("L2W", (d, H1)), ("L2b", (d,)), ("L3W", (H3, d)), ("L3b", (H3,)),
            ("L4W", (I, H3)), ("L4b", (I,))]


def param_count(S, d):
    return sum(int(np.prod(s)) for _, s in shapes(S, d))


def unflat(P, S, d):
    out, o = {}, 0
    for name, shape in shapes(S, d):
        n = int(np.prod(shape))
        out[name] = P[o:o + n].reshape(shape)
        o += n
    assert o == P.size
    return out


def relerr(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def _side(z, key, kinks):
    """z > 0, except where `kinks[key]` = (flat indices, bool side) says otherwise"""
    pos = z > 0
    if kinks and key in kinks:
        idx, side = kinks[key]
        pos.reshape(-1)[idx] = side
    return pos


def forward(P, x, masks, S, d, p=0.5, kinks=None):
    """x [B][I] float64; masks [B][d] keep flags (training) or None (evaluation).  Returns every tensor by name."""
    W = unflat(np.asarray(P, np.float64), S, d)
    x = np.asarray(x, np.float64).reshape(-1, S * S)
    c = dict(x=x, W=W, p=p)
    c["z1"] = x @ W["L1W"].T + W["L1b"]
    c["pos1"] = _side(c["z1"], "z1", kinks)
    c["h1"] = np.where(c["pos1"], c["z1"], 0.0)
    c["z2"] = c["h1"] @ W["L2W"].T + W["L2b"]
    c["code"] = np.tanh(c["z2"])
    c["keep"] = None if masks is None else np.asarray(masks, np.float64).reshape(-1, d) / (1.0 - p)
    c["h2"] = c["code"] if masks is None else c["code"] * c["keep"]
    c["z3"] = c["h2"] @ W["L3W"].T + W["L3b"]
    c["pos3"] = _side(c["z3"], "z3", kinks)
    c["h3"] = np.where(c["pos3"], c["z3"], 0.0)
    c["z4"] = c["h3"] @ W["L4W"].T + W["L4b"]
    c["y"] = sigmoid(c["z4"])
    return c


def criterion(y, t, kinks=None):
    """nn.AbsCriterion, size-averaged: (loss, dL/dy)"""
    t = np.asarray(t, np.float64).reshape(y.shape)
    pos = (y - t) >= 0
    if kinks and "y" in kinks:
        idx, side = kinks["y"]
        pos.reshape(-1)[idx] = side
    return float(np.abs(y - t).mean()), np.where(pos, 1.0, -1.0) / y.size


def backward(c, dy):
    """dy = dL/dy [B][I] -> (flat parameter gradient, dict of dz4 dz3 dz2 dz1)"""
    W = c["W"]
    dz4 = dy.reshape(c["y"].shape) * (1.0 - c["y"]) * c["y"]
    dh3 = dz4 @ W["L4W"]
    dz3 = np.where(c["pos3"], dh3, 0.0)
    dh2 = dz3 @ W["L3W"]
    dcode = dh2 if c["keep"] is None else dh2 * c["keep"]
    dz2 = dcode * (1.0 - c["code"] ** 2)
    dh1 = dz2 @ W["L2W"]
    dz1 = np.where(c["pos1"], dh1, 0.0)
    g = [dz1.T @ c["x"], dz1.sum(0), dz2.T @ c["h1"], dz2.sum(0), dz3.T @ c["h2"], dz3.sum(0), dz4.T @ c["h3"], dz4.sum(0)]
    return np.concatenate([a.ravel() for a in g]), dict(dz4=dz4, dz3=dz3, dz2=dz2, dz1=dz1)


def adam(P, g, m, v, t, h=HYPER):
    """stock optim.adam, in place on P, m, v; returns the new step count"""
    t += 1
    m *= h["beta1"]
    m += (1 - h["beta1"]) * g
    v *= h["beta2"]
    v += (1 - h["beta2"]) * g * g
    step = h["lr"] * np.sqrt(1 - h["beta2"] ** t) / (1 - h["beta1"] ** t)
    P -= step * m / (np.sqrt(v) + h["eps"])
    return t


def train_step(st, images, masks, S, d, h=HYPER, kinks=None):
    """one batch on st = dict(P, m, v, t) (float64, updated in place).  Returns (loss, gradient incl. penalty, cache)."""
    x = np.asarray(images, np.float64).reshape(-1, S * S)
    c = forward(st["P"], x, masks, S, d, h["p_drop"], kinks)
    loss, dy = criterion(c["y"], x, kinks)
    g, dz = backward(c, dy)
    c.update(dz)
    if h["L1"] != 0 or h["L2"] != 0:
        g = g + h["L1"] * np.sign(st["P"]) + h["L2"] * st["P"]
    st["t"] = adam(st["P"], g, st["m"], st["v"], st["t"], h)
    return loss, g, c


def loop(st, batches, S, d, h=HYPER):
    """batches: [(images, masks)]; returns the losses"""
    return [train_step(st, im, mk, S, d, h)[0] for im, mk in batches]


def fresh_state(P):
    return dict(P=np.asarray(P, np.float64).copy(), m=np.zeros(P.size), v=np.zeros(P.size), t=0)


def make_case(S, B, d, seed, w_scale=10.0):
    """seeded float32 inputs.  The weights are the script's initialisation scaled by w_scale (N(0,1) * 0.005 alone leaves
    every activation within 1e-2 of its bias, which would hide a wrong layer behind the tolerance).  Targets are the
    images; any image pixel closer than 1e-3 to the initial output is moved until none is, so that no element sits on
    the criterion's kink (the tie rule has its own test)."""
    rng = np.random.default_rng(seed)
    P = np.concatenate([rng.standard_normal(int(np.prod(s))) * ((0.005 if n[-1] == "W" else 0.001) * w_scale)
                        for n, s in shapes(S, d)]).astype(np.float32)
    images = rng.uniform(0.05, 0.95, (B, 1, S, S)).astype(np.float32)
    masks = (rng.uniform(size=(B, d)) >= 0.5).astype(np.float32)
    for _ in range(20):
        y = forward(P, images.reshape(B, -1), masks, S, d)["y"].reshape(images.shape)
        near = np.abs(y - images) < 1e-3
        if not near.any():
            break
        images[near] += np.where(images[near] < 0.5, 0.01, -0.01).astype(np.float32)
    else:
        raise AssertionError("make_case: could not move the targets off the initial outputs")
    return dict(P=P, images=images, masks=masks)
