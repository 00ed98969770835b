"""Seeded cases, a float64 PyTorch D and the data-parallel restatement of the coarse-to-fine nets at fine size S
(train_c2f.lua --fineSize 16, 32 or 64), for tests/test_c2f_sizes.py and tests/test_gpu_c2f_sizes.py.

The counterparts of c2f_utils.py, torch_ref_c2f.py and dp_ref_c2f.py with S an argument; G's restatement
(torch_ref_c2f.G_forward) and its layout do not depend on S and are used as they are."""
import numpy as np
import torch
import torch.nn.functional as F

import c2f_utils as CU
from face_generator_b200 import layouts as LY
from oracle import oracle as O
from oracle import oracle_c2f_sized as OS
from torch_ref import _split, d_sigmoid, prelu
from torch_ref_c2f import maxpool2, trained_like


def make_case(B, C, seed, init="trained", fine_size=32):
    """c2f_utils.make_case at fine size S: images, noise and masks [.][.][S][S] / [.][mask_per_sample(S)]"""
    S = fine_size
    rng = np.random.default_rng(seed)
    sl = 1.0 if init == "smooth" else 0.25
    gG, gD = (1.0, 0.8) if init == "smooth" else (1.2, 1.0)
    PG = LY.trained_like_init(LY.c2f_G_layout(C), rng, gG, slope=sl)
    PD = LY.trained_like_init(LY.c2f_D_layout(C, S), rng, gD, slope=sl)
    real_diff, cond_real = LY.c2f_pairs(B // 2, C, rng, S)
    _, cond_fake = LY.c2f_pairs(B // 2, C, rng, S)
    _, cond_G = LY.c2f_pairs(B, C, rng, S)
    M = OS.mask_per_sample(S)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(PG=f(PG), PD=f(PD), real_diff=real_diff, cond_D=f(np.concatenate([cond_real, cond_fake])),
                noise_D=f(rng.uniform(-1, 1, (B // 2, 1, S, S))), cond_G=cond_G,
                noise_G=f(rng.uniform(-1, 1, (B, 1, S, S))),
                masks_D=f(rng.random((B, M)) < 0.5), masks_G=f(rng.random((B, M)) < 0.5))


def oracle_iteration(case, B, C, fine_size, hyper=None, state=None):
    st = state or CU.fresh_state(case)
    res = OS.f64.train_iteration(fine_size, B, C, hyper or CU.HYPER, case["real_diff"], case["cond_D"], case["noise_D"],
                                 case["cond_G"], case["noise_G"], case["masks_D"], case["masks_G"], st)
    res["state"] = st
    return res


def D_forward(P, diff, cond, masks, C=3, branch=None, route=None, fine_size=32):
    """torch_ref_c2f.D_forward at fine size S: View(256*(S/4)^2) before the Linear"""
    p = _split(P, OS.D_layout(C, fine_size))
    B, Fl = diff.shape[0], OS.flat(fine_size)
    x = diff + cond  # CAddTable
    for i in range(4):
        x = prelu(F.conv2d(x, p["c%dW" % (i + 1)], p["c%db" % (i + 1)], padding=1), p["a%d" % (i + 1)], branch,
                  "z%d" % (i + 1))
        if i in (1, 3):
            x = maxpool2(x, route, "p%d" % (i + 1))
    x = x.reshape(B, Fl) * masks[:, :Fl] * 2.0  # nn.Dropout p=0.5 (v2), then View in (c,h,w) order
    h = prelu(F.linear(x, p["L1W"], p["L1b"]), p["a5"], branch, "zl1") * masks[:, Fl:] * 2.0
    return d_sigmoid(F.linear(h, p["L2W"], p["L2b"])).reshape(B)


def trained_like_D(C, rng, fine_size):
    return trained_like(OS.D_layout(C, fine_size), OS.D_param_count(C, fine_size), rng)


def make_masks(B, rng, fine_size):
    return (rng.random((B, OS.mask_per_sample(fine_size))) < 0.5).astype(np.float64)


def make_pairs(B, C, rng, fine_size):
    """fine ~ U[0,1), coarse = 2x avg-down then 2x nearest-up, diff = fine - coarse, all [B][C][S][S]"""
    S = fine_size
    fine = rng.random((B, C, S, S))
    small = fine.reshape(B, C, S // 2, 2, S // 2, 2).mean(axis=(3, 5))
    coarse = np.repeat(np.repeat(small, 2, axis=2), 2, axis=3)
    return fine - coarse, coarse


def rank_step(case, st, B, C, world, allreduce, fine_size, hyper=None):
    """dp_ref_c2f.rank_step at fine size S (netpair.cu::pair_train_step on the c2f nets for world > 1, restated with
    the CPU oracle)"""
    hp = hyper or CU.HYPER
    Bh = B // 2
    G, D = OS.f64.G(fine_size), OS.f64.D(fine_size)
    fake = G.forward(st["PG"], case["noise_D"], case["cond_D"][Bh:])
    inputs = np.concatenate([case["real_diff"].astype(np.float64), fake])
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)])
    out = D.forward(st["PD"], inputs, case["cond_D"], case["masks_D"])
    lossD = O.f64.bce_fwd(out, targets)
    gD, _ = D.backward(O.f64.bce_bwd(out, targets), want_ddiff=False)
    conf = np.array([np.sum((out > 0.5) & (targets > 0.5)), np.sum((out <= 0.5) & (targets > 0.5)),
                     np.sum((out > 0.5) & (targets < 0.5)), np.sum((out <= 0.5) & (targets < 0.5))], np.float64)
    red = allreduce(np.concatenate([gD, conf]))
    gD, conf = red[:-4] / world, red[-4:]
    lossD += O.f64.penalty_clamp(st["PD"], gD, hp["D_L1"], hp["D_L1"], hp["D_L2"], hp["D_clamp"])
    st["tD"] += 1
    O.f64.adam(st["PD"], gD, st["mD"], st["vD"], st["tD"], hp["lr_D"], hp["beta1"], hp["beta2"], hp["eps"])
    diff = G.forward(st["PG"], case["noise_G"], case["cond_G"])
    out = D.forward(st["PD"], diff, case["cond_G"], case["masks_G"])
    ones = np.ones(B)
    lossG = O.f64.bce_fwd(out, ones)
    _, ddiff = D.backward(O.f64.bce_bwd(out, ones), want_dP=False)
    gG = allreduce(G.backward(ddiff)) / world
    l1g = hp["G_L2"] if (hp["G_L1"] != 0 or hp["G_L2"] != 0) else 0.0
    lossG += O.f64.penalty_clamp(st["PG"], gG, hp["G_L1"], l1g, hp["G_L2"], hp["G_clamp"])
    st["tG"] += 1
    O.f64.adam(st["PG"], gG, st["mG"], st["vG"], st["tG"], hp["lr_G"], hp["beta1"], hp["beta2"], hp["eps"])
    return dict(lossD=lossD, lossG=lossG, conf=conf, gradD=gD, gradG=gG)
