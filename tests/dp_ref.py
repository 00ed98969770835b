"""Data-parallel semantics of the train step, restated with the CPU oracle (test infrastructure).

Mirrors face_generator_b200/csrc/netpair.cu::pair_train_step on the 32x32 nets for world > 1: every rank computes the
gradient of ITS shard (BatchNorm statistics stay per replica), the flat gradient (+ confusion counts in the tail)
is sum-all-reduced, scaled by 1/N, then penalty -> clamp -> Adam run identically on every rank
(SURVEY.md section 8e)."""
import numpy as np

from oracle import oracle as O
import parity_utils as PU


def rank_step(case, st, B, C, world, allreduce, hyper=None):
    """case: this rank's inputs; st: replicated state (updated in place); allreduce(np.ndarray) -> summed copy."""
    hp = hyper or PU.HYPER
    Bh = B // 2
    G, D = O.f64.G(), O.f64.D()
    # ---- D step ----
    fake = G.forward(st["PG"], case["noise_D"], C, True, st["bnG"])
    inputs = np.concatenate([case["real"].astype(np.float64), fake])
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)])
    out = D.forward(st["PD"], inputs, case["masks_D"])
    lossD = O.f64.bce_fwd(out, targets)
    gD, _ = D.backward(O.f64.bce_bwd(out, targets), want_dimg=False)
    conf = np.array([np.sum((out > 0.5) & (targets > 0.5)), np.sum((out <= 0.5) & (targets > 0.5)),
                     np.sum((out > 0.5) & (targets < 0.5)), np.sum((out <= 0.5) & (targets < 0.5))], np.float64)
    red = allreduce(np.concatenate([gD, conf]))
    gD, conf = red[:-4] / world, red[-4:]
    lossD += O.f64.penalty_clamp(st["PD"], gD, hp["D_L1"], hp["D_L1"], hp["D_L2"], hp["D_clamp"])
    st["tD"] += 1
    O.f64.adam(st["PD"], gD, st["mD"], st["vD"], st["tD"], hp["lr_D"], hp["beta1"], hp["beta2"], hp["eps"])
    # ---- G step ----
    img = G.forward(st["PG"], case["noise_G"], C, True, st["bnG"])
    out = D.forward(st["PD"], img, case["masks_G"])
    ones = np.ones(B)
    lossG = O.f64.bce_fwd(out, ones)
    _, dimg = D.backward(O.f64.bce_bwd(out, ones), want_dP=False)
    gG = G.backward(dimg)
    gG = allreduce(gG) / world
    l1g = hp["G_L2"] if (hp["G_L1"] != 0 or hp["G_L2"] != 0) else 0.0
    lossG += O.f64.penalty_clamp(st["PG"], gG, hp["G_L1"], l1g, hp["G_L2"], hp["G_clamp"])
    st["tG"] += 1
    O.f64.adam(st["PG"], gG, st["mG"], st["vG"], st["tG"], hp["lr_G"], hp["beta1"], hp["beta2"], hp["eps"])
    return dict(lossD=lossD, lossG=lossG, conf=conf, gradD=gD, gradG=gG)
