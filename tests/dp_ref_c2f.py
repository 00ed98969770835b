"""Data-parallel semantics of the coarse-to-fine train step, restated with the CPU oracle (test infrastructure).
Mirrors face_generator_b200/csrc/netpair.cu::pair_train_step on the c2f nets for world > 1: per-shard gradients, one
sum-all-reduce of the flat gradient (+ the confusion counts in its tail) per optimizer step, 1/N, then penalty -> clamp -> Adam
identically on every rank (adversarial_c2f.lua:56-76, :104-112; SURVEY.md section 8e)."""
import numpy as np

from oracle import oracle as O
from oracle import oracle_c2f as OC
import c2f_utils as CU


def rank_step(case, st, B, C, world, allreduce, hyper=None):
    hp = hyper or CU.HYPER
    Bh = B // 2
    G, D = OC.f64.G(), OC.f64.D()
    # ---- D step ----
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
    # ---- G step ----
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
