"""Data-parallel semantics of fg_s16_train_step restated with the CPU oracle (test infrastructure): the same scheme as
dp_ref.py (per-rank gradient of the rank's shard, sum-all-reduce of the flat gradient + confusion counts, 1/N, then
penalty -> clamp -> Adam identically on every rank) on the --scale 16 nets (netpair.cu::pair_train_step)."""
import numpy as np

from oracle import oracle as O
from oracle import oracle_s16 as OS
import s16_utils as SU


def rank_step(case, st, B, C, world, allreduce, hyper=None):
    """case: this rank's inputs; st: replicated state dict PD, PG, mD, vD, mG, vG, bn (updated in place)."""
    hp = hyper or SU.HYPER
    t = O.f64
    Bh = B // 2
    g, d = OS.f64.G(), OS.f64.D()
    fake = g.forward(st["PG"], case["noise_D"], C, st["bn"])
    x = np.concatenate([case["real"].astype(np.float64), fake])
    tg = np.concatenate([np.ones(Bh), np.zeros(Bh)])
    out = d.forward(st["PD"], x, case["masks_D"], True)
    lossD = t.bce_fwd(out, tg)
    gD, _ = d.backward(t.bce_bwd(out, tg))
    conf = np.array([np.sum((out > 0.5) & (tg > 0.5)), np.sum((out <= 0.5) & (tg > 0.5)), np.sum((out > 0.5) & (tg < 0.5)),
                     np.sum((out <= 0.5) & (tg < 0.5))], np.float64)
    red = allreduce(np.concatenate([gD, conf]))
    gD, conf = red[:-4] / world, red[-4:]
    lossD += t.penalty_clamp(st["PD"], gD, hp["D_L1"], hp["D_L1"], hp["D_L2"], hp["D_clamp"])
    t.adam(st["PD"], gD, st["mD"], st["vD"], 1, hp["lr_D"], hp["beta1"], hp["beta2"], hp["eps"])
    img = g.forward(st["PG"], case["noise_G"], C, st["bn"])
    outG = d.forward(st["PD"], img, case["masks_G"], True)
    ones = np.ones(B)
    lossG = t.bce_fwd(outG, ones)
    _, dimg = d.backward(t.bce_bwd(outG, ones))
    gG = allreduce(g.backward(dimg)) / world
    lossG += t.penalty_clamp(st["PG"], gG, hp["G_L1"], hp["G_L2"], hp["G_L2"], hp["G_clamp"])
    t.adam(st["PG"], gG, st["mG"], st["vG"], 1, hp["lr_G"], hp["beta1"], hp["beta2"], hp["eps"])
    return dict(lossD=lossD, lossG=lossG, conf=conf, gradD=gD, gradG=gG)


def fresh_state(case):
    PD, PG = case["PD"].astype(np.float64), case["PG"].astype(np.float64)
    return dict(PD=PD, PG=PG, mD=np.zeros_like(PD), vD=np.zeros_like(PD), mG=np.zeros_like(PG), vG=np.zeros_like(PG),
                bn=SU.bn_init())
