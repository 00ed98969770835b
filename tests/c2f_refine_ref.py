"""float64 restatement of sample.lua:176-214 c2f(images, G, D, fineSize) (fg_c2f_refine), for
tests/test_c2f_refine_cpu.py and tests/test_gpu_c2f_refine.py: image.scale from oracle_data, G and D from the sized
coarse-to-fine oracle, then sample.lua's pick rule on the float32-rounded predictions."""
import numpy as np

from oracle import oracle_c2f_sized as OS
from oracle import oracle_data as OD


def lua_pick(predictions):
    """sample.lua:199-207 as written, on one image's predictions (a sequence of float32)"""
    maxval, pick = None, None
    for j, v in enumerate(predictions):
        if maxval is None or v > maxval:
            maxval, pick = v, j
    return pick


def pick_rule(pred):
    """the same rule on pred [N][tries], vectorised: the first maximum; a NaN wins only at t = 0"""
    pred = np.asarray(pred)
    pick = np.argmax(np.where(np.isnan(pred), -np.inf, pred), axis=1)
    pick[np.isnan(pred[:, 0])] = 0
    return pick.astype(np.int32)


def refine(PG, PD, images, S, noise, masks, training, diff=None):
    """images [N][C][in][in], noise [N*tries][1][S][S], masks [N*tries][mask] (or None when not training) ->
    dict(up [N][C][S][S], diff [N*tries][C][S][S], pred [N][tries] float64, pick [N] of the float32 pred, out [N][C][S][S]).
    diff: G's output of an earlier call on the same PG, images and noise (G does not depend on `training`)."""
    N, C = images.shape[:2]
    tries = noise.shape[0] // N
    up = OD.scale(np.asarray(images, np.float64), S, S)
    cond = np.repeat(up, tries, axis=0)
    if diff is None:
        diff = OS.f64.G(S).forward(PG, noise, cond)
    pred = OS.f64.D(S).forward(PD, diff, cond, masks if training else None, training=bool(training)).reshape(N, tries)
    pick = pick_rule(pred.astype(np.float32))
    out = up + diff.reshape(N, tries, C, S, S)[np.arange(N), pick]
    return dict(up=up, diff=diff, pred=pred, pick=pick, out=out)
