"""Writes ae_step_s16_b4.npz: one train_autoencoder.lua batch step of the float64 restatement tests/ae_ref.py with L1 / L2
penalties on, on the seeded case ae_ref.make_case(16, 4, 64, seed=2025).  The inputs are stored in full; the gradient,
parameters and Adam moments after the step as every 397th entry."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ae_ref as R  # noqa: E402

S, B, D, SEED = 16, 4, 64, 2025
case = R.make_case(S, B, D, seed=SEED)
st = R.fresh_state(case["P"])
h = dict(R.HYPER, L1=1e-5, L2=1e-4)
loss, g, c = R.train_step(st, case["images"], case["masks"], S, D, h)
sel = np.arange(0, st["P"].size, 397)
np.savez_compressed(os.path.join(HERE, "ae_step_s16_b4.npz"), S=S, B=B, d=D, seed=SEED, L1=h["L1"], L2=h["L2"],
                    images=case["images"], masks=case["masks"], loss=loss, sel=sel, g=g[sel], P=st["P"][sel], m=st["m"][sel],
                    v=st["v"][sel], code=c["code"], y=c["y"])
