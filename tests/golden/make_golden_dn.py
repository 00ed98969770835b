"""Writes dn_step_c1_s16_b4.npz: one train_denoiser.lua batch step (AE update, then AE2 update on one Adam state) of the
float64 restatement tests/dn_ref.py, on the seeded case dn_ref.make_case(1, 16, 4, seed=2024).  The inputs are stored
in full; the parameters and Adam moments after the step as every 997th entry (the full vectors would be 12 MB)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import dn_ref as R  # noqa: E402

C, S, B, SEED = 1, 16, 4, 2024
case = R.make_case(C, S, B, seed=SEED)
n = R.param_count(C, S)
st = dict(P1=case["P1"].astype(np.float64), P2=case["P2"].astype(np.float64), m=np.zeros(n), v=np.zeros(n), t=0,
          bn1=R.bn_init(), bn2=R.bn_init())
losses, _ = R.train_step(st, case["images"], case["noise"], case["masks"], C, S)
sel = np.arange(0, n, 997)
np.savez_compressed(os.path.join(HERE, "dn_step_c1_s16_b4.npz"), C=C, S=S, B=B, seed=SEED, images=case["images"],
                    noise=case["noise"], masks=case["masks"], losses=np.array(losses), sel=sel, P1=st["P1"][sel],
                    P2=st["P2"][sel], m=st["m"][sel], v=st["v"][sel], bn1=st["bn1"], bn2=st["bn2"])
