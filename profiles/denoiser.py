"""Time of one train_denoiser.lua batch step (fg_dn_train_step: AE update, then AE2 update) at batch 128, C = 3, for
S = 32 and S = 16, eager (option use_graph 0) and replayed from a captured CUDA graph.  Noise and dropout masks are
drawn on the device from the step seed; the images are a device buffer, so no host transfer is timed.

Per configuration one JSON line: ms per step (best of `--rounds` windows of `--steps` steps, CUDA events), kernel
launches per step (fg_kernel_launches), and the HBM lower bound of the step computed from its shapes:
  - two Adam passes over one decoder's parameters, each reading p, g, m, v and writing p, m, v (28 B per parameter);
  - per Linear weight, 7 passes of 4 B: the fp32 pack, its FP16 split for forward and data gradient (read + write),
    the three forwards' operand reads, the two data gradients' reads, the weight gradient write / unpack;
that is bytes / 3.35e12 B/s, the H100 SXM data-sheet bandwidth.  Then the card's name and power limit, read in the same
run.

usage:  python profiles/denoiser.py [--steps 20] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import denoiser as D  # noqa: E402

HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:
        return "unknown (%s)" % e, "unknown"


def hbm_bytes(C, S):
    n = D.param_count(C, S)
    lin = 2048 * 8 * (S - 4) ** 2 + C * S * S * 2048
    return 2 * 28 * n + 2 * 7 * 4 * lin


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    B, C = 128, 3
    ctx = fg.Context(0, max_batch=B, channels=C)
    rng = np.random.default_rng(0)
    h = D.dn_hyper_default()
    for S in (32, 16):
        dn = D.Denoiser(ctx, S)
        for net in (0, 1):
            dn.set_params(net, D.init_params(C, S, rng))
        images = ctx.dev_array(rng.uniform(0, 1, (B, C, S, S)).astype(np.float32))
        for use_graph in (0, 1):
            ctx.set_option("use_graph", use_graph)
            seed = [0]

            def step():
                seed[0] += 1
                dn.train_step(h, images, seed=seed[0], B=B)

            for _ in range(3):
                step()
            l0 = ctx.launches()
            step()
            launches = ctx.launches() - l0
            best = float("inf")
            for _ in range(a.rounds):
                ctx.sync()
                ctx.event_record(0)
                for _ in range(a.steps):
                    step()
                ctx.event_record(1)
                ctx.sync()
                best = min(best, ctx.event_elapsed_ms(0, 1) / a.steps)
            bound = hbm_bytes(C, S) / HBM * 1e3
            print(json.dumps(dict(S=S, C=C, B=B, mode="replayed" if use_graph else "eager", ms_per_step=round(best, 4),
                                  launches_per_step=launches, hbm_bound_ms=round(bound, 4),
                                  share_of_bound=round(bound / best, 3), params_per_decoder=dn.n)))
        ctx.set_option("use_graph", 1)
        ctx.dev_free(images)
        dn.close()
    name, limit = card()
    print(json.dumps(dict(card=name, power_limit=limit)))
    ctx.close()


if __name__ == "__main__":
    main()
