"""Time of one train_autoencoder.lua batch step (fg_ae_train_step) at batch 128, --noiseDim 256, for S = 32 and S = 16,
replayed from its captured CUDA graph on a device buffer of images (no host transfer is timed), and of an epoch of
10 000 images fed from a DeviceDataset (79 batches, the last of 16).

Per S one JSON line: ms per step (best of `--rounds` windows of `--steps` steps, CUDA events), kernel launches per step
(fg_kernel_launches), the epoch enqueued without waiting (stats == NULL) against the same epoch with a synchronise per
step, and the per-kernel split of an eager, timed step from the library's timer names (`ae.*`; the elementwise kernels
and the optimizer are the remainder).  Then the card's name and power limit, read in the same run.  Needs a GPU.

usage:  python profiles/autoencoder.py [--steps 2000] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import autoencoder as A  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402

TIMERS = ["ae.L%d.%s" % (l, k) for l in (1, 2, 3, 4) for k in ("fwd", "dgrad", "wgrad")]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def epoch_ms(ae, ds, h, sync, seed):
    batches = A.epoch_batches(ds.size(), 128, np.random.default_rng(seed))
    ae.ctx.sync()
    t0 = time.perf_counter()
    for k, idx in enumerate(batches):
        ae.train_step_dataset(ds, h, idx, seed=k, sync=sync)
    ae.ctx.sync()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    B, d = 128, 256
    ctx = fg.Context(0, max_batch=B, channels=1)
    rng = np.random.default_rng(0)
    h = A.ae_hyper_default()
    ds = DeviceDataset(ctx, rng.integers(0, 256, (10000, 1, 64, 64), dtype=np.uint8))
    for S in (32, 16):
        ae = A.Autoencoder(ctx, S, d)
        ae.set_params(A.init_params(S, d, rng))
        images = ctx.dev_array(rng.uniform(0, 1, (B, 1, S, S)).astype(np.float32))
        seed = [0]

        def step():
            seed[0] += 1
            ae.train_step(h, images, seed=seed[0], B=B, sync=False)

        for _ in range(20):
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
        epoch_ms(ae, ds, h, False, 1)  # warm the tail batch's graph
        epoch_ms(ae, ds, h, False, 1)
        enq = min(epoch_ms(ae, ds, h, False, 2 + r) for r in range(a.rounds))
        syn = min(epoch_ms(ae, ds, h, True, 2 + r) for r in range(a.rounds))
        ctx.timing_enable(True)  # a timed step runs eagerly, one event pair per named kernel
        for _ in range(50):
            step()
        ctx.sync()
        split = {}
        for name in TIMERS:
            ms, n = ctx.timing_get(name)
            if n:
                split[name] = round(ms / n * 1e3, 2)
        ctx.timing_enable(False)
        print(json.dumps(dict(S=S, B=B, noise_dim=d, params=ae.n, ms_per_step=round(best, 4), launches_per_step=launches,
                              epoch_10000_enqueued_ms=round(enq, 2), epoch_10000_sync_per_step_ms=round(syn, 2),
                              linear_kernels_us=split, linear_kernels_total_us=round(sum(split.values()), 1))))
        ctx.dev_free(images)
        ae.close()
    name, limit = card()
    print(json.dumps(dict(card=name, power_limit=limit)))
    ds.close()
    ctx.close()


if __name__ == "__main__":
    main()
