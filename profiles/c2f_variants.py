"""Time of the captured device-fed coarse-to-fine train step (fg_c2f_train_step_dataset) for each pair of
models_c2f.lua's nets, colour, batch 256, fine sizes 32 and 64 (coarse size S/2):
  create_G_d / create_D_c (the default pair), each other generator with create_D_c and each other discriminator
  with create_G_d
Every pair gets 3 warm-up calls (eager, captured, replayed), then `--rounds` windows of `--steps` calls, the pairs of a
group alternating window by window, timed with CUDA events on the ctx stream.  A group is the default pair and up to
`--group` - 1 others of one size (at fine size 64 a pair's buffers take about 18 GB at batch 256, so not all six fit
on one card at once); the default pair's line is printed once per group.  Every call reads its statistics, as the
Lua loop does.  One JSON line per pair with the median ms per step, then the card's name and power limit, read in the
same run.

usage:  python profiles/c2f_variants.py [--steps 10] [--rounds 5] [--sizes 32,64]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from disc_variants import card, windowed  # noqa: E402

C, B = 3, 256
PAIRS = [("create_G_d", "create_D_c"), ("create_G_a", "create_D_c"), ("create_G_b", "create_D_c"),
         ("create_G_c", "create_D_c"), ("create_G_d", "create_D_a"), ("create_G_d", "create_D_b")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", default="32,64")
    ap.add_argument("--group", type=int, default=3)
    a = ap.parse_args()
    imgs = np.random.default_rng(0).integers(0, 256, (2048, C, 64, 64), dtype=np.uint8)
    h = fg.hyper_default()
    others = PAIRS[1:]
    groups = [[PAIRS[0]] + others[i:i + a.group - 1] for i in range(0, len(others), a.group - 1)]
    for S, group in [(int(s), g) for s in a.sizes.split(",") for g in groups]:
        nets = []
        for gen, disc in group:
            rng = np.random.default_rng(1)
            ctx = fg.Context(0, max_batch=B, channels=C)
            net = fg.C2f(ctx, S, gen, disc)
            net.set_params(fg.lib.NET_G, rng.uniform(-0.05, 0.05, net.nG).astype(np.float32))
            net.set_params(fg.lib.NET_D, rng.uniform(-0.02, 0.02, net.nD).astype(np.float32))
            ds = DeviceDataset(ctx, imgs)
            seed = [100]

            def step(net=net, ds=ds, seed=seed, S=S):
                seed[0] += 1
                return net.train_step_dataset(ds, h, B, S // 2, seed[0])
            for _ in range(3):
                step()
            nets.append((gen, disc, ctx, net, ds, step, []))
        for _ in range(a.rounds):
            for gen, disc, ctx, net, ds, step, times in nets:
                times.append(windowed(ctx, step, a.steps))
        for gen, disc, ctx, net, ds, step, times in nets:
            print(json.dumps({"fine_size": S, "generator": gen, "discriminator": disc, "batch": B, "channels": C,
                              "ms_per_step": round(float(np.median(times)), 3), "ms_min": round(min(times), 3),
                              "ms_max": round(max(times), 3), "G_params": net.nG, "D_params": net.nD}), flush=True)
            ds.close()
            net.close()
            ctx.close()
    name, limit = card()
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
