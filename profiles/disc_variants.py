"""Time of the captured device-fed train step (fg_train_step_dataset / fg_s16_train_step_dataset) on each discriminator
of models.lua, colour, batch 256:
  32x32  create_D32b (the default) and create_D32
  s16    create_D16_d (the default), create_D16, create_D16_b and create_D16_c
Every net gets 3 warm-up calls (eager, captured, replayed), then `--rounds` windows of `--steps` calls, the nets of a
size alternating window by window, timed with CUDA events on the ctx stream.  Every call reads its statistics, as the
Lua loop does.  One JSON line per net with the median ms per step, then the card's name and power limit, read in the
same run.

usage:  python profiles/disc_variants.py [--steps 10] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402

C, B = 3, 256
SIZES = [("32x32", ["create_D32b", "create_D32"]),
         ("s16", ["create_D16_d", "create_D16", "create_D16_b", "create_D16_c"])]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()[0]
    return [s.strip() for s in out.split(",")]


def windowed(ctx, fn, steps):
    ctx.sync()
    ctx.event_record(0)
    for _ in range(steps):
        fn()
    ctx.event_record(1)
    ctx.sync()
    return ctx.event_elapsed_ms(0, 1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    imgs = np.random.default_rng(0).integers(0, 256, (4096, C, 32, 32), dtype=np.uint8)
    h = fg.hyper_default()
    for kind, names in SIZES:
        nets = []
        for name in names:
            rng = np.random.default_rng(1)
            if kind == "32x32":
                ctx = fg.Context(0, max_batch=B, channels=C, discriminator=name)
                net = ctx
            else:
                ctx = fg.Context(0, max_batch=B, channels=C)
                net = fg.S16(ctx, discriminator=name)
            net.set_params(fg.lib.NET_G, rng.uniform(-0.05, 0.05, net.nG).astype(np.float32))
            net.set_params(fg.lib.NET_D, rng.uniform(-0.02, 0.02, net.nD).astype(np.float32))
            ds = DeviceDataset(ctx, imgs)
            seed = [100]

            def step(ctx=ctx, net=net, ds=ds, seed=seed):
                seed[0] += 1
                return ds.train_step(h, B, seed[0]) if net is ctx else net.train_step_dataset(ds, h, B, seed[0])
            for _ in range(3):
                step()
            nets.append((name, ctx, net, ds, step, []))
        for _ in range(a.rounds):
            for name, ctx, net, ds, step, times in nets:
                times.append(windowed(ctx, step, a.steps))
        for name, ctx, net, ds, step, times in nets:
            print(json.dumps({"nets": kind, "discriminator": name, "batch": B, "channels": C,
                              "ms_per_step": round(float(np.median(times)), 3),
                              "ms_min": round(min(times), 3), "ms_max": round(max(times), 3),
                              "D_params": net.nD}), flush=True)
            ds.close()
            if net is not ctx:
                net.close()
            ctx.close()
    name, limit = card()
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
