"""Time of one loop body with several D and G iterations (train.lua / train_c2f.lua --D_iterations, --G_iterations).

For (d, g) in (1, 1), (2, 1), (1, 2), (2, 2), on
  32x32  the 32x32 nets at batch 256
  s16    the --scale 16 nets at batch 256
  c2f    the coarse-to-fine nets at S = 32, batch 32 and 256 (--coarseSize 16)
and two feeds:
  host   host float32 inputs stacked per iteration, uploaded by fg_*_train_step_iters (fg_*_train_step for 1 + 1)
  device fg_*_train_step_dataset_iters on a DeviceDataset (fg_*_train_step_dataset for 1 + 1): draws inside the step
Every call reads its statistics, as the Lua loops do.  All eight variants of a configuration run alternately in one
process: 3 warm-up calls each (eager, captured, replayed), then `--rounds` windows of `--steps` calls per variant, timed
with CUDA events on the ctx stream.  One JSON line per variant with ms per loop body and the kernels one call counts
(fg_kernel_launches), then the card's name and power limit, read in the same run.

usage:  python profiles/iterations.py [--steps 5] [--rounds 4]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import layouts as LY  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from face_generator_b200.lib import NET_D, NET_G  # noqa: E402

C, CS = 3, 16
ITERS = [(1, 1), (2, 1), (1, 2), (2, 2)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:  # the numbers are still printed; the card is then unknown
        return "unknown (%s)" % e, "unknown"


def windowed(ctx, fn, steps):
    ctx.sync()
    ctx.event_record(0)
    for _ in range(steps):
        fn()
    ctx.event_record(1)
    ctx.sync()
    return ctx.event_elapsed_ms(0, 1) / steps


def host_inputs(rng, kind, B, d, g, S):
    f = lambda a: np.ascontiguousarray(a, np.float32)
    Bh = B // 2
    if kind in ("32x32", "s16"):
        return [f(rng.random((d, Bh, C, S, S))), f(rng.uniform(-1, 1, (d, Bh, 100))), f(rng.uniform(-1, 1, (g, B, 100)))]
    return [f(rng.uniform(-0.3, 0.3, (d, Bh, C, S, S))), f(rng.random((d, B, C, S, S))), f(rng.uniform(-1, 1, (d, Bh, 1, S, S))),
            f(rng.random((g, B, C, S, S))), f(rng.uniform(-1, 1, (g, B, 1, S, S)))]


def run(kind, B, imgs, steps, rounds):
    ctx = fg.Context(0, max_batch=B, channels=C)
    rng = np.random.default_rng(1)
    if kind == "32x32":
        net, S = ctx, 32
        net.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
        net.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    elif kind == "s16":
        net, S = fg.S16(ctx), 16
        net.set_params(NET_G, (rng.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32))
        net.set_params(NET_D, (rng.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32))
    else:
        net, S = fg.C2f(ctx), 32
        net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
        net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C), rng, 1.0))
    ds = DeviceDataset(ctx, imgs)
    hyper = fg.hyper_default()
    seed = [0]
    variants = {}
    for d, g in ITERS:
        inp = host_inputs(rng, kind, B, d, g, S)

        def host(d=d, g=g, inp=inp):
            seed[0] += 1
            if (d, g) == (1, 1):
                net.train_step(hyper, B, *[a[0] for a in inp], None, None, seed[0])
            else:
                net.train_step_iters(hyper, B, d, g, *inp, None, None, seed[0])

        def device(d=d, g=g):
            seed[0] += 1
            one = (d, g) == (1, 1)
            if kind == "32x32":
                ds.train_step(hyper, B, seed[0]) if one else ds.train_step_iters(hyper, B, d, g, seed[0])
            elif kind == "s16":
                net.train_step_dataset(ds, hyper, B, seed[0]) if one else net.train_step_dataset_iters(ds, hyper, B, d, g, seed[0])
            elif one:
                net.train_step_dataset(ds, hyper, B, CS, seed[0])
            else:
                net.train_step_dataset_iters(ds, hyper, B, d, g, CS, seed[0])

        variants[(d, g, "host")] = host
        variants[(d, g, "device")] = device
    launches = {}
    for k, fn in variants.items():
        for _ in range(3):  # eager, captured, replayed
            fn()
        l0 = ctx.launches()
        fn()
        launches[k] = ctx.launches() - l0
    res = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            res[k].append(windowed(ctx, fn, steps))
    for (d, g, feed), r in res.items():
        ms = float(np.mean(r))
        print(json.dumps(dict(trainer=kind, batch=B, D_iterations=d, G_iterations=g, feed=feed, timed_calls=steps * len(r),
                              ms_per_call=round(ms, 3), ms_per_call_rounds=[round(x, 3) for x in r],
                              kernels_per_call=launches[(d, g, feed)])), flush=True)
    ds.close()
    if net is not ctx:
        net.close()
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=4, help="alternating windows per variant")
    a = ap.parse_args()
    assert a.steps * a.rounds >= 20, "time at least 20 calls per variant"
    imgs = np.random.default_rng(0).integers(0, 256, (1000, C, 64, 64), dtype=np.uint8)
    run("32x32", 256, imgs, a.steps, a.rounds)
    run("s16", 256, imgs, a.steps, a.rounds)
    for B in (32, 256):
        run("c2f", B, imgs, a.steps, a.rounds)
    name, limit = card()
    print(json.dumps(dict(card=name, power_limit=limit)), flush=True)


if __name__ == "__main__":
    main()
