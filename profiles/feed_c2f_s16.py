"""Host-fed versus device-fed train steps of the coarse-to-fine trainer (train_c2f.lua) and train.lua --scale 16.

host   the way lua/adversarial_c2f_b200.lua and lua/adversarial_b200.lua feed the step: a host float32 cache of the
       epoch's images (the coarse / diff tensors of dataset_c2f.lua _toResult, or the 16x16 images of dataset.lua),
       per step a random index draw, row copies into the batch tensors, uniform noise on the host, and host pointers
       into fg_c2f_train_step / fg_s16_train_step (which upload them).
device fg_c2f_train_step_dataset / fg_s16_train_step_dataset on a DeviceDataset of the same images (uint8 64x64).

Both variants read the step statistics every step, as the Lua loops do, so any host work shows up in the step time.
They run alternately in one process: 5 warm-up steps each, then `--rounds` windows of `--steps` steps per variant,
timed with CUDA events on the ctx stream (fg_event_record).  The input assembly alone is timed the same way: for
"host" the host-side batch assembly plus the upload of the five (c2f) / three (s16) inputs, for "device" the draw,
pair-gather and noise kernels the device-fed step launches.  One JSON line per configuration, then the card.

usage:  python profiles/feed_c2f_s16.py [--steps 5] [--rounds 4]
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
from face_generator_b200.lib import NET_D, NET_G, _check  # noqa: E402

N_EPOCH, C, CS = 1000, 3, 16  # train_c2f.lua / train.lua defaults: --N_epoch 1000, colour, --coarseSize 16


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


def compare(ctx, variants, steps, rounds, warmup=5):
    """variants: {name: (step_fn, assemble_fn)}; alternates them; ms per step / per assembly for each round"""
    for step, _ in variants.values():
        for _ in range(warmup):
            step()
    res = {k: {"step": [], "assemble": []} for k in variants}
    for _ in range(rounds):
        for k, (step, assemble) in variants.items():
            res[k]["step"].append(windowed(ctx, step, steps))
            res[k]["assemble"].append(windowed(ctx, assemble, steps))
    return res


def report(trainer, B, res, steps):
    for k, r in res.items():
        ms = float(np.mean(r["step"]))
        print(json.dumps(dict(trainer=trainer, batch=B, feed=k, timed_steps=steps * len(r["step"]), ms_per_step=round(ms, 3),
                              ms_per_step_rounds=[round(x, 3) for x in r["step"]], images_per_s=round(B / ms * 1e3, 1),
                              input_assembly_ms=round(float(np.mean(r["assemble"])), 3))), flush=True)


def c2f(imgs, B, steps, rounds):
    ctx = fg.Context(0, max_batch=B, channels=C)
    net = fg.C2f(ctx)
    rng = np.random.default_rng(1)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C), rng, 1.0))
    ds = DeviceDataset(ctx, imgs)
    hyper = fg.hyper_default(D_L1=1e-7, D_L2=0.0)  # train_c2f.lua:26-29
    # the host cache of one epoch (TRAIN_DATA = _toResult of N_epoch images)
    coarse, diff = np.empty((N_EPOCH, C, 32, 32), np.float32), np.empty((N_EPOCH, C, 32, 32), np.float32)
    for s in range(0, N_EPOCH, B):
        idx = np.arange(s, min(s + B, N_EPOCH))
        _, coarse[idx], diff[idx] = ds.gather_c2f(idx, CS)
    Bh, seed = B // 2, [0]
    dev = [ctx.dev_array(np.zeros(n, np.float32)) for n in (Bh * C * 1024, B * C * 1024, Bh * 1024, B * C * 1024, B * 1024)]
    didx = ctx.dev_array(np.zeros(B, np.float32))  # int32 indices, same byte size

    def host_inputs():  # adversarial_c2f_b200.lua:46-61
        r, f, g = rng.integers(0, N_EPOCH, Bh), rng.integers(0, N_EPOCH, Bh), rng.integers(0, N_EPOCH, B)
        return (diff[r], np.concatenate([coarse[r], coarse[f]]), rng.uniform(-1, 1, (Bh, 1, 32, 32)).astype(np.float32),
                coarse[g], rng.uniform(-1, 1, (B, 1, 32, 32)).astype(np.float32))

    def host_step():
        seed[0] += 1
        net.train_step(hyper, B, *host_inputs(), None, None, seed[0])

    def host_assemble():
        for p, a in zip(dev, host_inputs()):
            _check(ctx.lib.fg_memcpy(ctx.h, p, a.ctypes.data, a.nbytes), "fg_memcpy")

    def device_step():
        seed[0] += 1
        net.train_step_dataset(ds, hyper, B, CS, seed[0])

    def device_assemble():  # the launches of fg_c2f_train_step_dataset before the step proper
        lib, s = ctx.lib, 8 * (seed[0] + 1)
        for k, (n, out) in enumerate(((Bh, (None, dev[1], dev[0])), (Bh, (None, dev[1] + Bh * C * 4096, None)),
                                      (B, (None, dev[3], None)))):
            _check(lib.fg_dataset_draw(ds.h, s + k, n, didx), "fg_dataset_draw")
            _check(lib.fg_dataset_gather_c2f(ds.h, didx, n, CS, *out), "fg_dataset_gather_c2f")
        _check(lib.fg_noise_uniform(ctx.h, s + 3, Bh * 1024, dev[2]), "fg_noise_uniform")
        _check(lib.fg_noise_uniform(ctx.h, s + 4, B * 1024, dev[4]), "fg_noise_uniform")

    res = compare(ctx, {"host": (host_step, host_assemble), "device": (device_step, device_assemble)}, steps, rounds)
    report("c2f", B, res, steps)
    for p in dev + [didx]:
        ctx.dev_free(p)
    ds.close()
    net.close()
    ctx.close()


def s16(imgs, B, steps, rounds):
    ctx = fg.Context(0, max_batch=B, channels=C)
    net = fg.S16(ctx)
    rng = np.random.default_rng(2)
    net.set_params(NET_G, (rng.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32))
    net.set_params(NET_D, (rng.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32))
    ds = DeviceDataset(ctx, imgs)
    hyper = fg.hyper_default()
    cache = np.concatenate([ds.gather(np.arange(s, min(s + B, N_EPOCH)), 16) for s in range(0, N_EPOCH, B)])
    Bh, seed = B // 2, [0]
    dev = [ctx.dev_array(np.zeros(n, np.float32)) for n in (Bh * C * 256, Bh * 100, B * 100)]
    didx = ctx.dev_array(np.zeros(B, np.float32))

    def host_inputs():  # adversarial_b200.lua:74-80
        return (cache[rng.integers(0, N_EPOCH, Bh)], rng.uniform(-1, 1, (Bh, 100)).astype(np.float32),
                rng.uniform(-1, 1, (B, 100)).astype(np.float32))

    def host_step():
        seed[0] += 1
        net.train_step(hyper, B, *host_inputs(), None, None, seed[0])

    def host_assemble():
        for p, a in zip(dev, host_inputs()):
            _check(ctx.lib.fg_memcpy(ctx.h, p, a.ctypes.data, a.nbytes), "fg_memcpy")

    def device_step():
        seed[0] += 1
        net.train_step_dataset(ds, hyper, B, seed[0])

    def device_assemble():  # the launches of fg_s16_train_step_dataset before the step proper
        lib, s = ctx.lib, 4 * (seed[0] + 1)
        _check(lib.fg_dataset_draw(ds.h, s, Bh, didx), "fg_dataset_draw")
        _check(lib.fg_dataset_gather_sized(ds.h, didx, Bh, 16, dev[0]), "fg_dataset_gather_sized")
        _check(lib.fg_noise_uniform(ctx.h, s + 1, Bh * 100, dev[1]), "fg_noise_uniform")
        _check(lib.fg_noise_uniform(ctx.h, s + 2, B * 100, dev[2]), "fg_noise_uniform")

    res = compare(ctx, {"host": (host_step, host_assemble), "device": (device_step, device_assemble)}, steps, rounds)
    report("s16", B, res, steps)
    for p in dev + [didx]:
        ctx.dev_free(p)
    ds.close()
    net.close()
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="steps per timed window")
    ap.add_argument("--rounds", type=int, default=4, help="alternating windows per variant")
    a = ap.parse_args()
    assert a.steps * a.rounds >= 20, "time at least 20 steps per variant"
    imgs = np.random.default_rng(0).integers(0, 256, (N_EPOCH, C, 64, 64), dtype=np.uint8)
    for B in (32, 256):
        c2f(imgs, B, a.steps, a.rounds)
    s16(imgs, 256, a.steps, a.rounds)
    name, limit = card()
    print(json.dumps(dict(card=name, power_limit=limit)), flush=True)


if __name__ == "__main__":
    main()
