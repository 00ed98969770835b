"""The coarse-to-fine train step (train_c2f.lua) at every pyramid level a 64x64 training set feeds: fine size
S in {16, 32, 64} with coarse size S/2, batch 32 (the script's default) and 256, colour.

For each (S, batch): one ctx and one fg_c2f_create_sized net, a DeviceDataset of 64x64 uint8 images, and two feeds that
run alternately in one process -- "host" (fg_c2f_train_step on host float32 arrays of pairs gathered once, uploaded by
the call) and "device" (fg_c2f_train_step_dataset: draws, pairs and noise on the GPU).  5 warm-up steps each, then
`--rounds` windows of `--steps` steps per feed, timed with CUDA events on the ctx stream.  Then two device-fed steps
with the layer timers on (the names "c2f.*" at S = 32, "c2f16.*" / "c2f64.*" otherwise), the net's device memory
(free memory before and after fg_c2f_create_sized), and the algorithmic FLOPs of one step from the shapes.  One JSON
line per configuration, the card (name, power limit, SM clocks) first.

usage:  python profiles/c2f_sizes.py [--steps 20] [--rounds 3] [--sizes 16,32,64] [--batches 32,256]
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

C = 3
LAYERS = (("G", ("c1", "c2", "c3", "c4", "c5")), ("D", ("c1", "c2", "c3", "c4", "L1", "L2")))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # the numbers are still printed; the card is then unknown
        return {"name": "unknown (%s)" % e}


def fwd_flops(S):
    """algorithmic FLOPs of one image's G and D forward at fine size S (multiply-adds x 2)"""
    g = 2 * S * S * ((C + 1) * 64 * 9 + 64 * 64 * 9 + 64 * 128 * 25 + 128 * 256 * 25 + 256 * C * 49)
    flat = 256 * (S // 4) ** 2
    d = 2 * (S * S * (C * 64 * 9 + 64 * 64 * 9) + (S // 2) ** 2 * (64 * 128 * 9 + 128 * 256 * 9) + flat * 512 + 512)
    return g, d


def windowed(ctx, fn, steps):
    ctx.sync()
    ctx.event_record(0)
    for _ in range(steps):
        fn()
    ctx.event_record(1)
    ctx.sync()
    return ctx.event_elapsed_ms(0, 1) / steps


def run(S, B, steps, rounds, imgs):
    import torch
    cs = S // 2
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.sync()
    free0 = torch.cuda.mem_get_info(0)[0]
    net = fg.C2f(ctx, S)
    ctx.sync()
    net_bytes = free0 - torch.cuda.mem_get_info(0)[0]
    rng = np.random.default_rng(1)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C, S), rng, 1.0))
    ds = DeviceDataset(ctx, imgs)
    hyper = fg.hyper_default(D_L1=1e-7, D_L2=0.0)  # train_c2f.lua:26-29
    Bh, seed = B // 2, [0]
    # host feed: one epoch's worth of pairs gathered once (the host cache of the Lua trainer), rows drawn per step
    n_cache = 1000
    _, coarse, diff = _gather_all(ds, n_cache, B, cs, S)

    def host_step():
        seed[0] += 1
        r, f, g = rng.integers(0, n_cache, Bh), rng.integers(0, n_cache, Bh), rng.integers(0, n_cache, B)
        net.train_step(hyper, B, diff[r], np.concatenate([coarse[r], coarse[f]]),
                       rng.uniform(-1, 1, (Bh, 1, S, S)).astype(np.float32), coarse[g],
                       rng.uniform(-1, 1, (B, 1, S, S)).astype(np.float32), None, None, seed[0])

    def device_step():
        seed[0] += 1
        net.train_step_dataset(ds, hyper, B, cs, seed[0])

    feeds = {"host": host_step, "device": device_step}
    for fn in feeds.values():
        for _ in range(5):
            fn()
    ms = {k: [] for k in feeds}
    for _ in range(rounds):
        for k, fn in feeds.items():
            ms[k].append(windowed(ctx, fn, steps))
    ctx.timing_enable(True)
    for _ in range(2):
        device_step()
    prefix = "c2f." if S == 32 else "c2f%d." % S
    layers = {}
    for net_, names in LAYERS:
        for nm in names:
            for kind in ("fwd", "dgrad", "wgrad"):
                t, n = ctx.timing_get("%s%s.%s.%s" % (prefix, net_, nm, kind))
                if n:
                    layers["%s.%s.%s" % (net_, nm, kind)] = round(t / 2, 4)
    t_all, _ = ctx.timing_get(prefix)
    ctx.timing_enable(False)
    g, d = fwd_flops(S)
    flops = B * (3.5 * g + 5.0 * d)  # executed passes per step: G fwd 1.5B + G bwd 2B; D fwd 2B + D dgrad 2B + D wgrad B
    out = dict(fine_size=S, coarse_size=cs, batch=B, timed_steps=steps * rounds, net_device_mib=round(net_bytes / 2**20, 1),
               G_fwd_gflop_per_image=round(g / 1e9, 3), D_fwd_gflop_per_image=round(d / 1e9, 3),
               step_tflop=round(flops / 1e12, 3), layer_ms_per_step=layers, timed_layers_ms_per_step=round(t_all / 2, 3))
    for k, v in ms.items():
        m = float(np.mean(v))
        out[k] = dict(ms_per_step=round(m, 3), ms_per_step_rounds=[round(x, 3) for x in v], images_per_s=round(B / m * 1e3, 1),
                      algorithmic_tflops=round(flops / (m / 1e3) / 1e12, 2))
    print(json.dumps(out), flush=True)
    ds.close()
    net.close()
    ctx.close()


def _gather_all(ds, n, B, cs, S):
    parts = [ds.gather_c2f(np.arange(s, min(s + B, n)) % ds.N, cs, S) for s in range(0, n, B)]
    return tuple(np.concatenate([p[k] for p in parts]) for k in range(3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="16,32,64")
    ap.add_argument("--batches", default="32,256")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    imgs = np.random.default_rng(0).integers(0, 256, (2000, 3, 64, 64), dtype=np.uint8)
    for S in (int(s) for s in a.sizes.split(",")):
        for B in (int(b) for b in a.batches.split(",")):
            run(S, B, a.steps, a.rounds, imgs)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
