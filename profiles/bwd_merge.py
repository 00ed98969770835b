"""A/B of option bwd_merge in one process: the train step at batch 256 (graphs on) with G's upsampled-layer
backward as one merged launch (1: G.C2, 2: G.C2 and G.C1) or as separate wgrad and dgrad launches (0).

Each setting is timed three times, interleaved, over 20 steps after 5 warm-up steps with the context's events.  Then
one timed pass per setting reports the per-step time of G.C2's and G.C1's backward (merged launch, or wgrad + dgrad).

    python profiles/bwd_merge.py [--batch 256] [--steps 20] [--settings 1,0,2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--settings", default="1,0,2")
    args = ap.parse_args()
    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_D, NET_G
    B, C = args.batch, 3
    settings = [int(s) for s in args.settings.split(",")]
    rng = np.random.default_rng(1)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    f = lambda a: np.ascontiguousarray(a, np.float32)
    real = ctx.dev_array(f(rng.random((B // 2, C, 32, 32))))
    nD, nG = ctx.dev_array(f(rng.uniform(-1, 1, (B // 2, 100)))), ctx.dev_array(f(rng.uniform(-1, 1, (B, 100))))
    h = fg.hyper_default()
    seed = [0]

    def step():
        seed[0] += 1
        ctx.train_step(h, B, real, nD, nG, None, None, seed[0], want_stats=False)

    ms = {s: [] for s in settings}
    for _ in range(args.rounds):
        for s in settings:
            ctx.set_option("bwd_merge", s)
            for _ in range(args.warmup):
                step()
            ctx.sync()
            ctx.event_record(0)
            for _ in range(args.steps):
                step()
            ctx.event_record(1)
            ctx.sync()
            ms[s].append(ctx.event_elapsed_ms(0, 1) / args.steps)
    layers = {}
    nprof = 5
    for s in settings:
        ctx.set_option("bwd_merge", s)
        for _ in range(args.warmup):
            step()
        ctx.timing_enable(True)  # clears the timers
        for _ in range(nprof):
            step()
        ctx.sync()
        row = {}
        for layer in ("G.C2", "G.C1"):
            for part in ("wgrad+dgrad", "wgrad", "dgrad"):
                name = "%s.%s" % (layer, part)
                t, n = ctx.timing_get(name)
                if part != "wgrad+dgrad":  # the prefix "G.C2.wgrad" also matches the merged timer
                    t -= ctx.timing_get(name + "+dgrad")[0] if part == "wgrad" else 0.0
                row[name] = round(t / nprof, 4)
            row[layer + ".backward"] = round(row[layer + ".wgrad+dgrad"] + row[layer + ".wgrad"] + row[layer + ".dgrad"], 4)
        ctx.timing_enable(False)
        layers[s] = row
    ctx.close()
    out = {"gpu": gpu_info(), "batch": B, "steps": args.steps, "rounds": args.rounds,
           "step_ms": {s: {"mean": round(float(np.mean(v)), 4), "min": round(min(v), 4), "max": round(max(v), 4),
                           "runs": [round(x, 4) for x in v]} for s, v in ms.items()},
           "images_per_s": {s: round(B / (float(np.mean(v)) / 1e3), 1) for s, v in ms.items()},
           "backward_ms_per_step": layers}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
