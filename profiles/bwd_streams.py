"""Option "bwd_streams" A/B in one process: the headline step (fg_train_step at batch 256, colour, inputs resident on the
device, bench.py's parameters, replayed CUDA graph) with the weight gradients on their own stream (1) and on the chain
(0), alternated over --rounds rounds of --steps synchronised steps each.  Prints ms per step for every round and the
mean of each setting, then one profiled step of each setting (torch.profiler, CUDA activities): for every stream the
kernels ran on, which kernels, how long they ran and how much of that a kernel of another stream ran too (for the
weight-gradient stream: the time it overlaps the chain and the side stream's generator forward).

The card's name and power limit are printed first; they belong beside any number quoted from this output.  The
profiled steps are not timings (the profiler slows the host); the alternated rounds are.

usage:  python profiles/bwd_streams.py [--rounds 5] [--steps 100] [--batch 256] [--trace-dir DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from step_overlap import card, union  # noqa: E402


def kernels_of(path):
    ev = json.load(open(path)).get("traceEvents", [])
    return [{"ts": float(e["ts"]), "dur": float(e["dur"]), "stream": e.get("args", {}).get("stream", e.get("tid")),
             "name": e["name"]} for e in ev if e.get("cat") == "kernel" and e.get("ph") == "X"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--trace-dir", default=None, help="keep the two Chrome traces here")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_D, NET_G

    B, C = a.batch, 3
    torch.cuda.init()
    print("card: %s" % card())
    ctx = fg.Context(0, max_batch=B, channels=C)
    rng = np.random.default_rng(1)  # bench.py's parameters and inputs
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    rng = np.random.default_rng(100)
    f = lambda x: np.ascontiguousarray(x, np.float32)
    host = (f(rng.random((B // 2, C, 32, 32))), f(rng.uniform(-1, 1, (B // 2, 100))), f(rng.uniform(-1, 1, (B, 100))))
    dev = [ctx.dev_array(x) for x in host]
    hyper = fg.hyper_default()
    seed = [0]

    def step():
        seed[0] += 1
        ctx.train_step(hyper, B, dev[0], dev[1], dev[2], None, None, seed[0], want_stats=False)

    modes = (0, 1)
    for m in modes:  # eager, captured, replayed: both graphs stay cached
        ctx.set_option("bwd_streams", m)
        for _ in range(a.warmup):
            step()
        ctx.sync()
    ms = {m: [] for m in modes}
    for r in range(a.rounds):
        for m in modes:
            ctx.set_option("bwd_streams", m)
            step()
            ctx.sync()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                step()
            ctx.sync()
            ms[m].append((time.perf_counter() - t0) * 1e3 / a.steps)
        print("round %d: %s" % (r, "  ".join("bwd_streams %d %.4f ms" % (m, ms[m][-1]) for m in modes)))
    for m in modes:
        print("bwd_streams %d: mean %.4f ms/step, range %.4f-%.4f" % (m, np.mean(ms[m]), min(ms[m]), max(ms[m])))
    print("gain: %.2f %%" % (100.0 * (np.mean(ms[0]) - np.mean(ms[1])) / np.mean(ms[0])))

    tdir = a.trace_dir or tempfile.mkdtemp()
    os.makedirs(tdir, exist_ok=True)
    streams = {}
    per_mode = {}
    for m in modes:
        ctx.set_option("bwd_streams", m)
        for _ in range(3):
            step()
        ctx.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            ctx.sync()
        path = os.path.join(tdir, "bwd_streams%d.json" % m)
        prof.export_chrome_trace(path)
        ks = kernels_of(path)
        per_mode[m] = ks
        streams[m] = sorted({k["stream"] for k in ks}, key=str)
        t0, t1 = min(k["ts"] for k in ks), max(k["ts"] + k["dur"] for k in ks)
        print("bwd_streams %d profiled step: %d kernels, span %.1f us, streams %s" % (m, len(ks), t1 - t0, streams[m]))
    # a replayed graph may run its branches on streams of its own, so every stream of each step is listed with the
    # kernels it ran: the weight-gradient stream is the one of bwd_streams 1 that runs wgrad_tc_kernel
    for m in modes:
        ks = per_mode[m]
        for s in streams[m]:
            mine = [(k["ts"], k["ts"] + k["dur"]) for k in ks if k["stream"] == s]
            other = [(k["ts"], k["ts"] + k["dur"]) for k in ks if k["stream"] != s]
            both = union(mine) + union(other) - union(mine + other)  # a kernel of s and one of another stream run
            names = sorted({k["name"].split("<")[0].split("(")[0] for k in ks if k["stream"] == s})
            print("bwd_streams %d stream %s%s: %d kernels, busy %.1f us, beside another stream %.1f us; kernels: %s"
                  % (m, s, " (new)" if m == 1 and s not in streams[0] else "", len(mine), union(mine), both,
                     ", ".join(names)[:300]))
    ctx.close()


if __name__ == "__main__":
    main()
