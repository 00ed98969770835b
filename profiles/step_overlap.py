"""Where the headline step's time goes across streams: torch.profiler (CUDA activities) over a few replayed
fg_train_step calls at batch 256 (colour, inputs resident on the device, bench.py's parameters), one synchronised call
per step.  Per step it prints every kernel (stream, start and end in us from the step's first kernel, grid, name), then:

  span          first kernel start to last kernel end
  busy          time at least one kernel runs (the union of the kernel intervals)
  overlap       time at least two kernels run at once, and the part of it where they run on different streams
  gaps          the idle time between the kernels of each stream, and of the device as a whole (span - busy)
  under a wave  the kernels with fewer CTAs than the card has SMs: count and summed duration

Profile runs only: the profiler slows the host and the numbers here are not step timings (bench.py's are).  The card's
name and power limit are printed first; they belong beside any number quoted from this output.

usage:  python profiles/step_overlap.py [--steps 3] [--batch 256] [--lib path/to/libfg_b200.so] [--trace out.json]
        [--quiet: the summaries only]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the trace does not depend on it
        return "nvidia-smi unavailable (%s)" % e


def union(iv):
    """total length of the union of intervals [(start, end)]"""
    tot, cur_s, cur_e = 0.0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    return tot + (cur_e - cur_s if cur_e is not None else 0.0)


def overlap(iv):
    """time covered by at least two of the intervals"""
    pts = sorted([(s, 1) for s, _ in iv] + [(e, -1) for _, e in iv])
    tot, depth, last = 0.0, 0, None
    for t, d in pts:
        if depth >= 2:
            tot += t - last
        depth += d
        last = t
    return tot


def summarise(kernels, sms):
    t0 = min(k["ts"] for k in kernels)
    iv = [(k["ts"], k["ts"] + k["dur"]) for k in kernels]
    by_stream = {}
    for k in kernels:
        by_stream.setdefault(k["stream"], []).append(k)
    cross = 0.0  # overlap between streams: all overlap minus what each stream overlaps with itself
    if len(by_stream) > 1:
        cross = overlap(iv) - sum(overlap([(k["ts"], k["ts"] + k["dur"]) for k in ks]) for ks in by_stream.values())
    gaps = {}
    for s, ks in by_stream.items():
        ks = sorted(ks, key=lambda k: k["ts"])
        span = ks[-1]["ts"] + ks[-1]["dur"] - ks[0]["ts"]
        gaps[s] = {"kernels": len(ks), "span_us": span,
                   "gaps_us": span - union([(k["ts"], k["ts"] + k["dur"]) for k in ks])}
    small = [k for k in kernels if k["ctas"] < sms]
    return {"kernels": len(kernels), "span_us": max(e for _, e in iv) - t0, "busy_us": union(iv),
            "overlap_us": overlap(iv), "cross_stream_overlap_us": cross, "streams": gaps,
            "under_one_wave": {"kernels": len(small), "sum_us": sum(k["dur"] for k in small)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--lib", default=None, help="the libfg_b200.so to load (default: the tree's)")
    ap.add_argument("--trace", default=None, help="also keep the Chrome trace here")
    ap.add_argument("--quiet", action="store_true")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function

    from face_generator_b200.lib import load_library
    load_library(a.lib)
    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_D, NET_G

    B, C = a.batch, 3
    torch.cuda.init()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print("card: %s  (%d SMs)" % (card(), sms))
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
        ctx.sync()

    for _ in range(a.warmup):  # eager, captured, replayed
        step()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            with record_function("step%d" % i):
                step()
    path = a.trace or os.path.join(tempfile.mkdtemp(), "step_overlap.json")
    prof.export_chrome_trace(path)
    ev = json.load(open(path)).get("traceEvents", [])
    steps = sorted([e for e in ev if e.get("name", "").startswith("step") and e.get("ph") == "X" and
                    e.get("cat") == "user_annotation"], key=lambda e: e["ts"])
    kernels = []
    for e in ev:
        if e.get("cat") != "kernel" or e.get("ph") != "X":
            continue
        g = e.get("args", {}).get("grid", [1, 1, 1])
        kernels.append({"ts": float(e["ts"]), "dur": float(e["dur"]), "stream": e.get("args", {}).get("stream", e.get("tid")),
                        "ctas": int(np.prod(g)), "grid": g, "name": e["name"]})
    for i, s in enumerate(steps):
        ks = sorted([k for k in kernels if s["ts"] <= k["ts"] <= s["ts"] + s["dur"]], key=lambda k: k["ts"])
        if not ks:
            print("step %d: no kernels recorded" % i)
            continue
        t0 = ks[0]["ts"]
        if not a.quiet:
            print("step %d kernels: stream  start_us  end_us  grid  name" % i)
            for k in ks:
                print("  %6s %9.1f %9.1f  %-14s %s" % (k["stream"], k["ts"] - t0, k["ts"] - t0 + k["dur"],
                                                      "x".join(map(str, k["grid"])), k["name"][:100]))
        print("step %d summary: %s" % (i, json.dumps(summarise(ks, sms))))
    ctx.close()


if __name__ == "__main__":
    main()
