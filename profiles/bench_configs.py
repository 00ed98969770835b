"""Secondary BASELINE.json configs, measured the same way bench.py measures the headline (CUDA events on the ctx
stream, warm-up, synchronise on both sides); one JSON line per config.  Informational: bench.py stays the headline.

  configs[3]  train_c2f.lua coarse-to-fine 16->32, SpatialConvolutionUpsample path  (batch 32 = script default, and 256)
  configs[4]  sample.lua 1024-image generation-only throughput (chunk 16 = script default, and 1024)
  configs[0]  gray batch 16 train step (the CPU-runnable case) on the GPU, for scale

usage:  python profiles/bench_configs.py [--steps 10] > configs.jsonl
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import layouts as LY  # noqa: E402
from face_generator_b200.lib import NET_D, NET_G  # noqa: E402

# algorithmic conv/linear FLOPs per image and pass (2*Cout*Cin*k*k*H*W), SURVEY.md 8a
C2F_G_FWD = 2 * 1024 * (4 * 64 * 9 + 64 * 64 * 9 + 64 * 128 * 25 + 128 * 256 * 25 + 256 * 3 * 49)
C2F_D_FWD = 2 * (1024 * (3 * 64 * 9 + 64 * 64 * 9) + 256 * (64 * 128 * 9 + 128 * 256 * 9) + 16384 * 512 + 512)
G_FWD = 2105.9e6


def timed(ctx, fn, k):
    ctx.sync()
    ctx.event_record(0)
    for _ in range(k):
        fn()
    ctx.event_record(1)
    ctx.sync()
    return ctx.event_elapsed_ms(0, 1) / k


def c2f(B, steps):
    C = 3
    ctx = fg.Context(0, max_batch=B, channels=C)
    net = fg.C2f(ctx)
    rng = np.random.default_rng(1)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C), rng, 1.0))
    real_diff, cond_r = LY.c2f_pairs(B // 2, C, rng)
    _, cond_f = LY.c2f_pairs(B // 2, C, rng)
    _, cond_G = LY.c2f_pairs(B, C, rng)
    cond_D = np.concatenate([cond_r, cond_f])
    nD = rng.uniform(-1, 1, (B // 2, 1, 32, 32)).astype(np.float32)
    nG = rng.uniform(-1, 1, (B, 1, 32, 32)).astype(np.float32)
    dev = [ctx.dev_array(a) for a in (real_diff, cond_D, nD, cond_G, nG)]
    hyper = fg.hyper_default(D_L1=1e-7, D_L2=0.0)  # train_c2f.lua:26-29
    seed = [0]

    def step():
        seed[0] += 1
        net.train_step(hyper, B, dev[0], dev[1], dev[2], dev[3], dev[4], None, None, seed[0], want_stats=False)

    def step_e2e():
        seed[0] += 1
        return net.train_step(hyper, B, real_diff, cond_D, nD, cond_G, nG, None, None, seed[0], want_stats=True)

    for _ in range(3):
        step()
    l0 = ctx.launches()
    ms = timed(ctx, step, steps)
    launches = (ctx.launches() - l0) // steps
    ms_e2e = timed(ctx, step_e2e, max(3, steps // 2))
    ctx.timing_enable(True)
    for _ in range(2):
        step()
    layers = {}
    for net_, names in (("G", ["c1", "c2", "c3", "c4", "c5"]), ("D", ["c1", "c2", "c3", "c4", "L1", "L2"])):
        for nm in names:
            for kind in ("fwd", "dgrad", "wgrad"):
                t, n = ctx.timing_get("c2f.%s.%s.%s" % (net_, nm, kind))
                if n:
                    layers["%s.%s.%s" % (net_, nm, kind)] = round(t / 2, 4)
    t_all, _ = ctx.timing_get("c2f.")
    ctx.timing_enable(False)
    # executed passes per iteration: G fwd 1.5B + G bwd 2B; D fwd 2B + D dgrad 2B + D wgrad B
    flops = B * (3.5 * C2F_G_FWD + 5.0 * C2F_D_FWD)
    out = {"config": "configs[3] train_c2f.lua colour 3x32x32, batch %d, 1 D-iter + 1 G-iter, Adam" % B,
           "metric": "c2f train images/sec", "value": B / (ms / 1e3), "unit": "images/s", "ms_per_step": ms,
           "e2e": {"value": B / (ms_e2e / 1e3), "unit": "images/s", "ms_per_step": ms_e2e},
           "algorithmic_tflops": flops / (ms / 1e3) / 1e12, "gpu_launches_per_step": int(launches), "dtype": "f32",
           "conv_ms_per_step": round(t_all / 2, 4), "layer_ms_per_step": layers}
    net.close()
    ctx.close()
    return out


def sample(chunk, steps, N=1024):
    C = 3
    ctx = fg.Context(0, max_batch=max(chunk, 4), channels=C)
    rng = np.random.default_rng(2)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    noise = rng.uniform(-1, 1, (N, 100)).astype(np.float32)
    d_noise = ctx.dev_array(noise)
    d_out = ctx.lib.fg_dev_alloc(N * C * 1024 * 4)
    from face_generator_b200.lib import _check

    def run_dev():
        _check(ctx.lib.fg_sample(ctx.h, d_noise, N, chunk, d_out), "fg_sample")

    def run_e2e():
        return ctx.sample(noise, chunk)  # host noise in, host images out

    run_dev()
    ms = timed(ctx, run_dev, steps)
    ms_e2e = timed(ctx, run_e2e, max(2, steps // 2))
    out = {"config": "configs[4] sample.lua %d images, chunk %d (train-mode BN per chunk, sample.lua:69-80)" % (N, chunk),
           "metric": "generation-only images/sec (G forward)", "value": N / (ms / 1e3), "unit": "images/s", "ms_per_call": ms,
           "e2e": {"value": N / (ms_e2e / 1e3), "unit": "images/s", "ms_per_call": ms_e2e, "d2h_bytes": N * C * 4096},
           "algorithmic_tflops": N * G_FWD / (ms / 1e3) / 1e12, "dtype": "f32"}
    ctx.lib.fg_dev_free(d_out)
    ctx.close()
    return out


def train_small(B, C, steps):
    ctx = fg.Context(0, max_batch=B, channels=C)
    rng = np.random.default_rng(3)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    real = rng.random((B // 2, C, 32, 32)).astype(np.float32)
    nD = rng.uniform(-1, 1, (B // 2, 100)).astype(np.float32)
    nG = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
    dev = [ctx.dev_array(a) for a in (real, nD, nG)]
    hyper = fg.hyper_default()
    seed = [0]

    def step():
        seed[0] += 1
        ctx.train_step(hyper, B, dev[0], dev[1], dev[2], None, None, seed[0], want_stats=False)

    for _ in range(3):
        step()
    ms = timed(ctx, step, steps)
    out = {"config": "configs[0] train.lua grayscale 1x32x32 batch %d on the GPU (the reference runs this one on the CPU)" % B,
           "metric": "train images/sec", "value": B / (ms / 1e3), "unit": "images/s", "ms_per_step": ms, "dtype": "f32"}
    ctx.close()
    return out


def train_s16(B, steps):
    """train.lua --scale 16 (G16 / D16_d, models.lua:27-51, :279-316): one adversarial.lua iteration on 16x16 images"""
    C = 3
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    ctx = fg.Context(0, max_batch=B, channels=C)
    net = fg.S16(ctx)
    rng = np.random.default_rng(4)
    nG, nD = net.count(NET_G), net.count(NET_D)
    # fan-in scaled synthetic weights, PReLU slopes 0.25 (single floats are the only size-1 tensors besides the last bias)
    net.set_params(NET_G, (rng.standard_normal(nG) * 0.02).astype(np.float32))
    net.set_params(NET_D, (rng.standard_normal(nD) * 0.02).astype(np.float32))
    real = rng.random((B // 2, C, 16, 16)).astype(np.float32)
    zD = rng.uniform(-1, 1, (B // 2, 100)).astype(np.float32)
    zG = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
    dev = [ctx.dev_array(a) for a in (real, zD, zG)]
    hyper = fg.hyper_default()
    seed = [0]

    def step():
        seed[0] += 1
        net.train_step(hyper, B, dev[0], dev[1], dev[2], None, None, seed[0], want_stats=False)

    def step_e2e():
        seed[0] += 1
        return net.train_step(hyper, B, real, zD, zG, None, None, seed[0], want_stats=True)

    for _ in range(3):
        step()
    ms = timed(ctx, step, steps)
    ms_e2e = timed(ctx, step_e2e, max(3, steps // 2))
    out = {"config": "train.lua --scale 16: colour 3x16x16, batch %d, G16 / D16_d, 1 D-iter + 1 G-iter, Adam" % B,
           "metric": "train images/sec", "value": B / (ms / 1e3), "unit": "images/s", "ms_per_step": ms,
           "e2e": {"value": B / (ms_e2e / 1e3), "unit": "images/s", "ms_per_step": ms_e2e}, "dtype": "f32"}
    net.close()
    ctx.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="", help="c2f | sample | small | s16")
    a = ap.parse_args()
    jobs = [("c2f", lambda: c2f(32, a.steps)), ("c2f", lambda: c2f(256, a.steps)), ("sample", lambda: sample(16, a.steps)),
            ("sample", lambda: sample(1024, a.steps)), ("small", lambda: train_small(16, 1, a.steps)),
            ("s16", lambda: train_s16(256, a.steps))]
    for kind, job in jobs:
        if not a.only or a.only == kind:
            print(json.dumps(job()), flush=True)
