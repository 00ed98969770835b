"""Time of the coarse-to-fine refinement (fg_c2f_refine, sample.lua:176-214) and of the whole pyramid sampler.

fg_c2f_refine on N = 1024 device-resident images, 10 tries, chunk = max_batch / 10, D in training mode (as sample.lua):
  S = 64 from 32x32 inputs, S = 32 from 16x16 inputs and S = 32 from 32x32 inputs (no rescale).
Per configuration one JSON line: ms per 1024 refined images (best of `--rounds` calls, CUDA events after a warm-up
call), refined images/s, then from one more call with the per-launch timers on (fg_timing_get): the ms of
refine_prep + refine_pick and their share of the call, the ms of G's and D's layers, and the algorithmic TFLOP/s of G's
convolutions (2 * Cin * Cout * k^2 per output pixel and layer, summed, over the time of G's convolution launches).
Then sample_pyramid 32 -> 64 and 16 -> 32 -> 64 for 1024 faces end to end (host clock; it returns host images), and
the card's name and power limit, read in the same run.  Parameters are random: the work does not depend on them.

usage:  python profiles/c2f_refine.py [--N 1024] [--max-batch 250] [--rounds 3]
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
from face_generator_b200 import layouts as LY  # noqa: E402
from face_generator_b200.lib import NET_D, NET_G  # noqa: E402
from face_generator_b200.pyramid import sample_pyramid  # noqa: E402

TRIES = 10


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:
        return ["unknown (%s)" % e, "unknown", "unknown"]


def g_flop_per_pixel(C):
    """create_G_d at one output pixel: (C+1)->64 3x3, 64->64 3x3, 64->128 5x5, 128->256 5x5, 256->C 7x7"""
    layers = [(C + 1, 64, 3), (64, 64, 3), (64, 128, 5), (128, 256, 5), (256, C, 7)]
    return sum(2 * ci * co * k * k for ci, co, k in layers)


def c2f_net(ctx, S, rng):
    net = fg.C2f(ctx, S)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(ctx.C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(ctx.C, S), rng, 1.0))
    return net


def refine_dev(ctx, net, images_dev, N, in_size, out_dev, chunk, seed):
    rc = ctx.lib.fg_c2f_refine(net.h, images_dev, N, in_size, TRIES, chunk, 1, None, None, seed, out_dev, None, None)
    if rc != 0:
        raise fg.FGError("fg_c2f_refine: " + ctx.lib.fg_last_error().decode())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1024)
    ap.add_argument("--max-batch", type=int, default=250)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    N, C, chunk = a.N, 3, a.max_batch // TRIES
    name, limit, clock = card()
    rng = np.random.default_rng(0)
    ctx = fg.Context(0, max_batch=a.max_batch, channels=C)
    nets = {32: c2f_net(ctx, 32, rng), 64: c2f_net(ctx, 64, rng)}
    for S, in_size in ((64, 32), (32, 16), (32, 32)):
        net = nets[S]
        images = ctx.dev_array(rng.random((N, C, in_size, in_size)).astype(np.float32))
        out = ctx.dev_array(np.zeros((N, C, S, S), np.float32))
        refine_dev(ctx, net, images, N, in_size, out, chunk, 1)  # warm-up: packs, modules
        best = float("inf")
        for r in range(a.rounds):
            ctx.event_record(0)
            refine_dev(ctx, net, images, N, in_size, out, chunk, 2 + r)
            ctx.event_record(1)
            best = min(best, ctx.event_elapsed_ms(0, 1))
        ctx.timing_enable(True)
        ctx.event_record(0)
        refine_dev(ctx, net, images, N, in_size, out, chunk, 9)
        ctx.event_record(1)
        timed = ctx.event_elapsed_ms(0, 1)
        pre = "c2f." if S == 32 else "c2f%d." % S
        own = ctx.timing_get(pre + "refine_prep")[0] + ctx.timing_get(pre + "refine_pick")[0]
        g_ms, d_ms = ctx.timing_get(pre + "G.")[0], ctx.timing_get(pre + "D.")[0]
        ctx.timing_enable(False)
        flop = N * TRIES * S * S * g_flop_per_pixel(C)
        print(json.dumps(dict(what="fg_c2f_refine", S=S, in_size=in_size, N=N, tries=TRIES, chunk=chunk,
                              ms_per_1024=round(best * 1024 / N, 2), images_per_s=round(N / best * 1e3, 1),
                              timed_call_ms=round(timed, 2), prep_pick_ms=round(own, 3),
                              prep_pick_share=round(own / timed, 4), G_conv_ms=round(g_ms, 2), D_layers_ms=round(d_ms, 2),
                              G_TFLOP=round(flop / 1e12, 2), G_conv_TFLOPs=round(flop / g_ms / 1e9, 1),
                              G_TFLOPs_over_call=round(flop / best / 1e9, 1), gpu=name, power_limit=limit,
                              max_sm_clock=clock)), flush=True)
        ctx.dev_free(images)
        ctx.dev_free(out)
    # the whole sampler: base G, then the levels, host images at the end
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    s16 = fg.S16(ctx)
    s16.set_params(NET_G, (rng.standard_normal(s16.nG) * 0.02).astype(np.float32))
    s16.set_bn_state(np.concatenate([np.zeros(256), np.ones(256), np.zeros(128), np.ones(128)]).astype(np.float32))
    for base, levels, label in ((ctx, [nets[64]], "32->64"), (s16, [nets[32], nets[64]], "16->32->64")):
        sample_pyramid(base, levels, N, TRIES, 16, 0)  # warm-up
        best = float("inf")
        for r in range(a.rounds):
            t0 = time.perf_counter()
            sample_pyramid(base, levels, N, TRIES, 16, 1 + r)
            best = min(best, time.perf_counter() - t0)
        print(json.dumps(dict(what="sample_pyramid", chain=label, N=N, tries=TRIES, ms_per_1024=round(best * 1e3 * 1024 / N, 2),
                              faces_per_s=round(N / best, 1), gpu=name, power_limit=limit, max_sm_clock=clock)), flush=True)
    s16.close()
    for n in nets.values():
        n.close()
    ctx.close()


if __name__ == "__main__":
    main()
