"""Time of one sample.lua run on the GPU (face_generator_b200.sheets.sample_run's work): N = 1024 images, chunk 16, for
the 3x32x32 nets and for --scale 16, without neighbours.

For each base, after a warm-up run, one JSON line reports (best of --rounds, CUDA events on the ctx stream):
  - generate (noise + G forward), score (the two live-dropout D passes), grid (the five fg_image_grid calls into one
    device buffer) and encode (the five fg_jpeg_encode calls, both coding passes, bytes to the host), and the whole
    sample_run writing its files into a temporary directory (host clock);
  - the encode of the largest sheet (random1024: 1024x1024 at 32x32, 512x512 at 16x16) on the one-CTA and on the
    multi-CTA entropy coder (fg_set_option "jpeg_route" 1 / 2), and the device time of each encoder kernel on that
    sheet under both routes, from torch.profiler in separate calls;
  - Pillow's Image.save(quality=75) of the same five sheets on one host thread, with its bytes checked equal;
  - the card's name, power limit and max SM clock, read in the same run.

usage:  python profiles/sample_sheets.py [--rounds 5]
"""
import argparse
import ctypes as C
import io
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import layouts as LY, sheets  # noqa: E402
from face_generator_b200.lib import NET_D, NET_G, NOISE_DIM, S16, _check  # noqa: E402
from jpeg_decode import card  # noqa: E402

ENC_KERNELS = ("jpeg_fdct_kernel", "jpeg_huff_kernel", "jpeg_stuff_kernel", "jpeg_blen_kernel", "jpeg_scan_kernel",
               "jpeg_zero_kernel", "jpeg_pack_kernel", "jpeg_ffcount_kernel", "jpeg_scatter_kernel")
N, CHUNK = 1024, 16


def make_base(ctx, s16):
    rng = np.random.default_rng(5)
    if s16:
        from oracle import oracle_s16 as OS
        base = S16(ctx)
        base.set_params(NET_G, LY.trained_like_init((OS.G_layout(3), OS.G_param_count(3)), rng, 1.0).astype(np.float32))
        base.set_params(NET_D, LY.trained_like_init((OS.D_layout(3), OS.D_param_count(3)), rng, 0.8).astype(np.float32))
        return base
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(3), rng, slope=0.25).astype(np.float32))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(3), rng, 1.4, slope=0.25).astype(np.float32))
    return ctx


def phases(ctx, base, s16, rounds):
    """per-phase milliseconds (best of rounds) of sample_run's work, and the five sheets [C][Hg][Wg] uint8"""
    lib, S = ctx.lib, (16 if s16 else 32)
    per = 3 * S * S
    noise, imgs = lib.fg_dev_alloc(4 * N * NOISE_DIM), lib.fg_dev_alloc(4 * N * per)
    out = lib.fg_dev_alloc(3 * (32 * S) ** 2)
    streams = sheets.run_streams(1, 1)
    dimg = sheets.DeviceImages(imgs, (N, 3, S, S))
    best = {}
    grids = []
    for r in range(rounds + 1):
        ms = {}
        ctx.event_record(0)
        _check(lib.fg_noise_uniform(ctx.h, streams[0], N * NOISE_DIM, noise), "fg_noise_uniform")
        if s16:
            for s in range(0, N, CHUNK):
                _check(lib.fg_s16_G_forward(base.h, noise + 4 * s * NOISE_DIM, CHUNK, 1, imgs + 4 * s * per), "G")
        else:
            _check(lib.fg_sample(ctx.h, noise, N, CHUNK, imgs), "fg_sample")
        ctx.event_record(1)
        preds = []
        for k in (1, 2):
            p = np.empty(N, np.float32)
            score = lib.fg_s16_D_score if s16 else lib.fg_D_score
            _check(score(base.h, imgs, N, CHUNK, 1, streams[k], p.ctypes.data_as(C.c_void_p)), "score")
            preds.append(p)
        ctx.event_record(2)
        order = [sheets.permutation(streams[3], N)[:256], None, np.argsort(-preds[0], kind="stable")[:64],
                 np.argsort(preds[1], kind="stable")[:64], sheets.permutation(streams[4], N)[:64]]
        nrows = (16, 32, 8, 8, 8)
        t_grid = t_enc = 0.0
        files = []
        for o, nrow in zip(order, nrows):
            Hg, Wg = sheets.grid_size(ctx, dimg.shape, nrow, 0, N if o is None else o.size)
            ctx.event_record(3)
            sheets.image_grid(ctx, dimg, nrow, 0, o, out=out)
            ctx.event_record(4)
            files.append(sheets.encode_jpeg(ctx, out, 75, shape=(3, Hg, Wg))[0])
            ctx.event_record(5)
            ctx.sync()
            t_grid += ctx.event_elapsed_ms(3, 4)
            t_enc += ctx.event_elapsed_ms(4, 5)
            if r == 0:
                g = np.empty((3, Hg, Wg), np.uint8)
                _check(lib.fg_memcpy(ctx.h, g.ctypes.data_as(C.c_void_p), out, g.nbytes), "fg_memcpy")
                grids.append((g, files[-1]))
        ctx.sync()
        ms = dict(generate=ctx.event_elapsed_ms(0, 1), score_x2=ctx.event_elapsed_ms(1, 2), grid_x5=t_grid, encode_x5=t_enc)
        if r:  # round 0 is the warm-up
            best = {k: min(v, best.get(k, v)) for k, v in ms.items()}
    for p in (noise, imgs, out):
        lib.fg_dev_free(p)
    return {k: round(v, 3) for k, v in best.items()}, grids


def routes(ctx, sheet, rounds):
    """encode milliseconds (best of rounds, host clock: the call returns synchronised) and per-kernel device ms of the
    largest sheet on the one-CTA (1) and multi-CTA (2) entropy coders"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib = ctx.lib
    dev = lib.fg_dev_alloc(sheet.nbytes)
    _check(lib.fg_memcpy(ctx.h, dev, sheet.ctypes.data_as(C.c_void_p), sheet.nbytes), "fg_memcpy")
    res = {}
    for route in (1, 2):
        ctx.set_option("jpeg_route", route)
        enc = lambda: sheets.encode_jpeg(ctx, dev, 75, shape=sheet.shape)[0]
        first = enc()
        ts = []
        for _ in range(rounds):
            t0 = time.perf_counter()
            assert enc() == first
            ts.append((time.perf_counter() - t0) * 1e3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            enc()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            for k in ENC_KERNELS:
                if k in ev.key:
                    kern[k] = round(kern.get(k, 0.0) + ev.device_time_total / 1000.0, 3)
        res[route] = dict(encode_ms=round(min(ts), 3), kernel_ms=kern, file=first)
    ctx.set_option("jpeg_route", 0)
    lib.fg_dev_free(dev)
    assert res[1]["file"] == res[2]["file"]
    return {("one_cta" if k == 1 else "multi_cta"): {a: b for a, b in v.items() if a != "file"} for k, v in res.items()}


def pillow(grids):
    try:
        from PIL import Image
    except ImportError:
        return None, None
    t0 = time.perf_counter()
    out = []
    for g, _ in grids:
        buf = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(g.transpose(1, 2, 0))).save(buf, "JPEG", quality=75)
        out.append(buf.getvalue())
    return round((time.perf_counter() - t0) * 1e3, 2), out == [f for _, f in grids]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    name, power, clock = card()
    ctx = fg.Context(0, max_batch=CHUNK, channels=3)
    for s16 in (False, True):
        base = make_base(ctx, s16)
        ph, grids = phases(ctx, base, s16, a.rounds)
        with tempfile.TemporaryDirectory() as tmp:
            sheets.sample_run(base, 1, tmp, N=N, chunk=CHUNK, seed=1)  # warm-up
            ts = []
            for r in range(a.rounds):
                t0 = time.perf_counter()
                sheets.sample_run(base, 2 + r, tmp, N=N, chunk=CHUNK, seed=1)
                ts.append((time.perf_counter() - t0) * 1e3)
        big = max((g for g, _ in grids), key=lambda g: g.size)
        pil_ms, equal = pillow(grids)
        print(json.dumps({
            "base": "scale16 3x16x16" if s16 else "3x32x32", "N": N, "chunk": CHUNK, "phases_ms": ph,
            "sample_run_ms": round(min(ts), 2), "sample_run_rounds_ms": [round(t, 2) for t in ts],
            "largest_sheet": list(big.shape), "largest_sheet_encode": routes(ctx, big, a.rounds),
            "sheet_bytes": [len(f) for _, f in grids], "pillow_encode_x5_ms_1thread": pil_ms,
            "bytes_equal_to_pillow": equal, "card": name, "power_limit": power, "max_sm_clock": clock}))
        if s16:
            base.close()
    ctx.close()


if __name__ == "__main__":
    main()
