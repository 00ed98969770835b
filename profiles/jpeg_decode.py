"""Throughput of fg_dataset_upload_jpeg against Pillow on one host thread.

The 64x64, quality 75, 4:2:0 faces of tests/golden/jpeg_corpus.npz (the dataset/generate_dataset.py form) are repeated
to N files (default 250 000, the size of that training set).  After a warm-up call, one JSON line reports:
  - the end-to-end time of fg_dataset_upload_jpeg on all N files (host parse + upload + decode, best of --rounds),
    as images/s and as GB/s of entropy-coded bytes;
  - the time of each kernel (jpeg_entropy_kernel, jpeg_idct_color_kernel) summed over the call, from torch.profiler
    in a separate call;
  - Pillow decoding the same bytes on one thread (--pillow files, in memory), in images/s;
  - the card's name and power limit, read in the same run.

usage:  python profiles/jpeg_decode.py [--N 250000] [--rounds 3] [--pillow 5000]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import face_generator_b200 as fg  # noqa: E402
import jpeg_utils as JU  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:
        return ["unknown (%s)" % e, "unknown", "unknown"]


def entropy_bytes(b):
    sos = b.index(b"\xff\xda")
    return len(b) - (sos + 2 + int.from_bytes(b[sos + 2:sos + 4], "big")) - 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=250000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pillow", type=int, default=5000)
    a = ap.parse_args()
    faces = [e.bytes for e in JU.load() if e.face]
    files = [faces[i % len(faces)] for i in range(a.N)]
    ent = sum(entropy_bytes(b) for b in files)
    ctx = fg.Context(0, max_batch=16, channels=3)
    ds = DeviceDataset(ctx, shape=(a.N, 3, 64, 64))
    offsets = np.zeros(a.N + 1, np.int64)
    offsets[1:] = np.cumsum([len(b) for b in files])
    data = np.frombuffer(b"".join(files), np.uint8)
    import ctypes as C

    def call():
        failed = C.c_int64(-1)
        rc = ds.lib.fg_dataset_upload_jpeg(ds.h, 0, a.N, data.ctypes.data_as(C.c_void_p),
                                           offsets.ctypes.data_as(C.c_void_p), C.byref(failed))
        assert rc == 0, ds.lib.fg_last_error()

    call()  # warm-up: scratch allocation, module load
    times = []
    for _ in range(a.rounds):
        t0 = time.perf_counter()
        call()  # returns after the decode has finished (it reads back the error flags)
        times.append(time.perf_counter() - t0)
    best = min(times)
    got = ds.download(0, len(faces))
    ref = {e.bytes: e.expected(3) for e in JU.load() if e.face}
    exact = all(np.array_equal(got[i], ref[faces[i]]) for i in range(len(faces)))
    # per kernel, in a separate profiled call
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        for k in ("jpeg_entropy_kernel", "jpeg_idct_color_kernel"):
            if k in ev.key:
                kern[k] = kern.get(k, 0.0) + ev.device_time_total / 1000.0  # ms
    # Pillow, one thread, same bytes in memory
    try:
        from PIL import Image
        n = min(a.pillow, a.N)
        t0 = time.perf_counter()
        for b in files[:n]:
            np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))
        pil = n / (time.perf_counter() - t0)
    except ImportError:
        pil = float("nan")
    name, power, clock = card()
    print(json.dumps({
        "files": a.N, "size": "64x64 q75 4:2:0", "entropy_MB": round(ent / 1e6, 1),
        "call_s": round(best, 4), "calls_s": [round(t, 4) for t in times],
        "images_per_s": round(a.N / best), "entropy_GB_per_s": round(ent / best / 1e9, 3),
        "kernel_ms": {k: round(v, 2) for k, v in kern.items()},
        "kernel_images_per_s": round(a.N / (sum(kern.values()) / 1000.0)) if kern else None,
        "pillow_images_per_s_1thread": round(pil), "speedup_vs_pillow": round(a.N / best / pil, 1) if pil == pil else None,
        "bitwise_equal_to_pillow": bool(exact), "card": name, "power_limit": power, "max_sm_clock": clock}))
    ds.close()
    ctx.close()


if __name__ == "__main__":
    main()
