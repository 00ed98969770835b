"""Throughput of fg_dataset_encode_jpeg and fg_dataset_jpeg_roundtrip against Pillow on one host thread.

N rows of 3x64x64 (default 264 660, the size of generate_dataset.py's out_aug_64x64), made of 160 distinct hashed
images of every kind in tests/jpeg_enc_ref.py, are encoded at quality 75.  After a warm-up call of each, one JSON line
reports:
  - the end-to-end time of DeviceDataset.encode_jpeg on all N rows (both coding passes, the copy to host bytes and the
    split into per-file bytes objects) and of jpeg_roundtrip in place, best of --rounds;
  - the time of each kernel summed over one call of each, from torch.profiler in separate calls;
  - Pillow's Image.save(quality=75) of the same rows on one thread (--pillow rows), in images/s, with its bytes
    checked equal to the GPU's in the same run;
  - the card's name, power limit and max SM clock, read in the same run.

usage:  python profiles/jpeg_encode.py [--N 264660] [--rounds 3] [--pillow 5000]
"""
import argparse
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import face_generator_b200 as fg  # noqa: E402
import jpeg_enc_ref as R  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from jpeg_decode import card  # noqa: E402

KERNELS = ("jpeg_fdct_kernel", "jpeg_huff_kernel", "jpeg_stuff_kernel", "jpeg_idct_color_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=264660)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pillow", type=int, default=5000)
    a = ap.parse_args()
    base = np.stack([R.content(R.KINDS[k % len(R.KINDS)], 900 + k, 3, 64, 64) for k in range(160)])
    order = R.hash_u32(77, a.N) % len(base)
    ctx = fg.Context(0, max_batch=16, channels=3)
    ds = DeviceDataset(ctx, base[order])

    def timed(f):
        f()  # warm-up: scratch allocation, module load
        ts = []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            f()  # both entry points return once their work is done
            ts.append(time.perf_counter() - t0)
        return ts

    files = []
    t_enc = timed(lambda: files.__setitem__(slice(None), ds.encode_jpeg(0, a.N, 75)))
    total = sum(len(b) for b in files)
    t_rt = timed(lambda: ds.jpeg_roundtrip(0, a.N, 75))  # in place: each round codes the last round's rows
    ds.upload(0, base[order])
    import torch
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for what, f in (("encode", lambda: ds.encode_jpeg(0, a.N, 75)), ("roundtrip", lambda: ds.jpeg_roundtrip(0, a.N, 75))):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            for k in KERNELS:
                if k in ev.key:
                    kern.setdefault(what, {})[k] = kern.get(what, {}).get(k, 0.0) + ev.device_time_total / 1000.0
    try:
        from PIL import Image
        n = min(a.pillow, a.N)
        rows = [np.ascontiguousarray(base[order[i]].transpose(1, 2, 0)) for i in range(n)]
        out = []
        t0 = time.perf_counter()
        for r in rows:
            buf = io.BytesIO()
            Image.fromarray(r).save(buf, "JPEG", quality=75)
            out.append(buf.getvalue())
        pil = n / (time.perf_counter() - t0)
        exact = out == files[:n]
    except ImportError:
        pil, exact = float("nan"), None
    name, power, clock = card()
    be, br = min(t_enc), min(t_rt)
    print(json.dumps({
        "rows": a.N, "size": "3x64x64 q75 4:2:0", "file_MB": round(total / 1e6, 1),
        "encode_s": round(be, 4), "encode_rounds_s": [round(t, 4) for t in t_enc], "encode_images_per_s": round(a.N / be),
        "roundtrip_s": round(br, 4), "roundtrip_rounds_s": [round(t, 4) for t in t_rt],
        "roundtrip_images_per_s": round(a.N / br),
        "kernel_ms": {w: {k: round(v, 2) for k, v in d.items()} for w, d in kern.items()},
        "pillow_images_per_s_1thread": round(pil) if pil == pil else None,
        "encode_speedup_vs_pillow": round(a.N / be / pil, 1) if pil == pil else None,
        "bytes_equal_to_pillow": exact, "card": name, "power_limit": power, "max_sm_clock": clock}))
    ds.close()
    ctx.close()


if __name__ == "__main__":
    main()
