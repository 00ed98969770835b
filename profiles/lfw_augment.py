"""Throughput of DeviceDataset.from_lfw (generate_dataset.py's augmented LFW set built on the GPU).

A seeded synthetic LFW-sized tree is written to a temporary directory: 13 233 photos of 250x250 (the JPEG photos of
tests/golden/lfw_aug.npz, drawn with a fixed seed) in LFW's Person_Name/Person_Name_000k.jpg layout.  After a
warm-up call on the first 512 photos, one JSON line reports:
  - from_lfw end to end on the whole tree (file reads, GPU decode, augmentation; 20 rows per photo), best of --rounds,
    as rows/s and photos/s;
  - fg_dataset_augment alone on one chunk of decoded photos (host clock around the call, which returns once the rows
    are written), as rows/s;
  - the device time of aug_crop_kernel and aug_minmax_kernel summed over one whole from_lfw call, from torch.profiler
    in a separate call;
  - tests/aug_ref.py building the 20 rows of one photo on one host thread (the CPU bar);
  - the card's name and power limit, read in the same run.

usage:  python profiles/lfw_augment.py [--photos 13233] [--rounds 2] [--ref-photos 3]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import face_generator_b200 as fg  # noqa: E402
import aug_ref as R  # noqa: E402
from face_generator_b200.dataset import DeviceDataset, lfw_aug_params  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:
        return ["unknown (%s)" % e, "unknown", "unknown"]


def write_tree(root, blobs, n, rng):
    pick = rng.integers(0, len(blobs), n)
    person, k = 0, 0
    for i in range(n):
        if k == 0 or rng.random() < 0.43:  # LFW: 13 233 photos of 5 749 people
            person, k = person + 1, 0
            os.makedirs(os.path.join(root, "Person_%05d" % person))
        k += 1
        with open(os.path.join(root, "Person_%05d" % person, "Person_%05d_%04d.jpg" % (person, k)), "wb") as f:
            f.write(blobs[pick[i]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--photos", type=int, default=13233)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--ref-photos", type=int, default=3)
    a = ap.parse_args()
    g = np.load(os.path.join(ROOT, "tests", "golden", "lfw_aug.npz"))
    blobs = [g["jpegs"][g["offsets"][k]:g["offsets"][k + 1]].tobytes() for k in range(len(g["names"]))]
    tmp = tempfile.mkdtemp(prefix="lfw_augment_")
    try:
        full, warm = os.path.join(tmp, "lfw"), os.path.join(tmp, "warm")
        os.makedirs(full)
        os.makedirs(warm)
        write_tree(full, blobs, a.photos, np.random.default_rng(13233))
        write_tree(warm, blobs, 512, np.random.default_rng(512))
        ctx = fg.Context(0, max_batch=16, channels=3)
        DeviceDataset.from_lfw(ctx, [warm]).close()
        times = []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            ds = DeviceDataset.from_lfw(ctx, [full])
            times.append(time.perf_counter() - t0)
            rows = ds.N
            ds.close()
        best = min(times)
        # fg_dataset_augment alone: one chunk of 2048 decoded photos -> 40 960 rows
        n = 2048
        src = DeviceDataset(ctx, shape=(n, 3, 250, 250))
        src.upload_jpeg(0, [blobs[i % len(blobs)] for i in range(n)])
        dst = DeviceDataset(ctx, shape=(n * 20, 3, 64, 64))
        augs = lfw_aug_params(43, 0, n, 19, 250, 250)
        dst.augment(src, 0, augs)
        aug_t = []
        for _ in range(3):
            t0 = time.perf_counter()
            dst.augment(src, 0, augs)
            aug_t.append(time.perf_counter() - t0)
        photos = src.download(0, len(blobs))
        exact = np.array_equal(dst.download(0, 40), R.augment_rows(photos, augs[:40]))
        src.close()
        dst.close()
        # per kernel, in a separate profiled call
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            DeviceDataset.from_lfw(ctx, [full]).close()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            for k in ("aug_crop_kernel", "aug_minmax_kernel", "jpeg_entropy_kernel", "jpeg_idct_color_kernel"):
                if k in ev.key:
                    kern[k] = kern.get(k, 0.0) + ev.device_time_total / 1000.0  # ms
        ctx.close()
        # the numpy reference, one thread, all 20 rows of a photo
        refa = lfw_aug_params(43, 0, a.ref_photos, 19, 250, 250)
        refa["src"] %= len(photos)
        t0 = time.perf_counter()
        R.augment_rows(photos, refa)
        ref_s = (time.perf_counter() - t0) / a.ref_photos
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    name, power, clock = card()
    print(json.dumps({
        "photos": a.photos, "rows": rows, "from_lfw_s": round(best, 3), "from_lfw_s_all": [round(t, 3) for t in times],
        "from_lfw_rows_per_s": round(rows / best), "from_lfw_photos_per_s": round(a.photos / best),
        "augment_call_s": round(min(aug_t), 4), "augment_rows_per_s": round(n * 20 / min(aug_t)),
        "kernel_ms_one_from_lfw": {k: round(v, 2) for k, v in kern.items()},
        "aug_crop_rows_per_s": round(rows / (kern["aug_crop_kernel"] / 1000.0)) if "aug_crop_kernel" in kern else None,
        "aug_ref_s_per_photo_1thread": round(ref_s, 3), "speedup_vs_aug_ref": round(a.photos / best * ref_s, 1),
        "bitwise_equal_to_aug_ref": bool(exact), "card": name, "power_limit": power, "max_sm_clock": clock}))


if __name__ == "__main__":
    main()
