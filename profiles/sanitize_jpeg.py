"""One small pass over the JPEG entry points (fg_jpeg_info, fg_dataset_upload_jpeg, fg_dataset_download), meant to
run under
   compute-sanitizer --tool memcheck python profiles/sanitize_jpeg.py
(out-of-bounds reads of the entropy bytes near interval ends, the band planes of the banded IDCT path, and the
refusal paths).  Expected: 0 errors."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import face_generator_b200 as fg  # noqa: E402
import jpeg_utils as JU  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from face_generator_b200.lib import FGError  # noqa: E402

corpus = JU.load()
ctx = fg.Context(0, max_batch=16, channels=3)
gray = fg.Context(0, max_batch=16, channels=1)
for e in corpus:
    H, W = e.cache_hw
    for Cs in ((3, 1) if e.C == 1 else (3,)):
        ds = DeviceDataset(ctx if Cs == 3 else gray, shape=(2, Cs, H, W))
        try:
            ds.upload_jpeg(1, [e.bytes])
            assert e.mismatch(ds.download(1, 1)[0]) is None, e.name
        except FGError:
            assert not e.supported, e.name
        ds.close()
faces = [e for e in corpus if e.face]
ds = DeviceDataset(ctx, shape=(40, 3, 64, 64))
ds.upload_jpeg(3, [faces[i % len(faces)].bytes for i in range(37)])
ds.close()
gray.close()
ctx.close()
print("sanitize_jpeg: done")
