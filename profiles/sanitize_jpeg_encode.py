"""One small pass over fg_dataset_encode_jpeg and fg_dataset_jpeg_roundtrip, meant to run under
   compute-sanitizer --tool memcheck python profiles/sanitize_jpeg_encode.py
(the edge clamps of the forward kernel at sizes that are not multiples of the MCU, its dummy blocks, the banded path of
rows wider than the shared-memory budget, the word buffers' first and last words, the stuffed output's end, and the
refusal paths).  Expected: 0 errors."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import face_generator_b200 as fg  # noqa: E402
import jpeg_enc_ref as R  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from face_generator_b200.lib import FGError  # noqa: E402

ctx = fg.Context(0, max_batch=16, channels=3)
gray = fg.Context(0, max_batch=16, channels=1)
for (H, W) in ((1, 1), (2, 3), (15, 17), (18, 34), (64, 64), (17, 2048)):
    for Cs, c in ((3, ctx), (1, gray)):
        rows = np.stack([R.content(k, H + W, Cs, H, W) for k in ("noise", "checker", "flat255")])
        ds = DeviceDataset(c, rows)
        for q in (1, 75, 100):
            assert ds.encode_jpeg(1, 2, q) == [R.encode(rows[k], q) for k in (1, 2)], (Cs, H, W, q)
        ds.jpeg_roundtrip(0, 3, 75)
        for bad in ((0, 4, 75), (0, 3, 0)):
            try:
                ds.jpeg_roundtrip(*bad)
                raise AssertionError("accepted %s" % (bad,))
            except FGError:
                pass
        ds.close()
gray.close()
ctx.close()
print("sanitize_jpeg_encode: done")
