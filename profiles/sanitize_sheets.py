"""One small pass over fg_image_grid, fg_jpeg_encode (both entropy coders), fg_dataset_nearest_sized and
fg_s16_D_score, meant to run under
   compute-sanitizer --tool memcheck python profiles/sanitize_sheets.py
(the grid's ragged last row, padding and device order; the multi-CTA coder's tile and segment edges at sizes that are
not multiples of the MCU, and its stuffed output's end; the nearest kernel at sizes 16 and 64).  Expected: 0 errors."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import face_generator_b200 as fg  # noqa: E402
import grid_ref as G  # noqa: E402
import jpeg_enc_ref as R  # noqa: E402
from face_generator_b200 import sheets  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from face_generator_b200.lib import S16  # noqa: E402

ctx = fg.Context(0, max_batch=16, channels=3)
rng = np.random.default_rng(1)
imgs = rng.uniform(-1, 1, (37, 3, 16, 16)).astype(np.float32)
for nrow, pad in ((8, 0), (5, 2), (40, 0)):
    assert (sheets.image_grid(ctx, imgs, nrow, pad) == G.grid(imgs, nrow, pad)).all()
for route in (1, 2):
    ctx.set_option("jpeg_route", route)
    for (Cs, H, W) in ((3, 1, 1), (3, 33, 97), (1, 129, 7), (3, 300, 260)):
        img = R.content("noise", H + W, Cs, H, W)
        assert sheets.encode_jpeg(ctx, img, 100)[0] == R.encode(img, 100), (route, Cs, H, W)
ctx.set_option("jpeg_route", 0)
rows = np.stack([R.content("noise", k, 3, 64, 64) for k in range(20)])
ds = DeviceDataset(ctx, rows)
for size in (16, 64):
    q = rng.random((5, 3, size, size)).astype(np.float32)
    idx, dist = np.empty(5, np.int32), np.empty(5, np.float32)
    assert ctx.lib.fg_dataset_nearest_sized(ds.h, size, q.ctypes.data, 5, idx.ctypes.data, dist.ctypes.data) == 0
ds.close()
net = S16(ctx)
preds = np.empty(20, np.float32)
x = rng.random((20, 3, 16, 16)).astype(np.float32)
assert ctx.lib.fg_s16_D_score(net.h, x.ctypes.data, 20, 16, 1, 3, preds.ctypes.data) == 0
net.close()
ctx.close()
print("sanitize_sheets: done")
