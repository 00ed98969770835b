"""One small pass over the augmentation entry points (fg_lfw_aug_params, fg_dataset_augment, DeviceDataset.from_lfw),
meant to run under
   compute-sanitizer --tool memcheck python profiles/sanitize_augment.py
(bilinear taps at the image edges and off it, flipped columns, the shared-memory passes at destination sizes 1x1 to
84x84, grayscale caches, and the refusal paths).  Expected: 0 errors."""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import face_generator_b200 as fg  # noqa: E402
import aug_ref as R  # noqa: E402
from face_generator_b200.dataset import DeviceDataset, lfw_aug_params  # noqa: E402
from face_generator_b200.lib import FGError  # noqa: E402
from test_gpu_augment import hand_made  # noqa: E402

rng = np.random.default_rng(1)
ctx = fg.Context(0, max_batch=16, channels=3)
gray = fg.Context(0, max_batch=16, channels=1)
srcs = rng.integers(0, 256, (3, 3, 176, 167), dtype=np.uint8)  # the smallest source the crop fits in
augs = np.concatenate([hand_made(3), lfw_aug_params(43, 0, 3, 4, 176, 167)])
for c, s in ((ctx, srcs), (gray, np.ascontiguousarray(srcs[:, :1]))):
    src = DeviceDataset(c, s)
    for Ho, Wo in ((1, 1), (84, 84), (64, 64), (32, 48), (84, 1)):
        dst = DeviceDataset(c, shape=(len(augs), s.shape[1], Ho, Wo))
        dst.augment(src, 0, augs)
        assert np.array_equal(dst.download(), R.augment_rows(s, augs, Ho, Wo)), (Ho, Wo)
        bad = augs.copy()
        bad[1]["src"] = 3
        try:
            dst.augment(src, 0, bad)
            raise AssertionError("not refused")
        except FGError:
            pass
        dst.close()
    src.close()
g = np.load(os.path.join(ROOT, "tests", "golden", "lfw_aug.npz"))
with tempfile.TemporaryDirectory() as tmp:
    for k, name in enumerate(g["names"]):
        os.makedirs(os.path.join(tmp, os.path.dirname(str(name))), exist_ok=True)
        with open(os.path.join(tmp, str(name)), "wb") as f:
            f.write(g["jpegs"][g["offsets"][k]:g["offsets"][k + 1]].tobytes())
    DeviceDataset.from_lfw(ctx, [tmp], augmentations=2, chunk=3).close()
gray.close()
ctx.close()
print("sanitize_augment: done")
