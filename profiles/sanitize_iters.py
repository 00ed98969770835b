"""One (2, 2) call of every multi-iteration entry point (host- and device-fed, eager, captured and replayed), meant to
run under
   compute-sanitizer --tool memcheck python profiles/sanitize_iters.py
(the per-iteration offsets into the stacked inputs and staging buffers, and the draws inside the captured step)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import layouts as LY  # noqa: E402
from face_generator_b200.dataset import DeviceDataset  # noqa: E402
from face_generator_b200.lib import NET_D, NET_G  # noqa: E402

rng = np.random.default_rng(0)
f = lambda a: np.ascontiguousarray(a, np.float32)
d, g = 2, 2
for C, B in ((3, 12), (1, 6)):  # ragged batches on purpose, below max_batch
    ctx = fg.Context(0, max_batch=16, channels=C)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    ds = DeviceDataset(ctx, rng.integers(0, 256, (33, 3, 50, 45), dtype=np.uint8))
    hyper = fg.hyper_default()
    Bh = B // 2
    masks = lambda n: f(rng.random((n, B, 1984)) < 0.5)
    for i in range(3):  # eager, captured, replayed
        st = ctx.train_step_iters(hyper, B, d, g, f(rng.random((d, Bh, C, 32, 32))), f(rng.uniform(-1, 1, (d, Bh, 100))),
                                  f(rng.uniform(-1, 1, (g, B, 100))), masks(d) if i == 0 else None, masks(g) if i == 0 else None,
                                  10 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
        st = ds.train_step_iters(hyper, B, d, g, 20 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    s16 = fg.S16(ctx)
    s16.set_params(NET_G, (rng.standard_normal(s16.count(NET_G)) * 0.02).astype(np.float32))
    s16.set_params(NET_D, (rng.standard_normal(s16.count(NET_D)) * 0.02).astype(np.float32))
    for i in range(3):
        st = s16.train_step_iters(hyper, B, d, g, f(rng.random((d, Bh, C, 16, 16))), f(rng.uniform(-1, 1, (d, Bh, 100))),
                                  f(rng.uniform(-1, 1, (g, B, 100))), None, None, 30 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
        st = s16.train_step_dataset_iters(ds, hyper, B, d, g, 40 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    s16.close()
    for S in (16, 64):
        net = fg.C2f(ctx, S)
        net.set_params(NET_G, (rng.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32))
        net.set_params(NET_D, (rng.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32))
        for i in range(3):
            st = net.train_step_iters(hyper, B, d, g, f(rng.uniform(-0.3, 0.3, (d, Bh, C, S, S))), f(rng.random((d, B, C, S, S))),
                                      f(rng.uniform(-1, 1, (d, Bh, 1, S, S))), f(rng.random((g, B, C, S, S))),
                                      f(rng.uniform(-1, 1, (g, B, 1, S, S))), None, None, 50 + i)
            assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
            st = net.train_step_dataset_iters(ds, hyper, B, d, g, S // 2, 60 + i)
            assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
        net.close()
    ds.close()
    ctx.close()
    print("ok", C, B, flush=True)
print("sanitize iterations done")
