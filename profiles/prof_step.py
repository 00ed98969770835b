"""ncu driver: a few fg_train_step iterations at batch 256 (colour), everything resident on the device.
   launch list :  ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file /tmp/launches.csv python profiles/prof_step.py 2
   one kernel  :  ncu --set full --clock-control none --import-source on -k regex:<name> -s <skip> -c <n> -o /tmp/prof_x python profiles/prof_step.py 2
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg
from face_generator_b200 import layouts as LY
from face_generator_b200.lib import NET_D, NET_G

B, C = 256, 3
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
rng = np.random.default_rng(1)
ctx = fg.Context(0, max_batch=B, channels=C)
for k, v in (a.split("=") for a in sys.argv[2:]):
    ctx.set_option(k, int(v))
ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
f = lambda a: np.ascontiguousarray(a, np.float32)
dev = [ctx.dev_array(f(a)) for a in (rng.random((B // 2, C, 32, 32)), rng.uniform(-1, 1, (B // 2, 100)), rng.uniform(-1, 1, (B, 100)))]
hyper = fg.hyper_default()
for i in range(steps):
    ctx.train_step(hyper, B, dev[0], dev[1], dev[2], None, None, i + 1, want_stats=False)
ctx.sync()
print("done", ctx.launches())
