"""ncu driver: 3 iterations of G forward+backward at B=256 (colour) so that
   tapconv launches per iteration = [G.C1 fwd, G.C2 fwd, G.C2 dgrad, G.C1 dgrad], wgrad = [G.C2 wgrad, G.C1 wgrad].
Usage:
   ncu --set full --clock-control none --import-source on -k regex:tapconv_tc -s 8 -c 4 -o /tmp/prof_tapconv python profiles/prof_g_convs.py
   ncu --set full --clock-control none --import-source on -k regex:wgrad_tc  -s 4 -c 2 -o /tmp/prof_wgrad  python profiles/prof_g_convs.py
"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg
from face_generator_b200 import layouts as LY
from face_generator_b200.lib import NET_G
B, C = 256, 3
impl = int(sys.argv[1]) if len(sys.argv) > 1 else 2
rng = np.random.default_rng(1)
ctx = fg.Context(0, max_batch=B, channels=C)
ctx.set_option("conv_impl", impl)
ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
noise = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
dimg = rng.standard_normal((B, C, 32, 32)).astype(np.float32)
for _ in range(3):
    ctx.G_forward(noise, want_images=False)
    ctx.zero_grads(NET_G)
    ctx.G_backward(dimg)
ctx.sync()
print("done", ctx.launches())
