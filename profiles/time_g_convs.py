"""times G's tensor-core conv launches (CUDA events via fg_timing); IMPL selects conv_impl.
With option bwd_merge (default 1) G.C2's weight and data gradient are one launch, timed as G.C2.wgrad+dgrad."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg
from face_generator_b200 import layouts as LY
from face_generator_b200.lib import NET_G
B, C = 256, 3
rng = np.random.default_rng(1)
ctx = fg.Context(0, max_batch=B, channels=C)
ctx.set_option("conv_impl", int(os.environ.get("IMPL", "2")))
ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
noise = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
dimg = rng.standard_normal((B, C, 32, 32)).astype(np.float32)
for it in range(6):
    if it == 2:
        ctx.timing_enable(True)
    ctx.G_forward(noise, want_images=False)
    ctx.zero_grads(NET_G)
    ctx.G_backward(dimg)
out = {}
for k in ("G.C1.fwd", "G.C2.fwd", "G.C2.wgrad+dgrad", "G.C2.dgrad", "G.C1.wgrad+dgrad", "G.C1.dgrad", "G.C2.wgrad",
          "G.C1.wgrad"):
    ms, n = ctx.timing_get(k)
    if k.endswith(".wgrad"):  # fg_timing_get matches by prefix: leave out the merged launch
        m2, n2 = ctx.timing_get(k + "+dgrad")
        ms, n = ms - m2, n - n2
    out[k] = round(ms / max(n, 1), 4)
print("IMPL", os.environ.get("IMPL", "2"), out)
