"""One small pass over every device entry point, meant to run under
   compute-sanitizer --tool memcheck python profiles/sanitize_smoke.py
(out-of-bounds / misaligned accesses in the hand-written kernels; TMA zero-fill reads are in-bounds by construction)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import face_generator_b200 as fg  # noqa: E402
from face_generator_b200 import layouts as LY, scoring as S  # noqa: E402
from face_generator_b200.dataset import DeviceDataset, noise_uniform  # noqa: E402
from face_generator_b200.lib import NET_D, NET_G  # noqa: E402

rng = np.random.default_rng(0)
for C, B, impl in ((3, 12, 2), (1, 6, 0)):  # ragged batches on purpose (not multiples of the 128-row tiles)
    ctx = fg.Context(0, max_batch=16, channels=C)
    ctx.set_option("conv_impl", impl)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    hyper = fg.hyper_default()
    real = rng.random((B // 2, C, 32, 32)).astype(np.float32)
    nD, nG = noise_uniform(ctx, 1, (B // 2, 100)), noise_uniform(ctx, 2, (B, 100))
    for opt in ("adam", "adagrad", "sgd"):
        ctx.set_optimizer(NET_D, opt, 0.5)
        ctx.set_optimizer(NET_G, opt, 0.5)
        st = ctx.train_step(hyper, B, real, nD, nG, None, None, 3)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    imgs = ctx.sample(noise_uniform(ctx, 4, (10, 100)), chunk=4)
    S.d_score(ctx, imgs, 4, training=True, seed=5)
    ds = DeviceDataset(ctx, rng.integers(0, 256, (33, 3, 50, 45), dtype=np.uint8))
    ds.gather(ds.draw(6, 7))
    ds.train_step(hyper, B, 7)
    for size in (16, 20, 1):
        ds.gather(ds.draw(8, 5), size)
    for cs in (16, 12, 1, 32):
        ds.gather_c2f(ds.draw(9, 5), cs)
    S.find_closest_neighbours(ds, imgs[:3])
    S.nearest(ctx, rng.random((3, 100)).astype(np.float32), rng.random((20, 100)).astype(np.float32))
    x = rng.standard_normal((3, 5, 8, 8)).astype(np.float32)
    ctx.upsample2_backward(ctx.upsample2_forward(x))
    ctx.avgpool2_backward(ctx.avgpool2_forward(x))
    ctx.maxpool2_backward(x, ctx.maxpool2_forward(x))
    ctx.dropout_forward(x, (rng.random(x.shape) < 0.5).astype(np.float32), 0.5)
    ctx.sigmoid_backward(ctx.sigmoid_forward(x), x)
    net = fg.C2f(ctx)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C), rng, 1.0))
    diff, cr = LY.c2f_pairs(B // 2, C, rng)
    _, cf = LY.c2f_pairs(B // 2, C, rng)
    _, cg = LY.c2f_pairs(B, C, rng)
    st = net.train_step(fg.hyper_default(D_L1=1e-7, D_L2=0.0), B, diff, np.concatenate([cr, cf]),
                        rng.uniform(-1, 1, (B // 2, 1, 32, 32)).astype(np.float32), cg,
                        rng.uniform(-1, 1, (B, 1, 32, 32)).astype(np.float32), None, None, 9)
    assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    for i, cs in enumerate((16, 8, 16)):  # device-fed: eager, captured, replayed
        st = net.train_step_dataset(ds, fg.hyper_default(D_L1=1e-7, D_L2=0.0), B, cs, 40 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    S.approx_parzen(net, diff[:2] + cr[:2], cr[:2], 5, rng)
    net.close()
    # the --scale 16 nets, three identical calls: eager, captured, replayed
    s16 = fg.S16(ctx)
    s16.set_params(NET_G, (rng.standard_normal(s16.count(NET_G)) * 0.02).astype(np.float32))
    s16.set_params(NET_D, (rng.standard_normal(s16.count(NET_D)) * 0.02).astype(np.float32))
    r16 = rng.random((B // 2, C, 16, 16)).astype(np.float32)
    zD, zG = rng.uniform(-1, 1, (B // 2, 100)).astype(np.float32), rng.uniform(-1, 1, (B, 100)).astype(np.float32)
    for i in range(3):
        st = s16.train_step(fg.hyper_default(), B, r16, zD, zG, None, None, 20 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
        st = s16.train_step_dataset(ds, fg.hyper_default(), B, 50 + i)
        assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    s16.close()
    # the 32x32 step through eager / capture / replay, on both operand splits
    for f16 in (1, 0):
        ctx.set_option("mma_f16", f16)
        for i in range(3):
            st = ctx.train_step(hyper, B, real, nD, nG, None, None, 30 + i)
            assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    # SpatialConvolutionUpsample with factor 2 (L-op), both directions
    from face_generator_b200.lib import _ptr
    xs = rng.standard_normal((2, 64, 8, 8)).astype(np.float32)
    ws = (rng.standard_normal((64, 64, 3, 3)) * 0.05).astype(np.float32)
    bs, ys = np.zeros(64, np.float32), np.empty((2, 16, 16, 16), np.float32)
    assert ctx.lib.fg_scu_forward(ctx.h, _ptr(xs), _ptr(ws), _ptr(bs), _ptr(ys), 2, 64, 8, 8, 16, 3, 2) == 0
    dxs, dws = np.empty_like(xs), np.zeros_like(ws)
    assert ctx.lib.fg_scu_backward_data(ctx.h, _ptr(ys), _ptr(ws), _ptr(dxs), 2, 64, 8, 8, 16, 3, 2) == 0
    assert ctx.lib.fg_scu_backward_filter(ctx.h, _ptr(xs), _ptr(ys), _ptr(dws), None, 2, 64, 8, 8, 16, 3, 2) == 0
    if C == 1:  # the autoencoder of train_autoencoder.lua is grayscale: three steps (eager, captured, replayed), host- and
        # device-fed with a ragged last batch, both forwards, the backward and the layer ops
        from face_generator_b200 import autoencoder as A
        ae = A.Autoencoder(ctx, 16, 64)
        ae.set_params(A.init_params(16, 64, rng) * 10)
        im = rng.random((B, 1, 16, 16)).astype(np.float32)
        for i in range(3):
            assert np.isfinite(ae.train_step(A.ae_hyper_default(L2=1e-4), im, seed=60 + i)["loss"])
            assert np.isfinite(ae.train_step_dataset(ds, A.ae_hyper_default(), np.arange(B - i, dtype=np.int32), seed=i)["loss"])
        ae.zero_grads()
        ae.backward(ae.forward(im, training=True, seed=3)[1])
        ae.reconstruct(im, chunk=4, training=True, seed=1)
        ae.encode(im, chunk=5)
        ae.close()
        from face_generator_b200.lib import _ptr
        v, o = rng.standard_normal(1000).astype(np.float32), np.empty(1000, np.float32)
        for fn in (ctx.lib.fg_relu_forward, ctx.lib.fg_tanh_forward):
            assert fn(ctx.h, _ptr(v), _ptr(o), v.size) == 0
        for fn in (ctx.lib.fg_relu_backward, ctx.lib.fg_tanh_backward):
            assert fn(ctx.h, _ptr(v), _ptr(v), _ptr(o), v.size) == 0
        assert ctx.lib.fg_abs_forward(ctx.h, _ptr(v), _ptr(o), v.size, _ptr(o[:1].copy())) == 0
        assert ctx.lib.fg_abs_backward(ctx.h, _ptr(v), _ptr(v), v.size, _ptr(o)) == 0
    ds.close()
    ctx.close()
    print("ok", C, B, impl, flush=True)
print("sanitize smoke done")
