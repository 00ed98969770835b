"""The device-resident dataset feeding the coarse-to-fine trainer (train_c2f.lua) and train.lua --scale 16.

CPU: the float64 restatement of dataset_c2f.lua:49-62 _toResult (c2f_pairs below, on oracle_data's image.scale) has
the properties its definition implies, and matches PyTorch where PyTorch has the same scaling rules.
GPU: fg_dataset_gather_sized / fg_dataset_gather_c2f against that restatement; the device-fed s16 / c2f steps are
bitwise the host-fed steps on the same (drawn, gathered) inputs; adversarial.train routes an S16 to the 16x16 nets."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import oracle_data as OD  # noqa: E402


def c2f_pairs(images_u8, indices, nb_channels, coarse_size):
    """dataset_c2f.lua:49-62 _toResult at fineSize 32 in float64: fine = image.scale(image.load(...), 32, 32),
    coarse = image.scale(image.scale(fine, cs, cs), 32, 32), diff = fine - coarse."""
    fine = OD.gather(images_u8, indices, nb_channels, 32)
    coarse = OD.scale(OD.scale(fine, coarse_size, coarse_size), 32, 32)
    return fine, coarse, fine - coarse


def test_c2f_pairs_identity_at_full_coarse_size():
    rng = np.random.default_rng(11)
    imgs = rng.integers(0, 256, (5, 3, 64, 64), dtype=np.uint8)
    fine, coarse, diff = c2f_pairs(imgs, [0, 3, 4], 3, 32)
    np.testing.assert_array_equal(coarse, fine)
    assert not diff.any()


def test_c2f_pairs_constant_image_has_no_detail():
    """image.scale computes its linear-interpolation weights (1 - f, f) in float32, so when 1 - f rounds, an
    enlarging row sums to 1 only within 2^-24 per weight: exact for cs = 1, 24, 32, within 1e-7 for 8, 12, 16."""
    imgs = np.full((2, 3, 50, 45), 173, np.uint8)
    for cs, bar in ((1, 1e-12), (24, 1e-12), (32, 1e-12), (8, 1e-7), (12, 1e-7), (16, 1e-7)):
        fine, coarse, diff = c2f_pairs(imgs, [0, 1], 3, cs)
        assert np.abs(diff).max() < bar
        np.testing.assert_allclose(fine, 173 / 255.0, atol=1e-12)


def test_c2f_pairs_diff_is_fine_minus_coarse():
    rng = np.random.default_rng(12)
    imgs = rng.integers(0, 256, (4, 3, 64, 64), dtype=np.uint8)
    for C in (3, 1):
        fine, coarse, diff = c2f_pairs(imgs, [3, 1, 1], C, 12)
        assert fine.shape == coarse.shape == diff.shape == (3, C, 32, 32)
        np.testing.assert_array_equal(fine - coarse, diff)


def test_c2f_pairs_vs_torch_interpolate():
    """coarse 16 from 32: an integer shrink factor ('area') and an enlargement (bilinear, align_corners), the cases
    where torch's rules coincide with image.scale (see test_scale_restatement_vs_torch_interpolate)."""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(13)
    imgs = rng.integers(0, 256, (3, 3, 64, 64), dtype=np.uint8)
    fine, coarse, diff = c2f_pairs(imgs, [0, 1, 2], 3, 16)
    t = F.interpolate(torch.tensor(fine), size=(16, 16), mode="area")
    ref = F.interpolate(t, size=(32, 32), mode="bilinear", align_corners=True).numpy()
    np.testing.assert_allclose(coarse, ref, rtol=0, atol=1e-6)
    np.testing.assert_allclose(diff, fine - ref, rtol=0, atol=1e-6)


# ---- GPU --------------------------------------------------------------------------------------------------------

SOURCES = [(3, 3, 64, 64), (3, 1, 64, 64), (1, 1, 64, 64), (3, 3, 50, 45), (3, 1, 50, 45), (1, 1, 50, 45)]


def _gather32(ds, idx):
    """fg_dataset_gather itself (DeviceDataset.gather goes through fg_dataset_gather_sized)."""
    import face_generator_b200 as fg
    idx = np.ascontiguousarray(idx, np.int32)
    out = np.empty((idx.size, ds.ctx.C, 32, 32), np.float32)
    rc = ds.lib.fg_dataset_gather(ds.h, idx.ctypes.data_as(ctypes.c_void_p), idx.size, out.ctypes.data_as(ctypes.c_void_p))
    if rc != 0:
        raise fg.FGError("fg_dataset_gather")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("Cs,C,Hs,Ws", SOURCES)
def test_gpu_gather_sized_matches_image_scale(Cs, C, Hs, Ws):
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset
    rng = np.random.default_rng(Hs * 100 + Ws + 10 * Cs + C)
    N, B = 29, 16
    imgs = rng.integers(0, 256, (N, Cs, Hs, Ws), dtype=np.uint8)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ds = DeviceDataset(ctx, imgs)
    idx = rng.integers(0, N, B)
    for size in (16, 8, 20, 32):
        got = ds.gather(idx, size)
        assert got.shape == (B, C, size, size)
        assert np.abs(got - OD.gather(imgs, idx, C, size)).max() < 2e-6
    np.testing.assert_array_equal(ds.gather(idx, 32), _gather32(ds, idx))
    np.testing.assert_array_equal(ds.gather(idx), _gather32(ds, idx))
    for bad in (0, 33):
        with pytest.raises(fg.FGError):
            ds.gather(idx, bad)
    with pytest.raises(fg.FGError):
        ds.gather([N], 16)
    ds.close()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("Cs,C,Hs,Ws", SOURCES)
def test_gpu_gather_c2f_matches_restatement(Cs, C, Hs, Ws):
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import _ptr
    rng = np.random.default_rng(Hs * 1000 + Ws + 10 * Cs + C)
    N, B = 31, 12
    imgs = rng.integers(0, 256, (N, Cs, Hs, Ws), dtype=np.uint8)
    ctx = fg.Context(0, max_batch=B, channels=C)
    ds = DeviceDataset(ctx, imgs)
    idx = rng.integers(0, N, B)
    fine32 = _gather32(ds, idx)
    for cs in (16, 8, 12, 24, 1, 32):
        fine, coarse, diff = ds.gather_c2f(idx, cs)
        rf, rc, rd = c2f_pairs(imgs, idx, C, cs)
        assert np.abs(fine - rf).max() < 2e-6
        assert np.abs(coarse - rc).max() < 2e-6
        assert np.abs(diff - rd).max() < 4e-6
        np.testing.assert_array_equal(fine, fine32)  # the same per-pixel code as fg_dataset_gather
        np.testing.assert_array_equal(diff, fine - coarse)
        if cs == 32:
            np.testing.assert_array_equal(coarse, fine)
            assert not diff.any()
        # any output may be NULL; the others are unchanged
        i32 = np.ascontiguousarray(idx, np.int32).ctypes.data_as(ctypes.c_void_p)
        only_coarse = np.empty_like(coarse)
        assert ds.lib.fg_dataset_gather_c2f(ds.h, i32, B, cs, None, _ptr(only_coarse), None) == 0
        np.testing.assert_array_equal(only_coarse, coarse)
        only_diff = np.empty_like(diff)
        assert ds.lib.fg_dataset_gather_c2f(ds.h, i32, B, cs, None, None, _ptr(only_diff)) == 0
        np.testing.assert_array_equal(only_diff, diff)
        assert ds.lib.fg_dataset_gather_c2f(ds.h, i32, B, cs, None, None, None) == 0
    for bad in (0, 33):
        with pytest.raises(fg.FGError):
            ds.gather_c2f(idx, bad)
    with pytest.raises(fg.FGError):
        ds.gather_c2f([0, N], 16)
    with pytest.raises(fg.FGError):
        ds.gather_c2f([-1], 16)
    ds.close()
    ctx.close()


def _s16_init(net, rng):
    from face_generator_b200.lib import NET_D, NET_G
    net.set_params(NET_G, (rng.standard_normal(net.count(NET_G)) * 0.02).astype(np.float32))
    net.set_params(NET_D, (rng.standard_normal(net.count(NET_D)) * 0.02).astype(np.float32))


def _state(net):
    from face_generator_b200.lib import NET_D, NET_G
    out = []
    for k in (NET_G, NET_D):
        m, v, t = net.get_adam_state(k)
        out += [net.get_params(k), net.get_grads(k), m, v, np.array([t])]
    return out


def _assert_same(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 1])
def test_gpu_s16_device_fed_step_equals_host_fed_step(C):
    """fg_s16_train_step_dataset == fg_s16_train_step on (gather(draw(4s), 16), uniform(4s+1), uniform(4s+2)), bitwise."""
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset, noise_uniform
    B = 64
    imgs = np.random.default_rng(40 + C).integers(0, 256, (300, 3, 64, 64), dtype=np.uint8)
    hyper = fg.hyper_default()
    res = []
    for mode in ("device", "host"):
        ctx = fg.Context(0, max_batch=B, channels=C)
        net = fg.S16(ctx)
        _s16_init(net, np.random.default_rng(41))
        ds = DeviceDataset(ctx, imgs)
        stats = []
        for seed in (5, 6, 7):  # eager, captured, replayed
            if mode == "device":
                st = net.train_step_dataset(ds, hyper, B, seed)
            else:
                real = ds.gather(ds.draw(4 * seed, B // 2), 16)
                nD = noise_uniform(ctx, 4 * seed + 1, (B // 2, 100))
                nG = noise_uniform(ctx, 4 * seed + 2, (B, 100))
                st = net.train_step(hyper, B, real, nD, nG, None, None, seed)
            stats.append(st)
        res.append((stats, _state(net) + [net.get_bn_state()]))
        ds.close()
        net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])


def _c2f_host_inputs(ctx, ds, B, cs, seed):
    from face_generator_b200.dataset import noise_uniform
    Bh = B // 2
    _, cr, dr = ds.gather_c2f(ds.draw(8 * seed, Bh), cs)
    _, cf, _ = ds.gather_c2f(ds.draw(8 * seed + 1, Bh), cs)
    _, cg, _ = ds.gather_c2f(ds.draw(8 * seed + 2, B), cs)
    nD = noise_uniform(ctx, 8 * seed + 3, (Bh, 1, 32, 32))
    nG = noise_uniform(ctx, 8 * seed + 4, (B, 1, 32, 32))
    return dr, np.concatenate([cr, cf]), nD, cg, nG


@pytest.mark.gpu
@pytest.mark.parametrize("C,cs", [(3, 16), (3, 8), (1, 16), (1, 8)])
def test_gpu_c2f_device_fed_step_equals_host_fed_step(C, cs):
    """Three consecutive fg_c2f_train_step_dataset calls at batch 256 (eager, captured, replayed) == fg_c2f_train_step on
    the same drawn pairs and noise, bitwise."""
    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    B = 256
    imgs = np.random.default_rng(50 + C).integers(0, 256, (600, 3, 64, 64), dtype=np.uint8)
    hyper = fg.hyper_default()
    res = []
    for mode in ("device", "host"):
        rng = np.random.default_rng(51)
        ctx = fg.Context(0, max_batch=B, channels=C)
        net = fg.C2f(ctx)
        net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
        net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C), rng, 1.0))
        ds = DeviceDataset(ctx, imgs)
        stats = []
        for seed in (3, 4, 5):
            if mode == "device":
                st = net.train_step_dataset(ds, hyper, B, cs, seed)
            else:
                st = net.train_step(hyper, B, *_c2f_host_inputs(ctx, ds, B, cs, seed), None, None, seed)
            assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
            stats.append(st)
        res.append((stats, _state(net)))
        ds.close()
        net.close()
        ctx.close()
    assert res[0][0] == res[1][0]
    _assert_same(res[0][1], res[1][1])


@pytest.mark.gpu
def test_gpu_device_fed_steps_reject_bad_arguments():
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset
    imgs = np.random.default_rng(60).integers(0, 256, (20, 3, 64, 64), dtype=np.uint8)
    hyper = fg.hyper_default()
    ctx, other = fg.Context(0, max_batch=16, channels=3), fg.Context(0, max_batch=16, channels=3)
    c2f, s16 = fg.C2f(ctx), fg.S16(ctx)
    ds, ds_other = DeviceDataset(ctx, imgs), DeviceDataset(other, imgs)
    for cs in (0, 33):
        with pytest.raises(fg.FGError):
            c2f.train_step_dataset(ds, hyper, 16, cs, 1)
    for B in (2, 15, 18):
        with pytest.raises(fg.FGError):
            c2f.train_step_dataset(ds, hyper, B, 16, 1)
        with pytest.raises(fg.FGError):
            s16.train_step_dataset(ds, hyper, B, 1)
    with pytest.raises(fg.FGError):
        c2f.train_step_dataset(ds_other, hyper, 16, 16, 1)
    with pytest.raises(fg.FGError):
        s16.train_step_dataset(ds_other, hyper, 16, 1)
    st = c2f.train_step_dataset(ds, hyper, 16, 16, 1)
    assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    st = s16.train_step_dataset(ds, hyper, 16, 1)
    assert np.isfinite(st["loss_D"]) and np.isfinite(st["loss_G"])
    for o in (ds, ds_other, c2f, s16):
        o.close()
    ctx.close()
    other.close()


@pytest.mark.gpu
def test_gpu_adversarial_train_routes_s16_to_the_16x16_nets():
    import face_generator_b200 as fg
    from face_generator_b200 import adversarial as A
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    imgs = np.random.default_rng(70).integers(0, 256, (64, 3, 64, 64), dtype=np.uint8)
    ctx = fg.Context(0, max_batch=16, channels=3)
    net = fg.S16(ctx)
    _s16_init(net, np.random.default_rng(71))
    ds = DeviceDataset(ctx, imgs)
    before32 = (ctx.get_params(NET_G), ctx.get_params(NET_D))
    before16 = (net.get_params(NET_G), net.get_params(NET_D))
    acc, conf, trained = A.train(net, ds, fg.hyper_default(), 16, n_epoch=48)
    assert conf.sum() == sum(b for _, b in A.epoch_batches(48, 16)) and 0.0 <= acc <= 1.0
    np.testing.assert_array_equal(ctx.get_params(NET_G), before32[0])
    np.testing.assert_array_equal(ctx.get_params(NET_D), before32[1])
    assert not np.array_equal(net.get_params(NET_G), before16[0])
    assert trained == 0 or not np.array_equal(net.get_params(NET_D), before16[1])
    ds.close()
    net.close()
    ctx.close()


def _gpu_count():
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for l in out.splitlines() if l.startswith("GPU "))
    except Exception:
        return 0


def _worker_c2f_dataset(rank, world, port, q):
    import torch.distributed as dist
    import face_generator_b200 as fg
    from face_generator_b200 import adversarial as A
    from face_generator_b200 import layouts as LY
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 16, 3
    rng = np.random.default_rng(80)  # the same start on both ranks
    ctx = fg.Context(rank, max_batch=B, channels=C)
    net = fg.C2f(ctx)
    net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
    net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C), rng, 1.0))
    ds = DeviceDataset(ctx, np.random.default_rng(81).integers(0, 256, (100, 3, 64, 64), dtype=np.uint8))
    ids = [ctx.dp_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.dp_init(ids[0], world, rank)
    net.dp_broadcast_params()
    seed0 = A.epoch_seed0(1, rank)  # per-rank streams: different pairs and noise on each rank
    for i in range(3):
        net.train_step_dataset(ds, fg.hyper_default(), B, 16, seed0 + i + 1)
    q.put((rank, net.get_params(NET_G), net.get_params(NET_D)))
    dist.barrier()
    ds.close()
    net.close()
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_dp_c2f_device_fed_replicas_stay_identical():
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, 29781
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker_c2f_dataset, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r = q.get(timeout=600)
        got[r[0]] = r
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    np.testing.assert_array_equal(got[0][1], got[1][1])
    np.testing.assert_array_equal(got[0][2], got[1][2])
