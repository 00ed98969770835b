"""Data parallel with the branched discriminators (needs >= 2 GPUs; skipped on one GPU): a two-rank step leaves every
rank with the mean of the per-shard gradients, which is the gradient of the concatenated batch for these mean losses,
and the confusion counts of both shards."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

pytestmark = pytest.mark.gpu


def _gpu_count():
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for l in out.splitlines() if l.startswith("GPU "))
    except Exception:
        return 0


def _worker(rank, world, port, name, q):
    import torch.distributed as dist
    import dbr_ref as R
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 8, 3
    S = R.NETS[name][0]
    ref = R.Net(name, C)
    rng = np.random.default_rng(901 + rank)
    real = rng.uniform(0, 1, (B // 2, C, S, S)).astype(np.float32)
    nD = rng.uniform(-1, 1, (B // 2, 100)).astype(np.float32)
    nG = rng.uniform(-1, 1, (B, 100)).astype(np.float32)
    mD = (rng.uniform(0, 1, (B, ref.mask)) >= 0.5).astype(np.float32)
    mG = (rng.uniform(0, 1, (B, ref.mask)) >= 0.5).astype(np.float32)
    # lr = 0, no penalty, no clamp: the buffers then hold the plain all-reduced mean gradient
    hyper = fg.hyper_default(lr_D=0.0, lr_G=0.0, D_L1=0.0, D_L2=0.0, G_L1=0.0, G_L2=0.0, D_clamp=0.0, G_clamp=0.0)
    ctx = fg.Context(rank, max_batch=B, channels=C, discriminator=name if S == 32 else "create_D32b")
    net = ctx if S == 32 else fg.S16(ctx, discriminator=name)
    PG = np.random.default_rng(900).uniform(-0.05, 0.05, net.nG).astype(np.float32)
    net.set_params(NET_G, PG)
    net.set_params(NET_D, R.make_params(ref, 902).astype(np.float32))
    args = (hyper, B, real, nD, nG, mD, mG)
    st1 = net.train_step(*args)
    single = (net.get_grads(NET_D), net.get_grads(NET_G), st1)
    ids = [ctx.dp_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.dp_init(ids[0], world, rank)
    st2 = net.train_step(*args)
    q.put((rank, single, (net.get_grads(NET_D), net.get_grads(NET_G), st2)))
    dist.barrier()
    if net is not ctx:
        net.close()
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("name,port", [("create_D32", 29801), ("create_D16_b", 29803)])
def test_dp_disc_two_gpus_average_gradients(name, port):
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    import parity_utils as PU
    world = 2
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker, args=(r, world, port, name, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r = q.get(timeout=600)
        got[r[0]] = r
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for k in (0, 1):  # D gradient, G gradient
        np.testing.assert_array_equal(got[0][2][k], got[1][2][k])  # replicas identical
        mean = 0.5 * (got[0][1][k].astype(np.float64) + got[1][1][k].astype(np.float64))
        assert PU.relerr(got[0][2][k], mean) < 2e-5
    conf = [a + b for a, b in zip(got[0][1][2]["conf"], got[1][1][2]["conf"])]
    assert got[0][2][2]["conf"] == conf == got[1][2][2]["conf"]
