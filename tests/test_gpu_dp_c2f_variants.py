"""Data parallel on a coarse-to-fine pair other than the default (create_G_a / create_D_b; needs >= 2 GPUs, skipped on
one): two processes, one per GPU, the c2f loop body inside a 2-rank group of the ctx's communicator.  Every rank must end
with the mean of the two per-shard gradients, the replicas must be identical, and the confusion counts must add up --
the counterpart of tests/test_gpu_dp.py::test_dp_c2f_two_gpus_average_gradients for the default pair."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

pytestmark = pytest.mark.gpu

GEN, DISC, S = "create_G_a", "create_D_b", 32


def _gpu_count():
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for line in out.splitlines() if line.startswith("GPU "))
    except Exception:
        return 0


def _worker(rank, world, port, q):
    import torch.distributed as dist
    import c2f_utils as CU
    import c2f_var_ref as V
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 8, 3
    base = V.make_case(B, C, S, GEN, DISC, seed=820)
    case = V.make_case(B, C, S, GEN, DISC, seed=821 + rank)
    # lr = 0, no penalty, no clamp: the gradient buffers then hold the plain all-reduced mean
    hyper = fg.hyper_default(**dict(CU.HYPER, lr_D=0.0, lr_G=0.0, D_L1=0.0, D_clamp=0.0, G_clamp=0.0))
    args = (hyper, B, case["real_diff"], case["cond_D"], case["noise_D"], case["cond_G"], case["noise_G"], case["masks_D"],
            case["masks_G"])
    # (a) this rank's shard alone
    ctx = fg.Context(rank, max_batch=B, channels=C)
    net = fg.C2f(ctx, S, GEN, DISC)
    net.set_params(NET_G, base["PG"])
    net.set_params(NET_D, base["PD"])
    st1 = net.train_step(*args)
    single = (net.get_grads(NET_D), net.get_grads(NET_G), st1)
    # (b) the same shard inside a 2-rank data-parallel group
    ids = [ctx.dp_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.dp_init(ids[0], world, rank)
    st2 = net.train_step(*args)
    q.put((rank, single, (net.get_grads(NET_D), net.get_grads(NET_G), st2)))
    dist.barrier()
    net.close()
    ctx.close()
    dist.destroy_process_group()


def test_dp_variant_pair_two_gpus_average_gradients():
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    import parity_utils as PU
    world, port = 2, 29771
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
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
    assert got[0][2][2]["conf"] == conf == got[1][2][2]["conf"]  # confusion counts ride the all-reduce
