"""Data-parallel parity on real GPUs (needs >= 2 GPUs; skipped on one GPU).
Two processes, one per GPU, NCCL all-reduce inside fg_train_step; checked against the oracle-based DP
restatement (tests/dp_ref.py) and for replica equality."""
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


def _worker(rank, world, port, impl, q):
    import torch.distributed as dist
    import parity_utils as PU
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 8, 3
    base = PU.make_case(B, C, seed=700)
    case = PU.make_case(B, C, seed=701 + rank)
    ctx = fg.Context(rank, max_batch=B, channels=C)
    ctx.set_option("conv_impl", impl)
    # rank 1 starts from garbage on purpose: fg_dp_broadcast_params must overwrite it with rank 0's
    ctx.set_params(NET_G, base["PG"] if rank == 0 else base["PG"] * 0 + 0.123)
    ctx.set_params(NET_D, base["PD"] if rank == 0 else base["PD"] * 0 - 0.321)
    ids = [ctx.dp_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.dp_init(ids[0], world, rank)
    ctx.dp_broadcast_params()
    st = ctx.train_step(fg.hyper_default(), B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
    q.put((rank, ctx.get_params(NET_D), ctx.get_params(NET_G), ctx.get_grads(NET_D), ctx.get_grads(NET_G), st))
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("impl", [0, 2])
def test_dp_two_gpus_match_oracle_and_each_other(impl):
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import threading
    import torch.multiprocessing as mp
    import parity_utils as PU
    import dp_ref
    world, port = 2, 29741 + impl
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker, args=(r, world, port, impl, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r = q.get(timeout=600)
        got[r[0]] = r
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    # replicas bit-identical after the step
    np.testing.assert_array_equal(got[0][1], got[1][1])
    np.testing.assert_array_equal(got[0][2], got[1][2])
    np.testing.assert_array_equal(got[0][3], got[1][3])
    assert got[0][5]["conf"] == got[1][5]["conf"] and sum(got[0][5]["conf"]) == 16  # global confusion counts
    # oracle emulation of the two ranks
    B, C = 8, 3
    base = PU.make_case(B, C, seed=700)
    cases, states = [], []
    for r in range(world):
        cs = PU.make_case(B, C, seed=701 + r)
        cs["PG"], cs["PD"] = base["PG"], base["PD"]
        cases.append(cs)
        states.append(PU.fresh_state(cs))
    bufs, lock, bar, out = {}, threading.Lock(), threading.Barrier(world), [None, None]

    def make_ar(rank):
        def ar(a):
            with lock:
                bufs[rank] = np.array(a, np.float64)
            bar.wait()
            tot = bufs[0] + bufs[1]
            bar.wait()
            return tot
        return ar

    ths = [threading.Thread(target=lambda r=r: out.__setitem__(r, dp_ref.rank_step(cases[r], states[r], B, C, world, make_ar(r))))
           for r in range(world)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    # gradients after all-reduce + 1/N + penalty + clamp (kink flips possible: 2e-2 bar, see DESIGN.md section 5)
    assert PU.relerr(got[0][3], out[0]["gradD"]) < 2e-2
    assert PU.relerr(got[0][4], out[0]["gradG"]) < 2e-2
    assert abs(got[0][5]["loss_D"] - out[0]["lossD"]) < 1e-4 * max(1, abs(out[0]["lossD"]))


def _worker_c2f(rank, world, port, q):
    import torch.distributed as dist
    import c2f_utils as CU
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 8, 3
    base = CU.make_case(B, C, seed=800, init="smooth")
    case = CU.make_case(B, C, seed=801 + rank, init="smooth")
    # lr = 0, no penalty, no clamp: the buffers then hold the plain all-reduced mean gradient
    hyper = fg.hyper_default(**dict(CU.HYPER, lr_D=0.0, lr_G=0.0, D_L1=0.0, D_clamp=0.0, G_clamp=0.0))
    args = (hyper, B, case["real_diff"], case["cond_D"], case["noise_D"], case["cond_G"], case["noise_G"], case["masks_D"],
            case["masks_G"])
    # (a) single-GPU reference of this rank's shard
    ctx = fg.Context(rank, max_batch=B, channels=C)
    net = fg.C2f(ctx)
    net.set_params(NET_G, base["PG"])
    net.set_params(NET_D, base["PD"])
    st1 = net.train_step(*args)
    single = (net.get_grads(NET_D), net.get_grads(NET_G), st1)
    # (b) the same shard inside a 2-rank data-parallel group (the c2f loop shares the ctx's communicator)
    ids = [ctx.dp_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.dp_init(ids[0], world, rank)
    st2 = net.train_step(*args)
    q.put((rank, single, (net.get_grads(NET_D), net.get_grads(NET_G), st2)))
    dist.barrier()
    net.close()
    ctx.close()
    dist.destroy_process_group()


def test_dp_c2f_two_gpus_average_gradients():
    """adversarial_c2f loop under data parallelism: every rank ends with the mean of the per-shard gradients."""
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    import parity_utils as PU
    world, port = 2, 29761
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker_c2f, args=(r, world, port, q)) for r in range(world)]
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


def _worker_resume(rank, world, port, q):
    import torch.distributed as dist
    import parity_utils as PU
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 8, 3
    base = PU.make_case(B, C, seed=900)
    ctx = fg.Context(rank, max_batch=B, channels=C)
    if rank == 0:  # "load_flat_checkpoint on rank 0": parameters, moments AND step counters t_D = 7, t_G = 5
        rng = np.random.default_rng(9)
        ctx.set_params(NET_G, base["PG"])
        ctx.set_params(NET_D, base["PD"])
        ctx.set_adam_state(NET_D, rng.standard_normal(ctx.nD) * 1e-3, rng.random(ctx.nD) * 1e-5, 7)
        ctx.set_adam_state(NET_G, rng.standard_normal(ctx.nG) * 1e-3, rng.random(ctx.nG) * 1e-5, 5)
    ids = [ctx.dp_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.dp_init(ids[0], world, rank)
    ctx.dp_broadcast_params()
    t0 = (ctx.get_adam_state(NET_D)[2], ctx.get_adam_state(NET_G)[2])
    for it in range(3):
        case = PU.make_case(B, C, seed=910 + 10 * it + rank)
        st = ctx.train_step(fg.hyper_default(), B, case["real"], case["noise_D"], case["noise_G"], case["masks_D"], case["masks_G"])
    q.put((rank, t0, (st["t_D"], st["t_G"]), ctx.get_params(NET_D), ctx.get_params(NET_G), ctx.get_adam_state(NET_D)[0]))
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


def test_dp_resume_broadcasts_step_counters():
    """fg_dp_broadcast_params carries t_D / t_G (Adam's bias correction depends on them): after a resume on rank 0
    only, replicas must stay bit-identical over the following steps."""
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, 29781
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker_resume, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r = q.get(timeout=600)
        got[r[0]] = r
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert got[0][1] == got[1][1] == (7, 5)
    assert got[0][2] == got[1][2] == (10, 8)
    for k in (3, 4, 5):
        np.testing.assert_array_equal(got[0][k], got[1][k])


def _worker_overlap(rank, world, port, q):
    import torch.distributed as dist
    import parity_utils as PU
    import face_generator_b200 as fg
    from face_generator_b200.lib import NET_D, NET_G
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, C = 16, 3
    base = PU.make_case(B, C, seed=800)
    cases = [PU.make_case(B, C, seed=801 + rank + 10 * s) for s in range(3)]
    res = []
    for overlap in (1, 0):
        ctx = fg.Context(rank, max_batch=B, channels=C)
        ctx.set_option("dp_overlap", overlap)
        ctx.set_params(NET_G, base["PG"])
        ctx.set_params(NET_D, base["PD"])
        ids = [ctx.dp_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        ctx.dp_init(ids[0], world, rank)
        ctx.dp_broadcast_params()
        sts = [ctx.train_step(fg.hyper_default(), B, cs["real"], cs["noise_D"], cs["noise_G"], cs["masks_D"], cs["masks_G"])
               for cs in cases]
        res.append((ctx.get_params(NET_D), ctx.get_params(NET_G), [s["loss_D"] for s in sts], [s["loss_G"] for s in sts],
                    [list(s["conf"]) for s in sts]))
        dist.barrier()
        ctx.close()
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def test_dp_overlap_matches_serial_schedule():
    """option dp_overlap: D's all-reduce + gate + optimizer on the communication stream while the G step's G forward
    runs -- three steps give the losses, confusion counts and (up to run-to-run rounding) parameters of the serial schedule,
    and the two ranks stay bit-identical."""
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, 29761
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker_overlap, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r = q.get(timeout=600)
        got[r[0]] = r[1]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    # Two RUNS are not bit-reproducible (the split-K weight-gradient kernels add their partial tiles with fp32 atomics in
    # arrival order), so overlap vs serial is compared like two runs of the same schedule: identical confusion counts,
    # losses to 1e-5, parameters equal except where Adam amplifies a rounding-level gradient difference to +-lr per step.
    # What must hold EXACTLY is that the two ranks of one run end with identical parameters -- a race between the
    # communication stream and the compute stream would hit the ranks differently.
    for r in range(world):
        ov, ser = got[r]
        assert ov[4] == ser[4]
        assert np.allclose(ov[2], ser[2], rtol=1e-5, atol=1e-6) and np.allclose(ov[3], ser[3], rtol=1e-5, atol=1e-6)
        for k in (0, 1):
            d = np.abs(ov[k].astype(np.float64) - ser[k])
            assert d.max() <= 3 * 2e-3 + 1e-6 and np.mean(d > 1e-5) < 0.05, (k, d.max(), np.mean(d > 1e-5))
    for mode in (0, 1):  # replicas identical under both schedules
        np.testing.assert_array_equal(got[0][mode][0], got[1][mode][0])
        np.testing.assert_array_equal(got[0][mode][1], got[1][mode][1])
