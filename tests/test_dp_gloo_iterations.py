"""world_size-2 data-parallel semantics of several D and G iterations per call (train.lua --D_iterations /
--G_iterations), restated on CPU with the fp64 oracle over gloo: what fg_train_step_iters does for world > 1.

Every D iteration: its own fakes, D forward/backward on this rank's shard, the flat gradient and the confusion counts
all-reduced, 1/N scaling, penalty -> clamp, the accuracy gate on the global accuracy, Adam -- identically on every
rank, before the next iteration's G forward.  Every G iteration: G step on this rank's shard, all-reduce, 1/N,
penalty -> clamp -> Adam.  BatchNorm statistics stay per replica."""
import os
import sys
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

D_IT, G_IT, B, C, WORLD = 2, 1, 4, 1, 2


def rank_step_iters(cases_D, cases_G, st, B, C, world, allreduce, accs, hyper=None, max_acc=1.01, interval=1):
    """cases_D / cases_G: this rank's inputs per D / G iteration; st: replicated state (updated in place)."""
    import parity_utils as PU
    from oracle import oracle as O
    from face_generator_b200.adversarial import gate
    hp = hyper or PU.HYPER
    Bh = B // 2
    G, D = O.f64.G(), O.f64.D()
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)])
    conf_sum, trained, losses = np.zeros(4), 0, []
    for case in cases_D:
        fake = G.forward(st["PG"], case["noise_D"], C, True, st["bnG"])
        out = D.forward(st["PD"], np.concatenate([case["real"].astype(np.float64), fake]), case["masks_D"])
        gD, _ = D.backward(O.f64.bce_bwd(out, targets), want_dimg=False)
        conf = np.array([np.sum((out > 0.5) & (targets > 0.5)), np.sum((out <= 0.5) & (targets > 0.5)),
                         np.sum((out > 0.5) & (targets < 0.5)), np.sum((out <= 0.5) & (targets < 0.5))], np.float64)
        red = allreduce(np.concatenate([gD, conf]))
        gD, conf = red[:-4] / world, red[-4:]
        conf_sum += conf
        losses.append(O.f64.bce_fwd(out, targets))
        O.f64.penalty_clamp(st["PD"], gD, hp["D_L1"], hp["D_L1"], hp["D_L2"], hp["D_clamp"])
        if gate(accs, (conf[0] + conf[3]) / (B * world), max_acc, interval):  # the gate sees the global accuracy
            trained += 1
            st["tD"] += 1
            O.f64.adam(st["PD"], gD, st["mD"], st["vD"], st["tD"], hp["lr_D"], hp["beta1"], hp["beta2"], hp["eps"])
    for case in cases_G:
        img = G.forward(st["PG"], case["noise_G"], C, True, st["bnG"])
        out = D.forward(st["PD"], img, case["masks_G"])
        _, dimg = D.backward(O.f64.bce_bwd(out, np.ones(B)), want_dP=False)
        gG = allreduce(G.backward(dimg)) / world
        l1g = hp["G_L2"] if (hp["G_L1"] != 0 or hp["G_L2"] != 0) else 0.0
        O.f64.penalty_clamp(st["PG"], gG, hp["G_L1"], l1g, hp["G_L2"], hp["G_clamp"])
        st["tG"] += 1
        O.f64.adam(st["PG"], gG, st["mG"], st["vG"], st["tG"], hp["lr_G"], hp["beta1"], hp["beta2"], hp["eps"])
    return dict(conf=conf_sum, trained=trained, lossD=losses)


def _cases(rank):
    import parity_utils as PU
    base = PU.make_case(B, C, seed=930)  # identical initial parameters on every rank
    cD = [PU.make_case(B, C, seed=931 + 10 * j + rank) for j in range(D_IT)]  # rank- and iteration-distinct shards
    cG = [PU.make_case(B, C, seed=971 + 10 * j + rank) for j in range(G_IT)]
    for c in cD + cG:
        c["PG"], c["PD"] = base["PG"], base["PD"]
    return base, cD, cG


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    import parity_utils as PU
    from oracle import oracle as O
    O.set_num_threads(2)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    base, cD, cG = _cases(rank)
    st = PU.fresh_state(base)

    def allreduce(a):
        t = torch.from_numpy(np.ascontiguousarray(a, np.float64).copy())
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return t.numpy()

    res = rank_step_iters(cD, cG, st, B, C, world, allreduce, [])
    q.put((rank, st["PD"].copy(), st["PG"].copy(), st["bnG"].copy(), res["conf"].copy(), res["trained"], st["tD"], st["tG"]))
    dist.barrier()
    dist.destroy_process_group()


def test_dp_world2_gloo_iterations_replicas_identical_and_equal_serial():
    import torch.multiprocessing as mp
    import parity_utils as PU
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, WORLD, 29737, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(WORLD):
        r = q.get(timeout=600)
        got[r[0]] = r
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    # replicas stay bit-identical through every iteration's all-reduce + optimizer
    np.testing.assert_array_equal(got[0][1], got[1][1])
    np.testing.assert_array_equal(got[0][2], got[1][2])
    assert got[0][4].sum() == D_IT * B * WORLD  # conf: global, summed over the D iterations
    assert got[0][5] == D_IT and got[0][6] == D_IT and got[0][7] == G_IT
    # BatchNorm running statistics are per replica (each rank's own fakes and samples)
    assert not np.array_equal(got[0][3], got[1][3])
    # serial emulation: both ranks in threads, the all-reduce an explicit sum of the two contributions
    bufs, lock, bar = {}, threading.Lock(), threading.Barrier(WORLD)

    def make_allreduce(rank):
        def ar(a):
            with lock:
                bufs[rank] = np.array(a, np.float64)
            bar.wait()
            tot = bufs[0] + bufs[1]
            bar.wait()
            return tot
        return ar

    states, outs = [None, None], [None, None]

    def run(rank):
        base, cD, cG = _cases(rank)
        states[rank] = PU.fresh_state(base)
        outs[rank] = rank_step_iters(cD, cG, states[rank], B, C, WORLD, make_allreduce(rank), [])

    ths = [threading.Thread(target=run, args=(r,)) for r in range(WORLD)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert np.abs(got[0][1] - states[0]["PD"]).max() < 1e-12
    assert np.abs(got[0][2] - states[0]["PG"]).max() < 1e-12


def test_one_iteration_each_is_the_single_iteration_dp_step():
    """d = g = 1 of the restatement is dp_ref.rank_step (the existing DP semantics), at world 1"""
    import dp_ref
    import parity_utils as PU
    base, cD, cG = _cases(0)
    case = dict(cD[0])
    case["noise_G"], case["masks_G"] = cG[0]["noise_G"], cG[0]["masks_G"]
    s1, s2 = PU.fresh_state(base), PU.fresh_state(base)
    dp_ref.rank_step(case, s1, B, C, 1, lambda a: np.array(a, np.float64))
    rank_step_iters([cD[0]], [cG[0]], s2, B, C, 1, lambda a: np.array(a, np.float64), [])
    for k in ("PD", "PG", "mD", "vD", "mG", "vG", "bnG"):  # the same fp64 arithmetic, up to summation order
        assert np.abs(s1[k] - s2[k]).max() <= 1e-12 * max(1.0, np.abs(s1[k]).max()), k
    assert s1["tD"] == s2["tD"] == 1 and s1["tG"] == s2["tG"] == 1
