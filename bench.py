#!/usr/bin/env python
"""bench.py -- images/sec of the GAN train step (adversarial.lua loop body: 1 D iteration + 1 G iteration,
both Adam updates) on synthetic 3x32x32 batches, batch 256 per GPU (BASELINE.json configs[1]; weak scaling).

  python bench.py --gpus N --steps K --warmup W              our arm (libfg_b200.so through the C ABI, sm_90a)
  python bench.py --impl reference --gpus N --steps K ...    the reference's CPU math (oracle fp32 port; Torch7
                                                             itself cannot run in this image, see DESIGN.md)
Prints ONE JSON line on rank 0.
"""
import os
import sys

# stdout carries exactly ONE line (the JSON result of rank 0).  NCCL logs to the process's stdout (fd 1) -- the box
# environment presets NCCL_DEBUG=VERSION, and settings made later in the process (NCCL_DEBUG_FILE, tried in round 2)
# were not picked up -- so: keep a private handle on the real stdout for the result line, point fd 1 at stderr for
# everything any native library prints, and raise NCCL's level to INFO (INIT lines: "... rank r nranks N ...") before
# anything else is imported, unless the caller already asked for INFO / TRACE.
_RESULT_OUT = os.fdopen(os.dup(1), "w")
os.dup2(2, 1)
if int(os.environ.get("WORLD_SIZE", "1")) > 1:
    if os.environ.get("NCCL_DEBUG", "").upper() not in ("INFO", "TRACE"):
        os.environ["NCCL_DEBUG"] = "INFO"
    os.environ.setdefault("NCCL_DEBUG_SUBSYS", "INIT")

import argparse  # noqa: E402
import json  # noqa: E402
import subprocess  # noqa: E402
import threading  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402


def emit(obj):
    """the one result line, on the real stdout"""
    _RESULT_OUT.write(json.dumps(obj) + "\n")
    _RESULT_OUT.flush()


ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
# The CPU port's GEMMs go through the OpenBLAS bundled with scipy, as Torch7's `nn` calls the system BLAS on a CPU box
# (FG_ORACLE_BLAS=0 falls back to the port's own blocked loops).  OpenBLAS worker threads must not fight spinning
# OpenMP threads, so OpenMP idles passively (read when libgomp initialises => set before any import).
USE_BLAS = os.environ.get("FG_ORACLE_BLAS", "1") != "0"
if USE_BLAS:
    os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")


def port_gemm(O):
    """-> description of the GEMM the fp32 oracle port uses in this process."""
    if USE_BLAS and O.use_blas(cpu_threads()):
        return "OpenBLAS sgemm (scipy.libs)"
    return "blocked OpenMP loops"


def workload_config(world, B=256):
    """the `config` object both arms print (the reference arm runs our arm's config, bench contract)"""
    return {"workload": "train.lua color 3x32x32 batch=256 per GPU (BASELINE configs[1]), 1 D-iter + 1 G-iter, Adam",
            "global_batch": B * world, "per_gpu_batch": B, "parallelism": "dp%d" % world, "dropout": "in-kernel RNG",
            "l2": "per-step working set (activations+grads ~1.5 GB) >> 50 MB L2, no explicit flush"}


class CpuPort:
    """The reference's CPU math (Torch7 `nn`: per-sample im2col + SGEMM, batch-parallel) as restated by the oracle's
    fp32 port, on all usable host threads: one adversarial.lua iteration at batch b."""

    def __init__(self):
        from oracle import oracle as O
        from face_generator_b200 import layouts as LY
        self.O, self.C = O, 3
        O.set_num_threads(cpu_threads())
        self.gemm = port_gemm(O)
        rng = np.random.default_rng(1)
        PG, PD = LY.trained_like_init(LY.G_layout(3), rng), LY.trained_like_init(LY.D_layout(3), rng, 1.4)
        self.st = dict(PD=PD, PG=PG, mD=np.zeros_like(PD), vD=np.zeros_like(PD), mG=np.zeros_like(PG), vG=np.zeros_like(PG),
                       tD=0, tG=0, bnG=np.concatenate([np.zeros(256), np.ones(256), np.zeros(128), np.ones(128)]).astype(np.float32))
        self.hyper = dict(lr_D=1e-3, lr_G=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, D_L1=0.0, D_L2=1e-4, G_L1=0.0, G_L2=0.0,
                          D_clamp=1.0, G_clamp=5.0)
        self.inputs = {}

    def step(self, b):
        if b not in self.inputs:
            rng = np.random.default_rng(b)
            self.inputs[b] = synth_inputs(b, self.C, 7) + ((rng.random((b, self.O.MASK_PER_SAMPLE)) < 0.7).astype(np.float32),)
        real, nD, nG, masks = self.inputs[b]
        t0 = time.perf_counter()
        self.O.f32.train_iteration(b, self.C, self.hyper, real, nD, nG, masks, masks, self.st, want_grads=False)
        return time.perf_counter() - t0

    def pick_batch(self, n_steps, budget_s):
        """largest b in {256,...,16} whose n_steps iterations fit the time budget (calibrated on one batch-16 step;
        the iteration cost is linear in b).  256 = the whole configs[1] step."""
        self.step(16)
        t16 = self.step(16)
        for b in (256, 128, 64, 32):
            if n_steps * t16 * b / 16.0 <= budget_s:
                return b
        return 16

METRIC = "32x32 GAN train images/sec (1 D-iter + 1 G-iter per batch, batch 256/GPU)"
# algorithmic FLOPs (SURVEY.md 8d): conv = 2*Cout*Cin*k*k*H*W per image per pass
F_GC2 = 2 * 128 * 256 * 25 * 32 * 32      # 1677.72 MF
F_GC1 = 2 * 256 * 128 * 25 * 16 * 16      # 419.43 MF
F_ITER_PER_IMG = 8.087e9                  # reference-executed FLOPs per batch-image per iteration


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d["hbm_gbs"], bf16=d["bf16_tflops"], bf16_sus=d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                    src="measured")
    # NVIDIA's data sheet for the H100 SXM (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s -- not reached figures
    return dict(hbm=3350.0, bf16=989.0, bf16_sus=989.0, src="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def cpu_threads():
    """The oracle port parallelises one sample's GEMM over 4-row blocks of <=256 output rows, so more than 32
    threads only add contention (measured: 128 threads are 10x slower than 32 on the GPU box's host)."""
    return max(1, min(os.cpu_count() or 1, 32))


def synth_inputs(B, C, seed):
    rng = np.random.default_rng(seed)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    return (f(rng.random((B // 2, C, 32, 32))), f(rng.uniform(-1, 1, (B // 2, 100))), f(rng.uniform(-1, 1, (B, 100))))


def run_reference(args, rank, world):
    """The reference's own CPU path on this box's host cores, same metric / config.  Each step is the full
    256-image iteration when K+W of them fit ~3 minutes, otherwise the largest power-of-two sample of the batch that
    does (`sample` says which)."""
    if rank != 0:
        return
    port = CpuPort()
    warm = max(1, min(args.warmup, 2))
    b = port.pick_batch(args.steps + warm, 170.0)
    for _ in range(warm):
        port.step(b)
    dt = sum(port.step(b) for _ in range(args.steps))
    v = b * args.steps / dt
    whole = "the whole 256-image batch" if b == 256 else "a %d-image sample of the 256-image batch" % b
    sample = "%s per step, %d steps, fp32 oracle port (THNN algorithm, %s), %d threads" % (whole, args.steps, port.gemm,
                                                                                         port.O.num_threads())
    emit({
        "impl": "reference", "metric": METRIC, "value": v, "unit": "images/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args.gpus),
        "reference_detail": {"device": "cpu", "images_per_step": b, "gemm": port.gemm},
        "cpu_baseline": {"value": v, "unit": "images/s", "cores": port.O.num_threads(), "kind": "port", "sample": sample},
        "e2e": {"value": v, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}})


def secondary_configs(steps=5):
    """the other BASELINE.json configs, measured like the headline (CUDA events on the ctx stream, warm-up, inputs in
    HBM; e2e with host buffers): configs[0] gray batch 16, configs[3] c2f batch 32 / 256, configs[4] sample.lua 1024."""
    sys.path.insert(0, os.path.join(ROOT, "profiles"))
    res = []
    try:
        import bench_configs as BC
        for job in (lambda: BC.train_small(16, 1, steps), lambda: BC.c2f(32, steps), lambda: BC.c2f(256, steps),
                    lambda: BC.sample(16, steps), lambda: BC.sample(1024, steps), lambda: BC.train_s16(256, steps)):
            r = job()
            r.pop("layer_ms_per_step", None)
            res.append(r)
    except Exception as e:
        res.append({"error": str(e)})
    return res


def dump_outputs(ctx, out_dir):
    """The state one train step leaves behind, as a caller of fg_train_step reads it back: updated parameters, the
    step's gradients and the BatchNorm running statistics (~43 MB of float32 for the colour nets)."""
    from face_generator_b200.lib import NET_D, NET_G
    os.makedirs(out_dir, exist_ok=True)
    arrays = {"params_G": ctx.get_params(NET_G), "params_D": ctx.get_params(NET_D), "grads_G": ctx.get_grads(NET_G),
              "grads_D": ctx.get_grads(NET_D), "bn_state_G": ctx.get_bn_state()}
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), np.ascontiguousarray(a, np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=256, help="per-GPU batch (BASELINE configs[1]: 256)")
    ap.add_argument("--conv-impl", type=int, default=-1, help="0 simt, 1 wgmma dense, 2 wgmma collapsed; -1 library default")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true", help="skip the configs[0]/[3]/[4] lines of the `secondary` block")
    ap.add_argument("--breakdown", action="store_true", help="per-layer kernel timings in kernel_ms_per_step")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed (parameters, gradients and BatchNorm "
                         "running state of rank 0) as DIR/<name>.npy in float32")
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if args.impl == "reference":
        return run_reference(args, rank, world)

    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.lib import NET_D, NET_G, PinnedArray
    B, C, K, W = args.batch, 3, args.steps, max(args.warmup, 3)
    dist = None
    # (NCCL's log -- INIT lines carry "nranks N" -- goes to stderr: see the top of this file)
    if world > 1:
        import torch.distributed as dist  # plumbing only: rendezvous, barrier, max-over-ranks
        dist.init_process_group("gloo")
    ctx = fg.Context(local, max_batch=B, channels=C)
    if args.conv_impl >= 0:
        ctx.set_option("conv_impl", args.conv_impl)
    rng = np.random.default_rng(1)  # identical initial parameters on every rank
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    if world > 1:
        ids = [ctx.dp_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        ctx.dp_init(ids[0], world, rank)
        ctx.dp_broadcast_params()
    hyper = fg.hyper_default()
    real, nD, nG = synth_inputs(B, C, 100 + rank)  # rank-distinct shards
    d_real, d_nD, d_nG = ctx.dev_array(real), ctx.dev_array(nD), ctx.dev_array(nG)
    p_real, p_nD, p_nG = PinnedArray(real.shape), PinnedArray(nD.shape), PinnedArray(nG.shape)
    p_real.array[:], p_nD.array[:], p_nG.array[:] = real, nD, nG

    def barrier():
        ctx.sync()
        if dist:
            dist.barrier()

    def max_over_ranks(x):
        if not dist:
            return x
        import torch
        t = torch.tensor([x], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0])

    seed = [1000 * rank]

    def step_resident():
        seed[0] += 1
        ctx.train_step(hyper, B, d_real, d_nD, d_nG, None, None, seed[0], want_stats=False)

    def step_e2e():
        seed[0] += 1
        # H2D of this step's inputs from pinned memory + D2H of the step's result (losses/stats) inside the call
        return ctx.train_step(hyper, B, p_real.addr, p_nD.addr, p_nG.addr, None, None, seed[0], want_stats=True)

    def timed(fn, k):
        barrier()
        ctx.event_record(0)
        for _ in range(k):
            fn()
        ctx.event_record(1)
        barrier()
        return max_over_ranks(ctx.event_elapsed_ms(0, 1))

    for _ in range(W):
        step_resident()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = ctx.launches()
    ms = timed(step_resident, K)
    launches = ctx.launches() - l0
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(ctx, args.dump_outputs)
    for _ in range(2):
        step_e2e()
    ms_e2e = timed(step_e2e, K)
    # dominant kernel family, timed live with CUDA events on the ctx stream (per launch)
    ctx.timing_enable(True)
    nprof = 3
    for _ in range(nprof):
        step_resident()
    fam = {}
    names = ["G.C2.fwd", "G.C2.dgrad", "G.C2.wgrad", "G.C1", "G.C3", "G.L1", "D.", "nccl"]
    if args.breakdown:
        names += ["G.C1.fwd", "G.C1.dgrad", "G.C1.wgrad", "G.C3.fwd", "G.C3.dgrad", "G.C3.wgrad"]
        names += ["D.%s.%s" % (l, k) for l in ("C1", "C2", "C3", "C4", "L1", "L2", "L3") for k in ("fwd", "dgrad", "wgrad")]
    for name in names:
        t, n = ctx.timing_get(name)
        fam[name] = (t / nprof, n // nprof)
    t_all = ctx.timing_get("G.")[0] + ctx.timing_get("D.")[0]
    # bandwidth-bound kernels: algorithmic bytes per step (fp32, B images in the G step + B/2 in the D step's G
    # forward) over the event-timed duration, against the measured HBM copy bandwidth
    act = B * 131072 * 4  # one [B][32][32][128] fp32 tensor
    hbm_bytes = {"hbm.G.bn2.stats": 1.5 * act,            # read z2
                 "hbm.G.bn2.apply": 1.5 * 2 * act,        # read z2, write h2
                 "hbm.G.bn2.bwd_reduce": 2 * act,         # read dh, z2
                 # read dh, z2; write dz2 (+ its TF32 hi/lo split on the 3xTF32 path; the FP16 split is a separate pass)
                 "hbm.G.bn2.bwd_apply": (3 if ctx.get_option("mma_f16") else 5) * act,
                 # the 3-channel-side 3x3 convolutions (k_conv_edge.cu): input + output of the images they process per step
                 "G.C3.fwd": 1.5 * B * 1024 * (128 + C) * 4,   # B/2 (D step) + B (G step) images
                 "G.C3.dgrad": B * 1024 * (C + 128) * 4,       # G step
                 "D.C1.fwd": 2 * B * 1024 * (C + 64) * 4,      # B (D step) + B (G step)
                 "D.C1.dgrad": B * 1024 * (64 + C) * 4,        # G step (gradient into G's image)
                 "hbm.optim.D": 28 * ctx.count(NET_D),    # p, g, m, v read; p, g, m, v... 7 streams x 4 B (SURVEY 8a X5)
                 "hbm.optim.G": 28 * ctx.count(NET_G)}
    hbm = {}
    for name, nbytes in hbm_bytes.items():
        t, n = ctx.timing_get(name)
        if n:
            hbm[name] = (nbytes, t / nprof)
    ctx.timing_enable(False)
    tf32_peak = tf32_peak_n128 = f16_peak = None
    if rank == 0:
        try:
            tf32_peak = ctx.tf32_peak(20000)
            os.environ["FG_TF32_PROBE_F16"] = "1"  # the same loop with f16 instructions (m64n256k16)
            f16_peak = ctx.tf32_peak(20000)
            os.environ.pop("FG_TF32_PROBE_F16")
            os.environ["FG_TF32_PROBE_N"] = "128"  # the N=128 instruction shape
            tf32_peak_n128 = ctx.tf32_peak(40000)
            os.environ.pop("FG_TF32_PROBE_N")
        except Exception as e:  # the probe must never cost the headline
            sys.stderr.write("tf32 peak probe failed: %s\n" % e)
    if rank != 0:
        return
    peaks = load_peaks()
    value = B * world * K / (ms / 1e3)
    e2e = B * world * K / (ms_e2e / 1e3)
    # G.C2 forward runs at B/2 (D step) and B (G step) per iteration: 1.5*B images of algorithmic work
    t_fwd = fam["G.C2.fwd"][0] / 1e3
    tf_fwd = 1.5 * B * F_GC2 / t_fwd / 1e12 if t_fwd > 0 else 0.0
    t_c2 = (fam["G.C2.fwd"][0] + fam["G.C2.dgrad"][0] + fam["G.C2.wgrad"][0]) / 1e3
    tf_c2 = 3.5 * B * F_GC2 / t_c2 / 1e12 if t_c2 > 0 else 0.0
    f16 = bool(ctx.get_option("mma_f16")) and ctx.get_option("conv_impl") == 2
    # f16 MMAs run at the bf16 dense rate, tf32 at half of it
    peak = peaks["bf16_sus"] if f16 else peaks["bf16_sus"] / 2.0
    mma_peak = f16_peak if f16 else tf32_peak
    # executed tensor-core work of that launch: 3 MMAs per logical MMA (3-term split), 9/25 of the taps (phase collapse)
    collapsed = ctx.get_option("conv_impl") == 2
    exec_ratio = 3.0 * (9.0 / 25.0 if collapsed else 1.0)
    out = {
        "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": workload_config(world, B),
        "config_detail": {"conv_impl": ctx.get_option("conv_impl"), "mma_f16": int(f16),
                          "operand_split": "3xFP16 (f16 wgmma, fp32 accumulate)" if f16 else "3xTF32 (tf32 wgmma)"},
        "e2e": {"value": e2e, "unit": "images/s", "ms_per_step": ms_e2e / K,
                "h2d_bytes_per_step": int(real.nbytes + nD.nbytes + nG.nbytes), "d2h_bytes_per_step": 40},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "roofline": {"kernel": "G.C2 5x5 conv 256->128 @32x32 forward (implicit GEMM M=B*1024,N=128,K=6400)",
                     "bound": "tensor", "achieved": tf_fwd, "peak": peak, "unit": "TFLOP/s",
                     "frac": tf_fwd / peak,
                     "traffic_note": "algorithmic bytes of the batch-256 launch: input hi+lo %s MB + output 134.2 MB + "
                                     "weights %s MB" % ("2x33.6" if f16 else "2x67.1", "4.7" if f16 else "9.4"),
                     "peak_source": ("%s bf16 %.1f TF (f16 MMAs run at the bf16 rate); algorithmic fp32 FLOPs" if f16 else
                                     "%s bf16 %.1f TF / 2 (tf32 MMAs run at half rate); algorithmic fp32 FLOPs") % (
                         peaks["src"], peaks["bf16_sus"]),
                     "executed_mma_tflops": tf_fwd * exec_ratio,
                     "executed_note": "%s MMAs actually issued: 3 per logical MMA (hi*hi + hi*lo + lo*hi)%s" % (
                         "f16" if f16 else "tf32", " x 9/25 taps (upsample folded into four 3x3 phase convolutions)" if collapsed else ""),
                     "measured_f16_peak": f16_peak,
                     "measured_tf32_peak": tf32_peak,
                     "measured_tf32_peak_n128": tf32_peak_n128,
                     "measured_tf32_peak_note": "fg_bench_tf32_peak: back-to-back tf32 wgmma m64n256k8, two warpgroups per SM, "
                                                "smem-resident operands, all SMs, run at bench clocks right after the timed region",
                     "frac_executed_vs_measured_mma_peak": (tf_fwd * exec_ratio / mma_peak) if mma_peak else None,
                     "frac_algorithmic_vs_measured_mma_peak": (tf_fwd / mma_peak) if mma_peak else None,
                     "family_fwd_dgrad_wgrad_tflops": tf_c2,
                     "step_algorithmic_tflops": F_ITER_PER_IMG * B * K / (ms / 1e3) / 1e12},
        "hbm_kernels": [{"kernel": k[4:] if k.startswith("hbm.") else k, "bytes_per_step": int(nb), "ms_per_step": round(ms_k, 4),
                         "achieved": round(nb / (ms_k / 1e3) / 1e9, 1), "peak": peaks["hbm"], "unit": "GB/s",
                         "frac": round(nb / (ms_k / 1e3) / 1e9 / peaks["hbm"], 3)} for k, (nb, ms_k) in hbm.items() if ms_k > 0],
        "kernel_ms_per_step": {k: round(v[0], 4) for k, v in fam.items()},
        "conv_ms_per_step": round(t_all / nprof, 4),
    }
    if world == 1 and not args.no_secondary:
        out["secondary"] = secondary_configs()
    ctx.close()
    if world == 1 and not args.no_cpu_baseline:
        # cpu_baseline leg: the checker's fp32 port timed as a reported baseline on a bounded sample (10-30 s)
        port = CpuPort()
        b = port.pick_batch(1, 30.0)
        t, it = 0.0, 0
        while it < 1 or (t < 10.0 and it < 12):
            t += port.step(b)
            it += 1
        out["cpu_baseline"] = {"value": b * it / t, "unit": "images/s", "cores": port.O.num_threads(), "kind": "port",
                               "sample": "%d iteration(s) at batch %d of %d (colour) of the fp32 oracle port (%s), %.1f s" % (
                                   it, b, B, port.gemm, t)}
    emit(out)


if __name__ == "__main__":
    main()
