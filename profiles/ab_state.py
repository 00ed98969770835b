"""Bit-for-bit A/B of two builds of libfg_b200.so.

`run` loads the library at --lib, and for each case (net, batch, options, step mode) runs 3 host-fed and 3 device-fed
seeded train steps, then one G forward / G backward / D forward / D backward call.  The step modes are the
single-iteration entries, the *_iters / *_dataset_iters entries at 2 D and 2 G iterations ("iters2x2"), and the single
entries with option debug_keep, saving every Dstep.* tensor after each step ("debug_keep").  The coarse-to-fine nets
also run at fine sizes 16 and 64.  The dbr group runs models.lua's other discriminators at batch 256: create_D32 on
the 32x32 nets, create_D16 / _b / _c on the --scale 16 nets.  It writes every piece of state as .npy under
--out/<case>/: parameters, gradients, optimizer m / v / t, BatchNorm running state, the step statistics, the outputs
of those calls and the generator's debug tensors, plus the kernel launches of each step (launches.json).  The L-op
convolutions (fg_conv2d_*) with the 3xFP16 split are one more case.  The denoiser and the autoencoder run 6 seeded train
steps with option mma_f16 switched off for the middle two, then save parameters, gradients, Adam and BatchNorm state and
forward outputs.  Each run also records the free device memory after fg_create at batch 256 (free_after_create.json).  `compare A B` reports, per case, the first array
that differs and the launches per step of both builds; a case differs when either does.

One build per process: both libraries export the same symbols.

The c2f group also runs the default pair at every fine size, batch 256 and 130, mma_f16 1 and 0; the c2fvar group (not
in the default --only) runs models_c2f.lua's other generators and discriminators, for builds that have them.

usage:  python profiles/ab_state.py run --lib face_generator_b200/libfg_b200.so --out /tmp/ab/new [--only 32,s16,dbr,c2f,lop,dn,ae]
        python profiles/ab_state.py compare /tmp/ab/old /tmp/ab/new
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

C = 3
OPTS_32 = [("default", {}), ("mma_f16=0", {"mma_f16": 0}), ("conv_impl=0", {"conv_impl": 0}),
           ("conv_impl=1", {"conv_impl": 1}), ("bn_epilogue=0", {"bn_epilogue": 0}), ("edge_impl=0", {"edge_impl": 0}),
           ("bwd_merge=0", {"bwd_merge": 0}), ("bwd_merge=2", {"bwd_merge": 2}), ("use_graph=0", {"use_graph": 0})]
OPTS_S16 = OPTS_32[:4]
G_DEBUG_32 = ["G." + n for n in ("z0", "h0", "z1", "h1", "z2", "h2", "z3", "y", "dz2", "dz1", "dz0",
                                 "bn_mean1", "bn_istd1", "bn_mean2", "bn_istd2")]
G_DEBUG_S16 = ["G." + n for n in ("z0", "z1", "z2", "z3", "bn_mean1", "bn_istd1", "bn_mean2", "bn_istd2")]
DSTEP = {"32": ("z1", "z2", "z3", "z4", "zl1", "zl2", "logit", "out"),
         "s16": ("z1", "z2", "z3", "z4", "zf", "ze1", "ze2", "logit", "out"),
         "c2f": ("z1", "z2", "z3", "z4", "zl1", "logit", "out")}
ITERS = 2  # D and G iterations of the "iters2x2" mode


def f32(a):
    return np.ascontiguousarray(a, np.float32)


def pair_state(net, bn):
    from face_generator_b200.lib import NET_D, NET_G
    out = {}
    for k, w in ((NET_G, "G"), (NET_D, "D")):
        m, v, t = net.get_adam_state(k)
        out.update({"params_" + w: net.get_params(k), "grads_" + w: net.get_grads(k), "adam_m_" + w: m, "adam_v_" + w: v,
                    "adam_t_" + w: np.array([t])})
    if bn:
        out["bn_state"] = net.get_bn_state()
    return out


def stats_array(st):
    return np.concatenate([np.ravel(np.asarray(st[k], np.float64)) for k in sorted(st)])


def steps(ctx, out, host_step, dev_step, net=None, kind=None):
    """3 host-fed, then 3 device-fed steps (eager, captured, replayed where the net captures graphs).  With `kind`
    (debug_keep set), the Dstep.* tensors of `net` after each step too."""
    launches = []
    for i in range(6):
        l0 = ctx.launches()
        st = host_step(10 + i) if i < 3 else dev_step(10 + i)
        ctx.sync()
        launches.append(ctx.launches() - l0)
        out["stats_%d" % i] = stats_array(st)
        for n in DSTEP.get(kind, ()):
            out["Dstep.%s_%d" % (n, i)] = net.debug_tensor("Dstep." + n)
    return launches


def n_rows(mode):
    """the stacked iterations of one host-fed input ([] for the single-iteration entries)"""
    return [ITERS] if mode == "iters2x2" else []


def case_32(B, opts, imgs, mode="step", discriminator=None):
    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    rng = np.random.default_rng(7)
    ctx = fg.Context(0, max_batch=B, channels=C, **({"discriminator": discriminator} if discriminator else {}))
    for k, v in opts.items():
        ctx.set_option(k, v)
    if mode == "debug_keep":
        ctx.set_option("debug_keep", 1)
    ctx.set_params(NET_G, LY.trained_like_init(LY.G_layout(C), rng))
    if discriminator:
        ctx.set_params(NET_D, f32(rng.standard_normal(ctx.count(NET_D)) * 0.02))
    else:
        ctx.set_params(NET_D, LY.trained_like_init(LY.D_layout(C), rng, 1.4))
    ds = DeviceDataset(ctx, imgs)
    h = fg.hyper_default()
    out = {}

    r = n_rows(mode)

    def host(seed):
        real = f32(rng.random(r + [B // 2, C, 32, 32]))
        zD, zG = f32(rng.uniform(-1, 1, r + [B // 2, 100])), f32(rng.uniform(-1, 1, r + [B, 100]))
        if r:
            return ctx.train_step_iters(h, B, ITERS, ITERS, real, zD, zG, None, None, seed)
        return ctx.train_step(h, B, real, zD, zG, None, None, seed)

    def dev(seed):
        return ds.train_step_iters(h, B, ITERS, ITERS, seed) if r else ds.train_step(h, B, seed)

    launches = steps(ctx, out, host, dev, ctx, "32" if mode == "debug_keep" else None)
    out.update(pair_state(ctx, True))
    out["G_forward"] = ctx.G_forward(f32(rng.uniform(-1, 1, (B, 100))), training=True)
    out["G_backward.dnoise"] = ctx.G_backward(f32(rng.standard_normal((B, C, 32, 32)) * 1e-2), want_dnoise=True)
    for n in G_DEBUG_32:
        out["debug." + n] = ctx.debug_tensor(n)
    out["D_forward"] = ctx.D_forward(f32(rng.random((B, C, 32, 32))), None, True, 3)
    out["D_backward.dimages"] = ctx.D_backward(f32(rng.standard_normal(B)), True, True)
    out["grads_G_after_calls"], out["grads_D_after_calls"] = ctx.get_grads(NET_G), ctx.get_grads(NET_D)
    out["sample_chunk16"] = ctx.sample(f32(rng.uniform(-1, 1, (40, 100))), 16)
    ds.close()
    ctx.close()
    return out, launches


def case_s16(B, opts, imgs, mode="step", discriminator=None):
    import face_generator_b200 as fg
    from face_generator_b200.dataset import DeviceDataset
    from face_generator_b200.lib import NET_D, NET_G
    rng = np.random.default_rng(41)
    ctx = fg.Context(0, max_batch=B, channels=C)
    for k, v in opts.items():
        ctx.set_option(k, v)
    if mode == "debug_keep":
        ctx.set_option("debug_keep", 1)
    net = fg.S16(ctx, **({"discriminator": discriminator} if discriminator else {}))
    net.set_params(NET_G, f32(rng.standard_normal(net.count(NET_G)) * 0.02))
    net.set_params(NET_D, f32(rng.standard_normal(net.count(NET_D)) * 0.02))
    ds = DeviceDataset(ctx, imgs)
    h = fg.hyper_default()
    out = {}

    r = n_rows(mode)

    def host(seed):
        real = f32(rng.random(r + [B // 2, C, 16, 16]))
        zD, zG = f32(rng.uniform(-1, 1, r + [B // 2, 100])), f32(rng.uniform(-1, 1, r + [B, 100]))
        if r:
            return net.train_step_iters(h, B, ITERS, ITERS, real, zD, zG, None, None, seed)
        return net.train_step(h, B, real, zD, zG, None, None, seed)

    def dev(seed):
        return net.train_step_dataset_iters(ds, h, B, ITERS, ITERS, seed) if r else net.train_step_dataset(ds, h, B, seed)

    launches = steps(ctx, out, host, dev, net, "s16" if mode == "debug_keep" else None)
    out.update(pair_state(net, True))
    out["G_forward"] = net.G_forward(f32(rng.uniform(-1, 1, (B, 100))), training=True)
    out["G_backward.dnoise"] = net.G_backward(f32(rng.standard_normal((B, C, 16, 16)) * 1e-2), want_dnoise=True)
    for n in G_DEBUG_S16:
        out["debug." + n] = net.debug_tensor(n)
    out["D_forward"] = net.D_forward(f32(rng.random((B, C, 16, 16))), None, True, 3)
    out["D_backward.dimg"] = net.D_backward(f32(rng.standard_normal(B)), True, True)
    out["grads_G_after_calls"], out["grads_D_after_calls"] = net.get_grads(NET_G), net.get_grads(NET_D)
    ds.close()
    net.close()
    ctx.close()
    return out, launches


def case_c2f(B, imgs, S=32, mode="step", generator="create_G_d", discriminator="create_D_c", opts=None):
    import face_generator_b200 as fg
    from face_generator_b200 import layouts as LY
    from face_generator_b200.dataset import DeviceDataset, noise_uniform
    from face_generator_b200.lib import NET_D, NET_G
    rng = np.random.default_rng(51)
    cs = S // 2  # train_c2f.lua --coarseSize
    ctx = fg.Context(0, max_batch=B, channels=C)
    for k, v in (opts or {}).items():
        ctx.set_option(k, v)
    if mode == "debug_keep":
        ctx.set_option("debug_keep", 1)
    # the default pair through the two-argument form, which every build of C2f takes
    default = (generator, discriminator) == ("create_G_d", "create_D_c")
    net = fg.C2f(ctx, S) if default else fg.C2f(ctx, S, generator, discriminator)
    if generator == "create_G_d":
        net.set_params(NET_G, LY.trained_like_init(LY.c2f_G_layout(C), rng, 1.2))
    else:
        net.set_params(NET_G, f32(rng.standard_normal(net.count(NET_G)) * 0.02))
    if discriminator == "create_D_c":
        net.set_params(NET_D, LY.trained_like_init(LY.c2f_D_layout(C, S), rng, 1.0))
    else:
        net.set_params(NET_D, f32(rng.standard_normal(net.count(NET_D)) * 0.02))
    ds = DeviceDataset(ctx, imgs)
    h = fg.hyper_default()
    out = {}
    Bh = B // 2
    r = n_rows(mode)

    def inputs(seed):
        _, cr, dr = ds.gather_c2f(ds.draw(8 * seed, Bh), cs, S)
        _, cf, _ = ds.gather_c2f(ds.draw(8 * seed + 1, Bh), cs, S)
        _, cg, _ = ds.gather_c2f(ds.draw(8 * seed + 2, B), cs, S)
        nD, nG = noise_uniform(ctx, 8 * seed + 3, (Bh, 1, S, S)), noise_uniform(ctx, 8 * seed + 4, (B, 1, S, S))
        return dr, np.concatenate([cr, cf]), nD, cg, nG

    def host(seed):
        if not r:
            return net.train_step(h, B, *inputs(seed), None, None, seed)
        # the iterations' inputs stacked: any rows do, these are the single step's of seeds 1000 * seed + j
        x = [f32(np.stack(a)) for a in zip(*(inputs(1000 * seed + j) for j in range(ITERS)))]
        return net.train_step_iters(h, B, ITERS, ITERS, *x, None, None, seed)

    def dev(seed):
        if r:
            return net.train_step_dataset_iters(ds, h, B, ITERS, ITERS, cs, seed)
        return net.train_step_dataset(ds, h, B, cs, seed)

    launches = steps(ctx, out, host, dev, net, "c2f" if mode == "debug_keep" else None)
    out.update(pair_state(net, False))
    _, cond, diff = ds.gather_c2f(ds.draw(99, B), cs, S)
    out["G_forward"] = net.G_forward(f32(rng.uniform(-1, 1, (B, 1, S, S))), cond)
    net.G_backward(f32(rng.standard_normal((B, C, S, S)) * 1e-2))
    out["D_forward"] = net.D_forward(diff, cond, None, True, 3)
    out["D_backward.ddiff"] = net.D_backward(f32(rng.standard_normal(B)), True, True)
    out["grads_G_after_calls"], out["grads_D_after_calls"] = net.get_grads(NET_G), net.get_grads(NET_D)
    ds.close()
    net.close()
    ctx.close()
    return out, launches


def case_lop(N=16, Cin=128, H=16, Cout=128, k=3):
    """fg_conv2d_* with mma_f16 1 at a shape that takes the 3xFP16 tensor-core path"""
    import face_generator_b200 as fg
    from face_generator_b200.lib import _check, _ptr
    rng = np.random.default_rng(3)
    ctx = fg.Context(0, max_batch=N, channels=C)
    ctx.set_option("mma_f16", 1)
    lib, hd = ctx.lib, ctx.h
    x, w = f32(rng.standard_normal((N, Cin, H, H))), f32(rng.standard_normal((Cout, Cin, k, k)) * 0.05)
    b, dy = f32(rng.standard_normal(Cout)), f32(rng.standard_normal((N, Cout, H, H)) * 1e-3)
    y, dx = np.empty((N, Cout, H, H), np.float32), np.empty((N, Cin, H, H), np.float32)
    dw, db = np.zeros((Cout, Cin, k, k), np.float32), np.zeros(Cout, np.float32)
    l0 = ctx.launches()
    _check(lib.fg_conv2d_forward(hd, _ptr(x), _ptr(w), _ptr(b), _ptr(y), N, Cin, H, H, Cout, k), "fg_conv2d_forward")
    _check(lib.fg_conv2d_backward_data(hd, _ptr(dy), _ptr(w), _ptr(dx), N, Cin, H, H, Cout, k), "fg_conv2d_backward_data")
    _check(lib.fg_conv2d_backward_filter(hd, _ptr(x), _ptr(dy), _ptr(dw), _ptr(db), N, Cin, H, H, Cout, k),
           "fg_conv2d_backward_filter")
    launches = [ctx.launches() - l0]
    ctx.close()
    return {"y": y, "dx": dx, "dw": dw, "db": db}, launches


def toggled_steps(ctx, step):
    """6 seeded steps, the middle two with mma_f16 0: the weight packs are remade under each key"""
    launches, stats = [], []
    for i in range(6):
        if i in (2, 4):
            ctx.set_option("mma_f16", 0 if i == 2 else 1)
        l0 = ctx.launches()
        st = step(20 + i)
        ctx.sync()
        launches.append(ctx.launches() - l0)
        stats.append(np.array([st[k] for k in sorted(st)], np.float64))
    return launches, np.stack(stats)


def case_dn(B=128, S=16):
    import face_generator_b200 as fg
    from face_generator_b200 import denoiser as DN
    rng = np.random.default_rng(61)
    ctx = fg.Context(0, max_batch=B, channels=C)
    dn = DN.Denoiser(ctx, S)
    for net in (0, 1):
        dn.set_params(net, DN.init_params(C, S, rng))
    h = DN.dn_hyper_default()
    imgs = f32(rng.random((B, C, S, S)))
    launches, stats = toggled_steps(ctx, lambda seed: dn.train_step(h, imgs, seed=seed))
    m, v, t = dn.get_adam_state()
    out = {"stats": stats, "adam_m": m, "adam_v": v, "adam_t": np.array([t])}
    for net in (0, 1):
        out.update({"params_%d" % net: dn.get_params(net), "grads_%d" % net: dn.get_grads(net),
                    "bn_state_%d" % net: dn.get_bn_state(net), "forward_eval_%d" % net: dn.forward(net, imgs, False)})
    out["denoise"] = dn.denoise(f32(rng.random((B, C, S, S))))
    dn.close()
    ctx.close()
    return out, launches


def case_ae(B=128, S=32, d=256):
    import face_generator_b200 as fg
    from face_generator_b200 import autoencoder as AE
    rng = np.random.default_rng(71)
    ctx = fg.Context(0, max_batch=B, channels=1)
    ae = AE.Autoencoder(ctx, S, d)
    ae.set_params(AE.init_params(S, d, rng))
    h = AE.ae_hyper_default()
    imgs = f32(rng.random((B, 1, S, S)))
    launches, stats = toggled_steps(ctx, lambda seed: ae.train_step(h, imgs, seed=seed))
    m, v, t = ae.get_adam_state()
    code, y = ae.forward(imgs, training=False)
    out = {"stats": stats, "params": ae.get_params(), "grads": ae.get_grads(), "adam_m": m, "adam_v": v,
           "adam_t": np.array([t]), "forward_code": code, "forward_out": y,
           "reconstruct": ae.reconstruct(f32(rng.random((B, 1, S, S))))}
    ae.close()
    ctx.close()
    return out, launches


def free_after_create(B=256):
    """free device memory (bytes) right after fg_create(max_batch B, 3 channels), and before it"""
    import face_generator_b200 as fg
    import torch
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    ctx = fg.Context(0, max_batch=B, channels=C)
    ctx.sync()
    after = torch.cuda.mem_get_info()[0]
    ctx.close()
    return {"before": before, "after": after, "used_by_create": before - after}


def run(args):
    from face_generator_b200.lib import load_library
    load_library(os.path.abspath(args.lib))
    only = set(args.only.split(","))
    imgs = np.random.default_rng(50).integers(0, 256, (600, C, 64, 64), dtype=np.uint8)
    cases = []
    for B in (256, 130):
        if "32" in only:
            cases += [("32.B%d.%s" % (B, n), lambda B=B, o=o: case_32(B, o, imgs)) for n, o in OPTS_32]
        if "s16" in only:
            cases += [("s16.B%d.%s" % (B, n), lambda B=B, o=o: case_s16(B, o, imgs)) for n, o in OPTS_S16]
    for mode in ("iters2x2", "debug_keep"):
        if "32" in only:
            cases.append(("32.B256.%s" % mode, lambda m=mode: case_32(256, {}, imgs, m)))
        if "s16" in only:
            cases.append(("s16.B256.%s" % mode, lambda m=mode: case_s16(256, {}, imgs, m)))
        if "c2f" in only:
            cases.append(("c2f.B256.%s" % mode, lambda m=mode: case_c2f(256, imgs, 32, m)))
    if "dbr" in only:  # models.lua's other discriminators, on the 32x32 and the --scale 16 nets
        cases.append(("dbr.D32.B256", lambda: case_32(256, {}, imgs, discriminator="create_D32")))
        cases += [("dbr.%s.B256" % d[7:], lambda d=d: case_s16(256, {}, imgs, discriminator=d))
                  for d in ("create_D16", "create_D16_b", "create_D16_c")]
    if "c2f" in only:
        cases.append(("c2f.B256.default", lambda: case_c2f(256, imgs)))
        cases += [("c2f%d.B256.default" % S, lambda S=S: case_c2f(256, imgs, S)) for S in (16, 64)]
        cases += [("c2f%d.B%d.mma_f16=%d" % (S, B, f), lambda S=S, B=B, f=f: case_c2f(B, imgs, S, opts={"mma_f16": f}))
                  for S in (16, 32, 64) for B in (256, 130) for f in (1, 0)]
    if "c2fvar" in only:  # models_c2f.lua's other generators and discriminators (builds that have them)
        cases += [("c2fvar.%s.%s.S%d" % (g[7:], d[7:], S), lambda g=g, d=d, S=S: case_c2f(256, imgs, S, "step", g, d))
                  for g, d in (("create_G_a", "create_D_c"), ("create_G_b", "create_D_c"), ("create_G_c", "create_D_c"),
                               ("create_G_d", "create_D_a"), ("create_G_d", "create_D_b")) for S in (16, 32, 64)]
    if "lop" in only:
        cases.append(("lop.conv2d_f16", case_lop))
    if "dn" in only:
        cases.append(("dn.S16.B128", case_dn))
    if "ae" in only:
        cases.append(("ae.S32.B128", case_ae))
    os.makedirs(args.out, exist_ok=True)
    mem = free_after_create()
    with open(os.path.join(args.out, "free_after_create.json"), "w") as f:
        json.dump(mem, f)
    print("free memory after fg_create(256, 3): %s" % mem, flush=True)
    for name, fn in cases:
        out, launches = fn()
        d = os.path.join(args.out, name)
        os.makedirs(d, exist_ok=True)
        for k, a in out.items():
            np.save(os.path.join(d, k + ".npy"), a)
        with open(os.path.join(d, "launches.json"), "w") as f:
            json.dump(launches, f)
        print("%-28s %3d arrays  launches/step %s" % (name, len(out), launches), flush=True)


def compare(args):
    bad = 0
    for name in sorted(os.listdir(args.A)):
        if name.endswith(".json"):
            print("%-28s A %s  B %s" % (name, *(open(os.path.join(d, name)).read() for d in (args.A, args.B))))
            continue
        da, db = os.path.join(args.A, name), os.path.join(args.B, name)
        la, lb = (json.load(open(os.path.join(d, "launches.json"))) for d in (da, db))
        keys = sorted(f[:-4] for f in os.listdir(da) if f.endswith(".npy"))
        first = None
        for k in keys:
            pb = os.path.join(db, k + ".npy")
            a = np.load(os.path.join(da, k + ".npy"))
            if not os.path.exists(pb):
                first = "%s: missing in B" % k
                break
            b = np.load(pb)
            if a.dtype != b.dtype or a.shape != b.shape or a.tobytes() != b.tobytes():
                n = int(np.sum(a != b)) if a.shape == b.shape else -1
                first = "%s: %d elements differ" % (k, n)
                break
        bad += first is not None or la != lb
        print("%-28s %-34s launches/step A %s  B %s" % (name, first or "identical (%d arrays)" % len(keys), la, lb))
    print("%d case(s) differ" % bad)
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("--lib", required=True)
    r.add_argument("--out", required=True)
    r.add_argument("--only", default="32,s16,dbr,c2f,lop,dn,ae")
    c = sub.add_parser("compare")
    c.add_argument("A")
    c.add_argument("B")
    args = ap.parse_args()
    if args.cmd == "run":
        run(args)
        return 0
    return compare(args)


if __name__ == "__main__":
    sys.exit(main())
