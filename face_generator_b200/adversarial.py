"""Host-side mirror of adversarial.lua's loop body ("trainBatch", adversarial.lua:54-300).

train_batch()        the fused L-step call (fg_train_step): what adversarial_b200.lua uses.
train_batch_modules() the same iteration composed from the L-net calls exactly like the reference's
                     fevalD / fevalG_on_D closures -- used to show the two levels agree.
"""
import numpy as np

from .lib import Context
from .nn import BCECriterion, FusedD, FusedG, interruptableAdam


def create_noise_inputs(n, rng, noise_dim=100):
    """NN_UTILS.createNoiseInputs (utils/nn_utils.lua:35-39): U(-1,1)."""
    return rng.uniform(-1.0, 1.0, (n, noise_dim)).astype(np.float32)


def train_batch(ctx: Context, hyper, real, noise_D, noise_G, masks_D=None, masks_G=None, seed=0, want_stats=True):
    B = 2 * (real.shape[0] if hasattr(real, "shape") else 0) or None
    assert B is not None
    return ctx.train_step(hyper, B, real, noise_D, noise_G, masks_D, masks_G, seed, want_stats)


def train_batch_modules(ctx: Context, hyper, real, noise_D, noise_G, masks_D, masks_G):
    G, D, crit = FusedG(ctx), FusedD(ctx), BCECriterion(ctx)
    Bh = real.shape[0]
    B = 2 * Bh
    out = {}
    # ---- D step (adversarial.lua:240-268) ----
    samples = G.forward(noise_D)  # createImages: G in training mode
    inputs = np.concatenate([real, samples]).astype(np.float32)
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)]).astype(np.float32)

    def fevalD():
        D.zeroGradParameters()
        D.masks = masks_D
        outputs = D.forward(inputs)
        f = crit.forward(outputs, targets)
        D.backward(inputs, crit.backward(outputs, targets), want_wgrad=True)
        out["loss_D_bce"] = f
        out["outputs_D"] = outputs.copy()
        return f

    interruptableAdam(fevalD, D, hyper)
    out["grad_D"] = ctx.get_grads(D.net)
    # ---- G step (adversarial.lua:275-288) ----
    targets1 = np.ones(B, np.float32)

    def fevalG_on_D():
        G.zeroGradParameters()
        samples = G.forward(noise_G)
        D.masks = masks_G
        outputs = D.forward(samples)
        f = crit.forward(outputs, targets1)
        df_do = D.backward(samples, crit.backward(outputs, targets1), want_wgrad=False)
        G.backward(noise_G, df_do)
        out["loss_G"] = f
        return f

    interruptableAdam(fevalG_on_D, G, hyper)
    out["grad_G"] = ctx.get_grads(G.net)
    return out


def gate(accs, tV, max_acc, interval):
    """doTrainD of adversarial.lua:154-178: append this D iteration's accuracy tV to the history `accs` (a list, kept
    to the last `interval` entries, updated in place) and train D only while the history's mean is below max_acc."""
    accs.append(float(tV))
    if len(accs) > interval:
        accs.pop(0)
    return sum(accs) / len(accs) < max_acc


def train_batch_iters_modules(ctx: Context, hyper, reals, noises_D, noises_G, masks_D, masks_G, accs=None, hook=None):
    """train_batch_modules for len(reals) D iterations and len(noises_G) G iterations (train.lua --D_iterations /
    --G_iterations): the sequence fg_train_step_iters runs, composed from the L-net calls.  Every D iteration goes
    through the accuracy gate (`gate`, history `accs`); a closed gate skips that iteration's optimizer step.
    hook(kind, j, outputs) (optional) runs after D iteration j's backward ("D") / G iteration j's backward ("G"),
    before penalty, clamp and optimizer: the parameters are those the iteration ran on, the gradients are raw.
    Returns per-iteration accuracies, gate decisions and losses."""
    G, D, crit = FusedG(ctx), FusedD(ctx), BCECriterion(ctx)
    accs = [] if accs is None else accs
    Bh = reals[0].shape[0]
    B = 2 * Bh
    targets = np.concatenate([np.ones(Bh), np.zeros(Bh)]).astype(np.float32)
    targets1 = np.ones(B, np.float32)
    out = {"acc_D": [], "trained": [], "loss_D": [], "loss_G": []}
    for j in range(len(reals)):
        # ---- D iteration j (adversarial.lua:240-268) ----
        inputs = np.concatenate([reals[j], G.forward(noises_D[j])]).astype(np.float32)

        def fevalD():
            D.zeroGradParameters()
            D.masks = None if masks_D is None else masks_D[j]
            outputs = D.forward(inputs)
            f = crit.forward(outputs, targets)
            D.backward(inputs, crit.backward(outputs, targets), want_wgrad=True)
            if hook:
                hook("D", j, outputs)
            tV = float(np.mean((outputs.reshape(-1) > 0.5) == (targets > 0.5)))
            go = gate(accs, tV, hyper.D_maxAcc, max(1, hyper.accs_interval))
            out["acc_D"].append(tV)
            out["trained"].append(go)
            out["loss_D"].append(f)
            return f if go else False

        interruptableAdam(fevalD, D, hyper)
    for j in range(len(noises_G)):
        # ---- G iteration j (adversarial.lua:275-288) ----
        def fevalG_on_D():
            G.zeroGradParameters()
            samples = G.forward(noises_G[j])
            D.masks = None if masks_G is None else masks_G[j]
            outputs = D.forward(samples)
            f = crit.forward(outputs, targets1)
            df_do = D.backward(samples, crit.backward(outputs, targets1), want_wgrad=False)
            G.backward(noises_G[j], df_do)
            if hook:
                hook("G", j, outputs)
            out["loss_G"].append(f)
            return f

        interruptableAdam(fevalG_on_D, G, hyper)
    return out


# ------------------------------------------------------------------------------------------------------------------
# the epoch loop around the batch body (adversarial.lua:29-76, :232-334)
# ------------------------------------------------------------------------------------------------------------------
def epoch_batches(n_epoch, batch_size):
    """(t, thisBatchSize) pairs of one epoch exactly as adversarial.lua:54-76 walks them: t advances by the
    half-batch `dataBatchSize = batchSize / 2` (:35) -- each iteration consumes batchSize/2 *real* examples --
    the batch shrinks at the tail (:56) and the loop stops at the first batch smaller than 4 (:73-76).
    Odd tail sizes (possible when N_epoch or batchSize/2 is odd) are rounded down to even: the reference's own
    `realDataSize = thisBatchSize / 2` is fractional there (SURVEY.md appendix 13) and the fused step needs an even batch."""
    assert batch_size >= 4 and batch_size % 2 == 0
    out, t = [], 1
    while t <= n_epoch:
        this = min(batch_size, n_epoch - t + 1)
        if this < 4:
            break
        out.append((t, this - this % 2))
        t += batch_size // 2
    return out


SEED_EPOCH_STRIDE = 1000000   # the Lua shim's offset: seeds of epoch e start at (e-1)*1e6 (adversarial_b200.lua)
SEED_RANK_STRIDE = 1 << 40    # data parallel: every rank draws its own indices / noise / dropout masks


def epoch_seed0(epoch, rank=0):
    """first step seed of `epoch` (1-based, = the global EPOCH of train.lua:198-208) on `rank`"""
    assert epoch >= 1 and rank >= 0
    return (epoch - 1) * SEED_EPOCH_STRIDE + rank * SEED_RANK_STRIDE


def train(ctx, dataset, hyper, batch_size, n_epoch=-1, rng=None, epoch=1, rank=0, confusion=None, progress=None,
          D_iterations=1, G_iterations=1):
    """One epoch of adversarial.train(dataset, maxAccuracyD, accsInterval) (adversarial.lua:29-334): one fused call
    per batch.  D_iterations / G_iterations are train.lua --D_iterations / --G_iterations (:33-34, in [1, 16]): with
    both 1 a batch is one fg_train_step, otherwise one fg_train_step_iters, whose D iterations each draw their own
    real half-batch and noise and whose G iterations each draw their own noise (adversarial.lua:240-288).

    ctx: a Context (the 32x32 nets) or an S16 built on one (train.lua --scale 16: the 16x16 nets, images [N][C][16][16]).
    dataset: array-like [N][C][32][32] float32 in [0,1] (what DATASET.loadImages returns, dataset.lua:43-75) or a
    face_generator_b200.dataset.DeviceDataset (then batch assembly and noise happen on the device, at 16x16 through
    fg_s16_train_step_dataset when ctx is an S16).
    hyper.D_maxAcc / hyper.accs_interval are the maxAccuracyD / accsInterval arguments.
    epoch / rank: the reference draws fresh math.random indices and uniform noise on every call
    (adversarial.lua:245, :276), so successive epochs must not replay the same draws: the step seeds (device-side
    indices, noise and dropout masks derive from them) are epoch_seed0(epoch, rank) + i, and the host generator used
    for host-resident datasets is derived from (epoch, rank) unless the caller passes (and keeps) its own `rng`.
    Returns (accuracy of D over the epoch = CONFUSION.totalValid (:316), confusion counts [4], D iterations that
    trained D)."""
    from .dataset import DeviceDataset
    from .lib import S16, check_iters
    d_it, g_it = check_iters(D_iterations, G_iterations)
    multi = (d_it, g_it) != (1, 1)
    seed0 = epoch_seed0(epoch, rank)
    rng = rng if rng is not None else np.random.default_rng([int(epoch), int(rank), 0x6661636573])
    on_device = isinstance(dataset, DeviceDataset)
    N = dataset.size() if on_device else len(dataset)
    n_epoch = N if n_epoch <= 0 else n_epoch                                   # :31-34
    conf = np.zeros(4, np.int64) if confusion is None else confusion
    trained = 0
    for i, (t, B) in enumerate(epoch_batches(n_epoch, batch_size)):
        seed = seed0 + i + 1
        if on_device and multi:
            if isinstance(ctx, S16):
                st = ctx.train_step_dataset_iters(dataset, hyper, B, d_it, g_it, seed)
            else:
                st = dataset.train_step_iters(hyper, B, d_it, g_it, seed)
        elif on_device and isinstance(ctx, S16):
            st = ctx.train_step_dataset(dataset, hyper, B, seed)               # the 16x16 real half, on the device
        elif on_device:
            st = dataset.train_step(hyper, B, seed)
        elif multi:
            # in the reference's order: every D iteration its real half then its noise (:244-252), then the G noise
            reals, noises_D = [], []
            for _ in range(d_it):
                reals.append(np.asarray(dataset)[rng.integers(0, N, B // 2)])
                noises_D.append(create_noise_inputs(B // 2, rng))
            noises_G = [create_noise_inputs(B, rng) for _ in range(g_it)]
            st = ctx.train_step_iters(hyper, B, d_it, g_it, np.ascontiguousarray(np.stack(reals), np.float32),
                                      np.stack(noises_D), np.stack(noises_G), None, None, seed)
        else:
            real = np.ascontiguousarray(np.asarray(dataset)[rng.integers(0, N, B // 2)], np.float32)  # :244-249
            st = ctx.train_step(hyper, B, real, create_noise_inputs(B // 2, rng), create_noise_inputs(B, rng), None, None, seed)
        conf += np.asarray(st["conf"], np.int64)                               # :112-117
        trained += int(st["trained_D"])
        if progress:
            progress(t + B, n_epoch)                                           # xlua.progress (:296)
    total = conf.sum()
    return (float(conf[0] + conf[3]) / total if total else 0.0), conf, trained
