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


def train(ctx, dataset, hyper, batch_size, n_epoch=-1, rng=None, epoch=1, rank=0, confusion=None, progress=None):
    """One epoch of adversarial.train(dataset, maxAccuracyD, accsInterval) (adversarial.lua:29-334) with the
    defaults D_iterations = G_iterations = 1 (train.lua:33-34), i.e. one fused fg_train_step per batch.

    ctx: a Context (the 32x32 nets) or an S16 built on one (train.lua --scale 16: the 16x16 nets, images [N][C][16][16]).
    dataset: array-like [N][C][32][32] float32 in [0,1] (what DATASET.loadImages returns, dataset.lua:43-75) or a
    face_generator_b200.dataset.DeviceDataset (then batch assembly and noise happen on the device, at 16x16 through
    fg_s16_train_step_dataset when ctx is an S16).
    hyper.D_maxAcc / hyper.accs_interval are the maxAccuracyD / accsInterval arguments.
    epoch / rank: the reference draws fresh math.random indices and uniform noise on every call
    (adversarial.lua:245, :276), so successive epochs must not replay the same draws: the step seeds (device-side
    indices, noise and dropout masks derive from them) are epoch_seed0(epoch, rank) + i, and the host generator used
    for host-resident datasets is derived from (epoch, rank) unless the caller passes (and keeps) its own `rng`.
    Returns (accuracy of D over the epoch = CONFUSION.totalValid (:316), confusion counts [4], batches that trained D)."""
    from .dataset import DeviceDataset
    from .lib import S16
    seed0 = epoch_seed0(epoch, rank)
    rng = rng if rng is not None else np.random.default_rng([int(epoch), int(rank), 0x6661636573])
    on_device = isinstance(dataset, DeviceDataset)
    N = dataset.size() if on_device else len(dataset)
    n_epoch = N if n_epoch <= 0 else n_epoch                                   # :31-34
    conf = np.zeros(4, np.int64) if confusion is None else confusion
    trained = 0
    for i, (t, B) in enumerate(epoch_batches(n_epoch, batch_size)):
        seed = seed0 + i + 1
        if on_device and isinstance(ctx, S16):
            st = ctx.train_step_dataset(dataset, hyper, B, seed)               # the 16x16 real half, on the device
        elif on_device:
            st = dataset.train_step(hyper, B, seed)
        else:
            real = np.ascontiguousarray(np.asarray(dataset)[rng.integers(0, N, B // 2)], np.float32)  # :244-249
            st = ctx.train_step(hyper, B, real, create_noise_inputs(B // 2, rng), create_noise_inputs(B, rng), None, None, seed)
        conf += np.asarray(st["conf"], np.int64)                               # :112-117
        trained += int(st["trained_D"])
        if progress:
            progress(t + B, n_epoch)                                           # xlua.progress (:296)
    total = conf.sum()
    return (float(conf[0] + conf[3]) / total if total else 0.0), conf, trained
