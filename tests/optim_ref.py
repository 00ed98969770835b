"""float64 restatement of the optimizer updates every parameter of every net goes through, for the tests: the
penalty and clamp of adversarial.lua, the interruptable optimizers (interruptable_optimizers.lua) and stock
optim.adam (adversarial_c2f.lua, train_denoiser.lua, train_autoencoder.lua), plus D's accuracy gate.

Every function works elementwise on numpy arrays or on torch tensors of the same dtype (the GPU tests run it in
float64 on the device, where the vectors have millions of elements).  Hyper-parameters are passed as the float32
values the library is handed (a Lua number multiplying a FloatTensor is rounded to float first), and everything is
evaluated in float64.  The optimizers return new arrays instead of updating in place."""
import math

import numpy as np


def _sqrt(a):
    return a.sqrt() if hasattr(a, "sqrt") else np.sqrt(a)


def _sign(a):
    """torch.sign: -1, 0 or 1; sign(0) = sign(-0) = 0"""
    return a.sign() if hasattr(a, "sign") else np.sign(a)


def _clamp(a, lo, hi):
    """Tensor:clamp(lo, hi) on the CPU (TH): NaN stays NaN"""
    return a.clamp(lo, hi) if hasattr(a, "clamp") else np.clip(a, lo, hi)


def f32(x):
    """the float32 value of a hyper-parameter, as float64"""
    return float(np.float32(x))


def penalty_terms(net_is_D, L1, L2):
    """(l1 weight, l2 weight) of the gradient penalty.  D: sign(P)*D_L1 + P*D_L2 (adversarial.lua:103-109).  G:
    sign(P)*G_L2 + P*G_L2 -- the L1 term is weighted by G_L2, not G_L1 (:218-224).  Off unless L1 or L2 is nonzero."""
    if L1 == 0 and L2 == 0:
        return 0.0, 0.0
    return (L1, L2) if net_is_D else (L2, L2)


def consumed_grad(g, p, scale=1.0, l1=0.0, l2=0.0, clamp=0.0):
    """the gradient the optimizer step consumes: the data-parallel scale first, then the penalty
    (adversarial.lua:108, :223), then the clamp (:121-123, :226-228; clamp 0 = off)"""
    g = g * f32(scale)
    if l1 != 0 or l2 != 0:
        g = g + (_sign(p) * f32(l1) + p * f32(l2))
    if clamp != 0:
        g = _clamp(g, -f32(clamp), f32(clamp))
    return g


def adam_step_size(lr, beta1, beta2, t):
    """stepSize = lr * sqrt(1 - beta2^t) / (1 - beta1^t) at the incremented t (interruptable_optimizers.lua:78,
    :86-88; optim.adam the same)"""
    b1, b2 = f32(beta1), f32(beta2)
    return f32(lr) * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)


def adam(x, g, m, v, t, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    """interruptableAdam (interruptable_optimizers.lua:69-90) and optim.adam (identical update): one step from state
    (m, v, t) with gradient g.  Returns (x, m, v, t)."""
    b1, b2 = f32(beta1), f32(beta2)
    t = t + 1                                                       # :78
    m = m * b1 + (1 - b1) * g                                       # :81
    v = v * b2 + (1 - b2) * g * g                                   # :82
    return adam_param(x, m, v, t, lr, beta1, beta2, eps), m, v, t


def adam_param(x, m, v, t, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
    """the parameter update of Adam step t from the updated moments m, v (interruptable_optimizers.lua:84-90)"""
    denom = _sqrt(v) + f32(eps)                                     # :84
    return x - adam_step_size(lr, beta1, beta2, t) * m / denom      # :86-90


def adagrad(x, g, var, t, lr=1e-3):
    """interruptableAdagrad (interruptable_optimizers.lua:7-46) with learningRateDecay 0 (train.lua never sets it):
    paramVariance += g^2; x -= lr * g / (sqrt(paramVariance) + 1e-10); evalCounter += 1.  Returns (x, var, t)."""
    var = var + g * g                                               # :37
    return adagrad_param(x, g, var, lr), var, t + 1


def adagrad_param(x, g, var, lr=1e-3):
    """the parameter update of Adagrad from the updated variance (interruptable_optimizers.lua:38-39)"""
    return x - f32(lr) * g / (_sqrt(var) + f32(1e-10))


def sgd(x, g, buf, t, lr=0.02, mom=0.0):
    """interruptableSgd (interruptable_optimizers.lua:97-167) with the options train.lua sets (learningRate, momentum;
    dampening defaults to the momentum, :105).  With momentum the first evaluation (evalCounter 0 before the call:
    no state.dfdx yet) clones the gradient into the buffer (:136-137); later ones blend it,
    buf = buf*mom + (1 - mom)*g (:139).  Without momentum the buffer is untouched.  Returns (x, buf, t)."""
    if mom != 0:
        mo = f32(mom)
        buf = g * 1.0 if t == 0 else buf * mo + (1 - mo) * g
        g = buf
    x = x - f32(lr) * g                                             # :159
    return x, buf, t + 1


def accuracy_gate(accs, tV, interval, max_acc):
    """adversarial.lua:156-178: append this batch's accuracy to D's history, keep the last `interval` entries and
    train D only while their mean is below maxAccuracyD.  Returns (new history, doTrainD)."""
    accs = list(accs) + [tV]
    if len(accs) > interval:
        accs.pop(0)
    return accs, (sum(accs) / len(accs)) < max_acc
