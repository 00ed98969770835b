"""Float64 restatement of nn.SpatialBatchNormalization (models.lua:65,70) composed with the shared-slope nn.PReLU
that follows it in G, in training and evaluate mode.

Torch's BatchNorm (THNN SpatialBatchNormalization) takes the batch mean first and then the mean squared deviation
from it (two passes), so a channel whose mean is large against its spread loses nothing to cancellation.  This module
does the same in float64, which makes it the yardstick for the CUDA statistics paths (tests/test_gpu_batchnorm.py).

Tensors are torch float64, NCHW (any number of trailing spatial dimensions); per-channel vectors have shape [C].
tests/test_bn_ref_cpu.py pins every function here to PyTorch autograd and to the C++ oracle."""
import torch

EPS = 1e-5
MOMENTUM = 0.1


def _cv(v, like):
    """per-channel vector [C] -> broadcastable against an NC... tensor"""
    return v.reshape((1, -1) + (1,) * (like.dim() - 2))


def _dims(z):
    return [0] + list(range(2, z.dim()))


def batch_stats(z):
    """two-pass batch mean and biased variance per channel"""
    mean = z.mean(dim=_dims(z))
    var = ((z - _cv(mean, z)) ** 2).mean(dim=_dims(z))
    return mean, var


def count(z):
    return z.numel() // z.shape[1]


def running_update(rm, rv, mean, var, n):
    """THNN's running statistics: momentum 0.1, the unbiased variance var * n / (n - 1)"""
    return (1 - MOMENTUM) * rm + MOMENTUM * mean, (1 - MOMENTUM) * rv + MOMENTUM * var * (n / (n - 1))


def prelu(u, slope, pos=None):
    """shared-slope PReLU; pos: the branch taken (u > 0 unless given, see kink_pos)"""
    if slope is None:
        return u
    return torch.where(u > 0 if pos is None else pos, u, slope * u)


def kink_pos(u, gpu_pos, margin, max_frac=2e-3):
    """branch decisions: u > 0, except where |u| < margin * max|u| (a pre-activation within rounding noise of PReLU's
    kink), where the CUDA path's own decision gpu_pos is taken.  Asserts that such elements are rare."""
    amb = u.abs() < margin * u.abs().max()
    assert int(amb.sum()) <= max(8, max_frac * u.numel()), (int(amb.sum()), u.numel())
    return torch.where(amb, gpu_pos, u > 0)


def forward_train(z, gamma, beta, slope=None, mean=None, pos=None):
    """training-mode forward.  mean: an externally supplied batch mean used for x_hat = (z - mean) * istd (the
    variance still comes from the data), so a test can leave the rounding of the mean under test out of the output.
    Returns dict(u = BN output, h = PReLU(u), mean, var, istd, xhat) with mean = the batch mean."""
    bm, var = batch_stats(z)
    istd = 1.0 / torch.sqrt(var + EPS)
    m = bm if mean is None else mean
    xhat = (z - _cv(m, z)) * _cv(istd, z)
    u = _cv(gamma, z) * xhat + _cv(beta, z)
    return dict(u=u, h=prelu(u, slope, pos), mean=bm, var=var, istd=istd, xhat=xhat)


def forward_eval(z, gamma, beta, rm, rv, slope=None):
    """evaluate-mode forward: the running statistics in place of the batch's"""
    u = _cv(gamma, z) * (z - _cv(rm, z)) / torch.sqrt(_cv(rv, z) + EPS) + _cv(beta, z)
    return prelu(u, slope)


def backward(z, gamma, beta, mean, istd, dh, slope=None, pos=None):
    """backward of PReLU(BN(z)) given the forward's mean and istd.  Returns (dz, dgamma, dbeta, dslope):
      u = gamma * xhat + beta,  g = dh * (u > 0 ? 1 : slope),  dslope = sum_{u <= 0} dh * u,
      dz = gamma * istd * (g - mean(g) - xhat * mean(g * xhat)),  dgamma = sum g * xhat,  dbeta = sum g."""
    d = _dims(z)
    xhat = (z - _cv(mean, z)) * _cv(istd, z)
    u = _cv(gamma, z) * xhat + _cv(beta, z)
    dslope = None
    g = dh
    if slope is not None:
        p = u > 0 if pos is None else pos
        g = torch.where(p, dh, slope * dh)
        dslope = torch.where(p, torch.zeros_like(u), dh * u).sum()
    dbeta, dgamma = g.sum(dim=d), (g * xhat).sum(dim=d)
    n = count(z)
    dz = _cv(gamma * istd, z) * (g - _cv(dbeta / n, z) - xhat * _cv(dgamma / n, z))
    return dz, dgamma, dbeta, dslope
