"""Independent (test-only) PyTorch fp64 restatement of the --scale 16 nets (models.lua:27-51
create_G_decoder_upsampling16, :279-316 create_D16_d).  tests/test_oracle_s16_vs_torch.py pins it to the C++ oracle on
the CPU; tests/test_gpu_c2f_s16_headline.py holds the CUDA path to it on the GPU at the BASELINE batch size.

branch: the PReLU branch hook of torch_ref.prelu, called with the names "z0", "y1", "y2" (G: Linear output, the two
BatchNorm outputs) and "z1".."z4", "zf", "ze1", "ze2" (D: the four convolutions, the conv branch's Linear, the dense
branch's two Linears)."""
import torch
import torch.nn.functional as F

from oracle import oracle_s16 as OS
from torch_ref import _split, d_sigmoid, prelu


def torch_G16(P, noise, C, branch=None, running=None):
    """running: the BatchNorm running statistics [mean1 256][var1 256][mean2 128][var2 128] (fg_s16_get_bn_state
    layout), updated in place as a training-mode forward of nn.SpatialBatchNormalization does (momentum 0.1, unbiased
    variance)"""
    p = _split(P, OS.G_layout(C))
    B = noise.shape[0]
    rs = (None,) * 4 if running is None else (running[0:256], running[256:512], running[512:640], running[640:768])
    h = prelu(F.linear(noise, p["L1W"], p["L1b"]).view(B, 128, 4, 4), p["a1"], branch, "z0")
    h = F.conv2d(F.interpolate(h, scale_factor=2, mode="nearest"), p["C1W"], p["C1b"], padding=2)
    h = prelu(F.batch_norm(h, rs[0], rs[1], p["g1"], p["be1"], training=True, momentum=0.1, eps=1e-5), p["a2"], branch, "y1")
    h = F.conv2d(F.interpolate(h, scale_factor=2, mode="nearest"), p["C2W"], p["C2b"], padding=2)
    h = prelu(F.batch_norm(h, rs[2], rs[3], p["g2"], p["be2"], training=True, momentum=0.1, eps=1e-5), p["a3"], branch, "y2")
    return torch.sigmoid(F.conv2d(h, p["C3W"], p["C3b"], padding=1))


def torch_D16(P, img, masks, C, branch=None):
    p = _split(P, OS.D_layout(C))
    B = img.shape[0]
    h = prelu(F.conv2d(img, p["c1W"], p["c1b"], padding=1), p["a1"], branch, "z1")
    h = prelu(F.conv2d(h, p["c2W"], p["c2b"], padding=1), p["a2"], branch, "z2")
    h = F.avg_pool2d(h, 2, 2)
    h = prelu(F.conv2d(h, p["c3W"], p["c3b"], stride=2, padding=1), p["a3"], branch, "z3")
    h = prelu(F.conv2d(h, p["c4W"], p["c4b"], stride=2, padding=1), p["a4"], branch, "z4")
    h = h * masks[:, :1024].reshape(B, 1024, 1, 1)  # SpatialDropout: no rescale
    fine = prelu(F.linear(h.reshape(B, 4096), p["F1W"], p["F1b"]), p["af"], branch, "zf")
    e = prelu(F.linear(img.reshape(B, -1), p["E1W"], p["E1b"]), p["ae1"], branch, "ze1") * masks[:, 1024:] * 2.0
    e = prelu(F.linear(e, p["E2W"], p["E2b"]), p["ae2"], branch, "ze2")
    return d_sigmoid(F.linear(torch.cat([fine, e], dim=1), p["JW"], p["Jb"])).reshape(B)
