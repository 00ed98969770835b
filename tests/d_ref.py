"""Float64 restatement of the 32x32 discriminator (models.lua:382-416) one kernel launch at a time, in the library's
own layouts, as the yardstick of tests/test_gpu_d_launches.py.

Layouts are the ones the CUDA path stores (and fg_debug_tensor returns):
  * activations NHWC: z_i [B][H][H][C], p_i [B][H/2][H/2][C]; the linear layers [B][512];
  * dropout keep flags [B][1984] per sample: the SpatialDropout flags of D.C1..C4 at MOFF = 0, 64, 192, 448, then the
    nn.Dropout flags of D.L1 at 960 and of D.L2 at 1472 (512 each);
  * D.L1 reads p4 through View(2048), which flattens [512][2][2] in (c, h, w) order: view2048 states that permutation
    of the NHWC tensor.

Every reduction also returns its condition: the sum of the absolute values of the summed terms, so that a checker
can hold a cancelling sum to |got - ref| <= tol * cond rather than to its own small value.  PReLU takes the slope
branch at z == 0 exactly (the kernels' `z > 0` rule).  tests/test_d_ref_cpu.py chains these functions into the whole
D and pins them to the C++ oracle.  Tensors are torch float64 on any device."""
import torch

MOFF = (0, 64, 192, 448)
MOFF_L1, MOFF_L2 = 960, 1472
COUT = (64, 128, 256, 512)
HW = (32, 16, 8, 4)
P_SPATIAL, P_DROP = 0.2, 0.5
BCE_EPS = 1e-12


def _flags(masks, moff, C, eval_scale):
    """[B][1][1][C] SpatialDropout factor: the keep flags in training, 1 - p_spatial in evaluate mode (masks None)"""
    if masks is None:
        return torch.tensor(eval_scale, dtype=torch.float64)
    return masks[:, moff:moff + C].reshape(-1, 1, 1, C)


def prelu(z, slope):
    return torch.where(z > 0, z, slope * z)


# ---- PReLU -> SpatialDropout (no rescale) -> SpatialAveragePooling(2, 2) (d_act_pool_fwd / _bwd) -------------------
def act_pool_fwd(z, slope, masks, moff, eval_scale=1 - P_SPATIAL):
    B, H, W, C = z.shape
    d = prelu(z, slope) * _flags(masks, moff, C, eval_scale)
    return d.reshape(B, H // 2, 2, W // 2, 2, C).mean(dim=(2, 4))


def act_pool_bwd(dp, z, slope, masks, moff, eval_scale=1 - P_SPATIAL):
    """dp [B][H/2][W/2][C] -> dict(dz, dslope, dslope_cond, dbias [C], dbias_cond [C]); dbias = column sums of dz (the
    gradient of the convolution bias in front)"""
    B, H, W, C = z.shape
    g = dp.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) * 0.25 * _flags(masks, moff, C, eval_scale)
    pos = z > 0
    dz = torch.where(pos, g, slope * g)
    t = torch.where(pos, torch.zeros_like(g), g * z)
    return dict(dz=dz, dslope=t.sum(), dslope_cond=t.abs().sum(), dbias=dz.sum(dim=(0, 1, 2)),
                dbias_cond=dz.abs().sum(dim=(0, 1, 2)))


# ---- PReLU -> nn.Dropout(p) (lin_act_drop_fwd / _bwd): kept / (1 - p) in training, identity in evaluate mode --------
def _drop(masks, moff, N, scale):
    if masks is None:
        return torch.tensor(1.0, dtype=torch.float64)
    return masks[:, moff:moff + N] * scale


def lin_act_drop_fwd(z, slope, masks, moff, scale=1 / (1 - P_DROP)):
    return prelu(z, slope) * _drop(masks, moff, z.shape[1], scale)


def lin_act_drop_bwd(dh, z, slope, masks, moff, scale=1 / (1 - P_DROP)):
    """-> dict(dz, dslope, dslope_cond)"""
    g = dh * _drop(masks, moff, z.shape[1], scale)
    pos = z > 0
    t = torch.where(pos, torch.zeros_like(g), g * z)
    return dict(dz=torch.where(pos, g, slope * g), dslope=t.sum(), dslope_cond=t.abs().sum())


# ---- the 3x3 "same" convolutions D.C1..C4 on NHWC tensors (W [Cout][Cin][3][3], Torch's layout) --------------------
def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def conv_fwd(x, W, b):
    return _nhwc(torch.nn.functional.conv2d(_nchw(x), W, b, padding=1))


def conv_dgrad(x_shape, W, dz):
    B, H, Wd, C = x_shape
    return _nhwc(torch.nn.grad.conv2d_input((B, C, H, Wd), W, _nchw(dz), padding=1))


def conv_wgrad(x, W_shape, dz):
    return torch.nn.grad.conv2d_weight(_nchw(x), W_shape, _nchw(dz), padding=1)


# ---- View(2048) of D.L1 ---------------------------------------------------------------------------------------------
def view2048(p4):
    """NHWC [B][2][2][512] -> the [B][2048] row Torch's View(2048) makes of [512][2][2]: column c * 4 + h * 2 + w"""
    return p4.reshape(-1, 2, 2, 512).permute(0, 3, 1, 2).reshape(-1, 2048)


def view2048_bwd(dx):
    """[B][2048] gradient in View(2048) order -> NHWC [B][2][2][512]"""
    return dx.reshape(-1, 512, 2, 2).permute(0, 2, 3, 1).contiguous()


# ---- nn.Linear(512, 1) = D.L3 (gemv_fwd / _dgrad / _wgrad) ----------------------------------------------------------
def gemv_fwd(h, w, b):
    """h [B][K], w [K], b [1] -> logit [B]"""
    return h @ w + b


def gemv_dgrad(dlogit, w):
    return dlogit[:, None] * w[None, :]


def gemv_wgrad(h, dlogit):
    """-> dict(dw [K], dw_cond [K], db, db_cond)"""
    return dict(dw=h.t() @ dlogit, dw_cond=h.abs().t() @ dlogit.abs(), db=dlogit.sum(), db_cond=dlogit.abs().sum())


# ---- nn.Sigmoid + nn.BCECriterion (sigmoid_bce) -----------------------------------------------------------------------
def sigmoid_out(logit):
    """D's output as the library stores it: float32 (a saturated output is exactly 0 or 1)"""
    return torch.sigmoid(logit).to(torch.float32).to(torch.float64)


def sigmoid_bce(logit, n_ones, y=None):
    """The loss step of one D pass: targets 1 for the first n_ones samples, 0 after; y: the stored sigmoid output
    (sigmoid_out(logit) unless given).  The 2015 Lua BCE (eps 1e-12, size-averaged) and its gradient composed with
    the sigmoid's.  conf = [target 1 & predicted 1, target 1 & predicted 0, target 0 & predicted 1, target 0 &
    predicted 0] with "predicted 1" = y > 0.5 (adversarial.lua:114): exactly 0.5 is predicted 0.
    -> dict(y, loss, loss_cond, dlogit, conf)"""
    if y is None:
        y = sigmoid_out(logit)
    B = y.shape[0]
    t = (torch.arange(B, device=y.device) < n_ones).to(torch.float64)
    terms = t * torch.log(y + BCE_EPS) + (1 - t) * torch.log(1 - y + BCE_EPS)
    grad = -(t - y) / (y * (1 - y + BCE_EPS) + BCE_EPS) / B
    p1, t1 = y > 0.5, t > 0.5
    conf = [int((t1 & p1).sum()), int((t1 & ~p1).sum()), int((~t1 & p1).sum()), int((~t1 & ~p1).sum())]
    return dict(y=y, loss=-terms.sum() / B, loss_cond=terms.abs().sum() / B, dlogit=grad * y * (1 - y), conf=conf)


def sigmoid_grad(dout, y):
    """fg_D_backward's dlogit from a given output gradient and the stored output"""
    return dout * y * (1 - y)
