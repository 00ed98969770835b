"""float64 restatement of models.lua's branched discriminators create_D32, create_D16, create_D16_b and create_D16_c.

Each net is built from a flat getParameters() vector P (module order through the ConcatTable) and per-sample keep
flags in module order.  The modules have hand-written backward passes (Torch7's updateGradInput / accGradParameters);
the forward is plain torch, so torch.autograd on the same graph checks them.  Images are NCHW.
"""
import numpy as np
import torch
import torch.nn.functional as F

P_DROP = 0.5
DENSE = ("dense", [], [(1024, True), (1024, False)])
# name -> (side, [(branch, [(Cout, k, stride, maxpool after the PReLU)], [(Linear out, Dropout after the PReLU)])],
#          (head Linear out, head Dropout)); every conv and Linear is followed by a PReLU, a conv branch ends in
#          SpatialDropout + View, the head is JoinTable(2) Linear PReLU Dropout Linear(1) Sigmoid  (models.lua)
NETS = {
    "create_D32": (32, [("fine", [(64, 3, 1, False), (64, 3, 1, True)], [(1024, False)]),
                        ("coarse", [(32, 5, 1, False), (32, 5, 1, True), (54, 5, 1, False), (54, 5, 1, True)],
                         [(1024, True), (1024, False)]),
                        DENSE], (1024, True)),
    "create_D16": (16, [("fine", [(64, 3, 1, False), (64, 3, 1, True)], [(1024, True)]),
                        ("coarse", [(32, 5, 1, False), (64, 5, 1, True)], [(1024, True)]),
                        DENSE], (1024, True)),
    "create_D16_b": (16, [("fine", [(64, 3, 1, False), (64, 3, 1, False), (128, 3, 1, False), (128, 3, 2, False)],
                           [(512, True)]),
                          ("coarse", [(64, 5, 1, False), (64, 5, 1, False), (128, 5, 1, False), (128, 5, 2, False)],
                           [(512, True)]),
                          DENSE], (1024, True)),
    "create_D16_c": (16, [("fine", [(64, 3, 1, False), (64, 3, 1, False), (128, 3, 1, False), (128, 3, 2, False),
                                    (512, 3, 2, False)], [(1024, False)]),
                          ("coarse", [(64, 5, 1, False), (64, 5, 1, False), (128, 5, 1, False), (128, 5, 2, False),
                                      (512, 5, 2, False)], [(1024, False)]),
                          DENSE], (1024, True)),
}


class Ctx:
    """one pass: parameters P, gradient accumulator gP, keep flags [B][mask] (training) or None (evaluate), route hook"""

    def __init__(self, P, keep, route=None):
        self.P, self.keep, self.route = P, keep, route
        self.gP = torch.zeros_like(P.detach())
        self.gabs = {}  # slope offset -> sum of |dY * z| over its terms: the scale of a slope gradient's rounding

    def p(self, off, shape):
        n = int(np.prod(shape))
        return self.P[off:off + n].reshape(shape)

    def acc(self, off, g):
        self.gP[off:off + g.numel()] += g.reshape(-1)


class Conv:
    def __init__(self, off, cin, cout, k, stride):
        self.off, self.cin, self.cout, self.k, self.stride = off, cin, cout, k, stride
        self.n = cout * cin * k * k + cout

    def fwd(self, c, x):
        self.x = x
        W, b = c.p(self.off, (self.cout, self.cin, self.k, self.k)), c.p(self.off + self.n - self.cout, (self.cout,))
        return F.conv2d(x, W, b, self.stride, (self.k - 1) // 2)

    def bwd(self, c, dy):
        W = c.p(self.off, (self.cout, self.cin, self.k, self.k)).detach()
        pad = (self.k - 1) // 2
        x = self.x.detach()
        c.acc(self.off, torch.nn.grad.conv2d_weight(x, W.shape, dy, self.stride, pad))
        c.acc(self.off + self.n - self.cout, dy.sum((0, 2, 3)))
        return torch.nn.grad.conv2d_input(x.shape, W, dy, self.stride, pad)


class Linear:
    def __init__(self, off, fin, fout):
        self.off, self.fin, self.fout = off, fin, fout
        self.n = fout * fin + fout

    def fwd(self, c, x):
        self.x = x
        return x @ c.p(self.off, (self.fout, self.fin)).t() + c.p(self.off + self.fout * self.fin, (self.fout,))

    def bwd(self, c, dy):
        c.acc(self.off, dy.t() @ self.x.detach())
        c.acc(self.off + self.fout * self.fin, dy.sum(0))
        return dy @ c.p(self.off, (self.fout, self.fin)).detach()


class PReLU:
    def __init__(self, off):
        self.off, self.n = off, 1

    def fwd(self, c, x):
        self.x = x
        return torch.where(x > 0, x, c.P[self.off] * x)

    def bwd(self, c, dy):
        x, a = self.x.detach(), c.P[self.off].detach()
        c.acc(self.off, (dy * x)[x <= 0].sum().reshape(1))
        c.gabs[self.off] = c.gabs.get(self.off, 0.0) + float((dy * x)[x <= 0].abs().sum())
        return torch.where(x > 0, dy, a * dy)


def first_max(win):
    """win [..., 4] in row-major window order -> index of the first strict maximum (THNN SpatialMaxPooling)"""
    idx = torch.zeros(win.shape[:-1], dtype=torch.long)
    best = win[..., 0].clone()
    for j in range(1, 4):
        take = win[..., j] > best
        idx[take] = j
        best = torch.where(take, win[..., j], best)
    return idx


class MaxPool:
    """nn.SpatialMaxPooling(2, 2); route(name, win) may replace the arg-max of some windows (win [B][C][H/2][W/2][4])"""

    def __init__(self, name):
        self.name, self.n = name, 0

    @staticmethod
    def windows(x):
        B, C, H, W = x.shape
        return x.reshape(B, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H // 2, W // 2, 4)

    def fwd(self, c, x):
        self.shape = x.shape
        win = self.windows(x)
        idx = first_max(win.detach())
        if c.route is not None:
            idx = c.route(self.name, win.detach(), idx)
        self.idx = idx
        return torch.gather(win, 4, idx.unsqueeze(-1)).squeeze(-1)

    def bwd(self, c, dy):
        B, C, H, W = self.shape
        win = torch.zeros(B, C, H // 2, W // 2, 4, dtype=dy.dtype)
        win.scatter_(4, self.idx.unsqueeze(-1), dy.unsqueeze(-1))
        return win.reshape(B, C, H // 2, W // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H, W)


class Dropout:
    """nn.SpatialDropout() (spatial: one flag per plane, no rescale, 1-p in evaluate) or nn.Dropout() (1/(1-p) in
    training, identity in evaluate); flags keep[:, moff:moff+width]"""

    def __init__(self, moff, width, spatial):
        self.moff, self.width, self.spatial, self.n = moff, width, spatial, 0

    def mul(self, c, x):
        if c.keep is None:
            return (1 - P_DROP) if self.spatial else 1.0
        k = c.keep[:, self.moff:self.moff + self.width]
        return k[:, :, None, None] if self.spatial else k / (1 - P_DROP)

    def fwd(self, c, x):
        return x * self.mul(c, x)

    def bwd(self, c, dy):
        return dy * self.mul(c, dy)


class View:
    n = 0

    def fwd(self, c, x):
        self.shape = x.shape
        return x.reshape(x.shape[0], -1)

    def bwd(self, c, dy):
        return dy.reshape(self.shape)


class Net:
    """one discriminator at C channels: branches (lists of modules), head modules, flat size, keep flags per sample"""

    def __init__(self, name, C):
        side, branches, (hout, hdrop) = NETS[name]
        self.name, self.C, self.side = name, C, side
        off, moff = 0, 0
        self.branches = []
        for bname, convs, lins in branches:
            mods, cin, s = [], C, side
            for i, (cout, k, stride, pool) in enumerate(convs):
                mods.append(Conv(off, cin, cout, k, stride)); off += mods[-1].n
                mods.append(PReLU(off)); off += 1
                s //= stride
                if pool:
                    mods.append(MaxPool("%s.%d" % (bname, i + 1)))
                    s //= 2
                cin = cout
            if convs:
                mods.append(Dropout(moff, cin, True)); moff += cin
            mods.append(View())
            fin = cin * s * s
            for fout, drop in lins:
                mods.append(Linear(off, fin, fout)); off += mods[-1].n
                mods.append(PReLU(off)); off += 1
                if drop:
                    mods.append(Dropout(moff, fout, False)); moff += fout
                fin = fout
            self.branches.append((bname, mods, fin))
        self.joint = sum(b[2] for b in self.branches)
        self.head = [Linear(off, self.joint, hout)]; off += self.head[-1].n
        self.head.append(PReLU(off)); off += 1
        if hdrop:
            self.head.append(Dropout(moff, hout, False)); moff += hout
        self.head.append(Linear(off, hout, 1)); off += self.head[-1].n
        self.n_params, self.mask = off, moff

    def forward(self, c, x):
        """x [B][C][S][S] -> logit [B]"""
        outs = []
        for _, mods, _ in self.branches:
            h = x
            for m in mods:
                h = m.fwd(c, h)
            outs.append(h)
        h = torch.cat(outs, 1)
        for m in self.head:
            h = m.fwd(c, h)
        return h[:, 0]

    def backward(self, c, dlogit):
        """after forward: dlogit [B] -> dx [B][C][S][S]; parameter gradients into c.gP"""
        d = dlogit[:, None]
        for m in reversed(self.head):
            d = m.bwd(c, d)
        dx, o = None, 0
        for _, mods, w in self.branches:
            g = d[:, o:o + w]
            o += w
            for m in reversed(mods):
                g = m.bwd(c, g)
            dx = g if dx is None else dx + g  # nn.ConcatTable: the branches' input gradients, summed in order
        return dx

    def param_tensors(self):
        """(name, offset, size) of every parameter tensor in getParameters() order"""
        out = []
        for bname, mods, _ in self.branches + [("head", self.head, 0)]:
            for i, m in enumerate(mods):
                if isinstance(m, Conv):
                    out += [("%s.%d.W" % (bname, i), m.off, m.n - m.cout), ("%s.%d.b" % (bname, i), m.off + m.n - m.cout, m.cout)]
                elif isinstance(m, Linear):
                    out += [("%s.%d.W" % (bname, i), m.off, m.fin * m.fout), ("%s.%d.b" % (bname, i), m.off + m.fin * m.fout, m.fout)]
                elif isinstance(m, PReLU):
                    out.append(("%s.%d.a" % (bname, i), m.off, 1))
        return out


def make_params(net, seed, near=True):
    """weights ~ U(-1/sqrt(fan_in), 1/sqrt(fan_in)); PReLU slopes 1 - k*1e-3 ("near": a flipped z <= 0 branch moves a
    gradient by ~1e-3 of one element, far below the 1e-4 normwise bar, where 0.25 would not be) or 0.25"""
    rng = np.random.default_rng(seed)
    P = np.zeros(net.n_params, np.float64)
    k = 0
    for _, mods, _ in net.branches + [("head", net.head, 0)]:
        for m in mods:
            if isinstance(m, Conv):
                bound = 1 / np.sqrt(m.cin * m.k * m.k)
                P[m.off:m.off + m.n] = rng.uniform(-bound, bound, m.n)
            elif isinstance(m, Linear):
                bound = 1 / np.sqrt(m.fin)
                P[m.off:m.off + m.n] = rng.uniform(-bound, bound, m.n)
            elif isinstance(m, PReLU):
                k += 1
                P[m.off] = 1 - 1e-3 * k if near else 0.25
    return P.astype(np.float32).astype(np.float64)


def run(net, P, x, keep, dout=None, route=None):
    """float64 forward (+ backward from d sigmoid output `dout`): (sigmoid out, dx, gP, ctx)"""
    c = Ctx(torch.as_tensor(P, dtype=torch.float64), None if keep is None else torch.as_tensor(keep, dtype=torch.float64),
            route)
    x = torch.as_tensor(x, dtype=torch.float64)
    logit = net.forward(c, x)
    out = torch.sigmoid(logit)
    if dout is None:
        return out.numpy(), None, None, c
    dlogit = torch.as_tensor(dout, dtype=torch.float64) * out * (1 - out)
    dx = net.backward(c, dlogit)
    return out.numpy(), dx.numpy(), c.gP.numpy(), c
