"""ctypes front-end of oracle/libfg_oracle_c2f_sized.so: the coarse-to-fine restatement (oracle_c2f.py) at a runtime
fine size S = train_c2f.lua --fineSize (16, 32 or 64).

TEST INFRASTRUCTURE ONLY (same rules as oracle.py).  PARITY UNPINNED.
The library is fg_oracle_c2f_sized.cpp: the whole of fg_oracle.cpp plus the sized nets, built with the flags of
oracle/Makefile by build() (called from __graft_entry__.build()).
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "fg_oracle_c2f_sized.cpp")
_SO = os.path.join(_HERE, "libfg_oracle_c2f_sized.so")
_FLAGS = ["-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-std=c++17", "-fno-fast-math"]  # oracle/Makefile's


def build(force=False):
    srcs = [_SRC] + [os.path.join(_HERE, f) for f in ("fg_oracle.cpp", "fg_oracle_c2f.h", "fg_oracle_s16.h")]
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        tmp = _SO + ".tmp"
        subprocess.check_call(["/usr/bin/g++"] + _FLAGS + ["-shared", "-o", tmp, _SRC, "-ldl"])
        os.replace(tmp, _SO)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.fgo_c2fs_D_param_count.restype = C.c_long
        for sfx in ("f64", "f32"):
            getattr(_lib, "fgo_c2fs_G_new_" + sfx).restype = C.c_void_p
            getattr(_lib, "fgo_c2fs_D_new_" + sfx).restype = C.c_void_p
    return _lib


def flat(S):
    """D.L1's input width: View(256*(S/4)^2) of [256][S/4][S/4]"""
    return 256 * (S // 4) ** 2


def mask_per_sample(S):
    return int(lib().fgo_c2fs_mask_per_sample(S))


def G_param_count(c):
    return int(O.lib().fgo_c2f_G_param_count(c))  # G does not depend on S


def D_param_count(c, S):
    return int(lib().fgo_c2fs_D_param_count(c, S))


def G_layout(c):
    from . import oracle_c2f as OC
    return OC.G_layout(c)


def D_layout(c, S):
    """name -> (offset, shape), getParameters order of create_D_c (models_c2f.lua:247-265) at fine size S."""
    cin, cout = [c, 64, 64, 128], [64, 64, 128, 256]
    items = []
    for i in range(4):
        items += [("c%dW" % (i + 1), (cout[i], cin[i], 3, 3)), ("c%db" % (i + 1), (cout[i],)), ("a%d" % (i + 1), (1,))]
    items += [("L1W", (512, flat(S))), ("L1b", (512,)), ("a5", (1,)), ("L2W", (1, 512)), ("L2b", (1,))]
    out, o = {}, 0
    for name, shape in items:
        out[name] = (o, shape)
        o += int(np.prod(shape))
    assert o == D_param_count(c, S)
    return out


class _T(O._T):
    def f(self, name):
        return getattr(lib(), "fgo_%s_%s" % (name, self.sfx))


class _C2fSized:
    def __init__(self, t):
        self.t = t

    def G(self, S):
        return _GNet(self.t, S)

    def D(self, S):
        return _DNet(self.t, S)

    def train_iteration(self, S, B, Cc, hyper, real_diff, condD, noiseD, condG, noiseG, masksD, masksG, state,
                        want_grads=True):
        """oracle_c2f train_iteration at fine size S; state: dict PD,PG,mD,vD,mG,vG (updated in place), tD,tG ints."""
        t = self.t
        hp = np.array([hyper[k] for k in ("lr_D", "lr_G", "beta1", "beta2", "eps", "D_L1", "D_L2", "G_L1", "G_L2",
                                          "D_clamp", "G_clamp")], np.float64)
        real_diff, condD, noiseD, condG, noiseG, masksD, masksG = map(
            t.a, (real_diff, condD, noiseD, condG, noiseG, masksD, masksG))
        tD, tG = C.c_int(state["tD"]), C.c_int(state["tG"])
        stats = np.zeros(8, np.float64)
        gD = np.zeros(state["PD"].size, t.dtype) if want_grads else None
        gG = np.zeros(state["PG"].size, t.dtype) if want_grads else None
        fake = np.zeros((B // 2, Cc, S, S), t.dtype)
        outD = np.zeros(B, t.dtype)
        t.f("c2fs_train_iteration")(S, B, Cc, t.p(hp), t.p(real_diff), t.p(condD), t.p(noiseD), t.p(condG),
                                    t.p(noiseG), t.p(masksD), t.p(masksG), t.p(state["PD"]), t.p(state["PG"]),
                                    t.p(state["mD"]), t.p(state["vD"]), t.p(state["mG"]), t.p(state["vG"]),
                                    C.byref(tD), C.byref(tG), t.p(stats), t.p(gD), t.p(gG), t.p(fake), t.p(outD))
        state["tD"], state["tG"] = tD.value, tG.value
        return dict(lossD=stats[0], lossG=stats[1], conf=stats[2:6].copy(), gradD=gD, gradG=gG, fake=fake, outD=outD)


class _GNet:
    def __init__(self, t, S):
        self.t, self.S = t, S
        self.h = C.c_void_p(t.f("c2fs_G_new")(S))

    def __del__(self):
        try:
            self.t.f("c2fs_G_free")(self.h)
        except Exception:
            pass

    def forward(self, P, noise, cond):
        t = self.t
        self.P, noise, cond = t.a(P), t.a(noise), t.a(cond)
        B, Cc = cond.shape[0], cond.shape[1]
        out = np.empty((B, Cc, self.S, self.S), t.dtype)
        t.f("c2fs_G_forward")(self.h, t.p(self.P), t.p(noise), t.p(cond), B, Cc, t.p(out))
        return out

    def backward(self, dout):
        t = self.t
        dP = np.zeros(self.P.size, t.dtype)
        t.f("c2fs_G_backward")(self.h, t.p(self.P), t.p(t.a(dout)), t.p(dP))
        return dP


class _DNet:
    def __init__(self, t, S):
        self.t, self.S = t, S
        self.h = C.c_void_p(t.f("c2fs_D_new")(S))

    def __del__(self):
        try:
            self.t.f("c2fs_D_free")(self.h)
        except Exception:
            pass

    def forward(self, P, diff, cond, masks=None, training=True):
        t = self.t
        self.P, diff, cond = t.a(P), t.a(diff), t.a(cond)
        B, Cc = diff.shape[0], diff.shape[1]
        self.B, self.C = B, Cc
        masks = t.a(masks) if masks is not None else None
        out = np.empty(B, t.dtype)
        t.f("c2fs_D_forward")(self.h, t.p(self.P), t.p(diff), t.p(cond), B, Cc, int(training), t.p(masks), t.p(out))
        return out

    def backward(self, dout, want_dP=True, want_ddiff=True):
        t = self.t
        dP = np.zeros(self.P.size, t.dtype) if want_dP else None
        dd = np.zeros((self.B, self.C, self.S, self.S), t.dtype) if want_ddiff else None
        t.f("c2fs_D_backward")(self.h, t.p(self.P), t.p(t.a(dout)), t.p(dP), t.p(dd))
        return dP, dd


f64 = _C2fSized(_T("f64", np.float64))
f32 = _C2fSized(_T("f32", np.float32))
