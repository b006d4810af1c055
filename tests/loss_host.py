"""The criteria's per-pixel math header (spann3r_b200/csrc/loss_math.cuh) compiled for the CPU with g++
(tests/native/loss_host_check.cpp, no fused multiply-add) and wrapped over numpy arrays; the tests of the criteria share
it (tests/test_loss_adversarial_cpu.py pins it against numpy, tests/test_loss_adversarial.py against the kernels)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="loss_host_"), "loss_host_check.so")
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                               os.path.join(HERE, "native", "loss_host_check.cpp"), "-o", so])
        L = C.CDLL(so)
        P, LL, F, D, I = C.c_void_p, C.c_longlong, C.c_float, C.c_double, C.c_int
        L.loss_norm3.argtypes = [P, LL, P]
        L.loss_align.argtypes = [P, LL, F, F, F, P]
        L.loss_stage_value.argtypes = [P, LL, F, F, P, I, P]
        L.loss_l21.argtypes = [P, P, LL, P, P]
        L.loss_conf_term.argtypes = [P, P, LL, F, P]
        L.loss_pred_grad.argtypes = [P, P, P, LL, D, D, D, I, P]
        L.loss_order_key.argtypes = [P, LL, P]
        L.loss_key_value.argtypes = [P, LL, P]
        L.loss_median.argtypes = [P, P, LL, F, F, P, I]
        L.loss_median.restype = F
        _LIB = L
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def norm3(v):
    v = _f32(v).reshape(-1, 3)
    out = np.empty(len(v), np.float32)
    lib().loss_norm3(_p(v), len(v), _p(out))
    return out


def align(p, factor, shift, mul):
    p = _f32(p).reshape(-1, 3)
    out = np.empty_like(p)
    lib().loss_align(_p(p), len(p), factor, shift, mul, _p(out))
    return out


def stage_value(p, factor, shift, centre, kind):
    p, c = _f32(p).reshape(-1, 3), _f32(centre).reshape(3)
    out = np.empty(len(p), np.float32)
    lib().loss_stage_value(_p(p), len(p), factor, shift, _p(c), kind, _p(out))
    return out


def l21(pr, gt):
    pr, gt = _f32(pr).reshape(-1, 3), _f32(gt).reshape(-1, 3)
    u, d = np.empty_like(pr), np.empty(len(pr), np.float32)
    lib().loss_l21(_p(pr), _p(gt), len(pr), _p(u), _p(d))
    return u, d


def conf_term(d, c, alpha):
    d, c = _f32(d), _f32(c)
    out = np.empty_like(d)
    lib().loss_conf_term(_p(d), _p(c), d.size, alpha, _p(out))
    return out


def pred_grad(p, u, d, g_d, scale, coef, log1p_mode):
    p, u, d = _f32(p).reshape(-1, 3), _f32(u).reshape(-1, 3), _f32(d)
    g = np.empty_like(p)
    lib().loss_pred_grad(_p(p), _p(u), _p(d), len(p), g_d, scale, coef, int(log1p_mode), _p(g))
    return g


def order_key(v):
    v = _f32(v)
    out = np.empty(v.shape, np.uint32)
    lib().loss_order_key(_p(v), v.size, _p(out))
    return out


def key_value(k):
    k = np.ascontiguousarray(k, dtype=np.uint32)
    out = np.empty(k.shape, np.float32)
    lib().loss_key_value(_p(k), k.size, _p(out))
    return out


def median(p, valid, factor, shift, centre, kind):
    """Lower median of stage_value(kind) over the valid points, by the kernels' radix select; NaN if none."""
    p, c = _f32(p).reshape(-1, 3), _f32(centre).reshape(3)
    v = np.ascontiguousarray(valid, dtype=np.uint8).reshape(-1)
    return np.float32(lib().loss_median(_p(p), _p(v), len(p), factor, shift, _p(c), kind))
