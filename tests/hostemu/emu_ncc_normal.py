"""ctypes front-end of tests/hostemu/libhostemu_ncc_normal.so: the NCC normal-equation math of csrc/ncc_normal.cu
(ncc_normal_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_ncc_normal.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_ncc_normal.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ncc_normal_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def ncc_normal(x, t, J, strides, P, p, eps=1e-5, weight=1.0):
    """ncc_normal.cu's math on the CPU: x, t [B, C, H, W]; J a flat fp32 array addressed by the element strides (pose, channel,
    parameter, pixel) with P parameters; p = 0 for the global NCC.  -> (A [B, P, P], g [B, P]) in float64, weight times the sums."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    t = np.ascontiguousarray(t, dtype=np.float32)
    J = np.ascontiguousarray(J, dtype=np.float32).reshape(-1)
    B, C, H, W = x.shape
    A = np.zeros((B, P, P), np.float64)
    g = np.zeros((B, P), np.float64)
    lib().emu_ncc_normal(_p(x), _p(t), _p(J), *(ctypes.c_long(int(s)) for s in strides), ctypes.c_int(B), ctypes.c_int(C),
                         ctypes.c_int(H), ctypes.c_int(W), ctypes.c_int(p), ctypes.c_int(P), ctypes.c_double(eps),
                         ctypes.c_double(weight), _p(A), _p(g))
    return A, g
