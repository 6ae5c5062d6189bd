"""ctypes front-end of tests/hostemu/libhostemu_metrics.so: the image-loss math of csrc/local_ncc.cu and csrc/sobel.cu
(local_ncc_math.cuh, sobel_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_metrics.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_metrics.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f)
            for f in ("common.cuh", "ncc_math.cuh", "local_ncc_math.cuh", "sobel_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def local_ncc(x1, x2, patch_size, gscore=None, eps=1e-5):
    """local_ncc.cu's math (box sums of double moments, adjoint box sums) on the CPU: (score [B], g_x1, g_x2)."""
    x1, x2 = _f(x1), _f(x2)
    B, C, H, W = x1.shape
    p = int(patch_size)
    stats = np.empty((B * C, 5, H - p + 1, W - p + 1), np.float32)
    score = np.empty(B, np.float32)
    dims = [ctypes.c_int(v) for v in (B, C, H, W, p)]
    lib().emu_local_ncc_fwd(_p(x1), _p(x2), *dims, ctypes.c_float(eps), _p(stats), _p(score))
    if gscore is None:
        return score
    g1, g2 = np.empty_like(x1), np.empty_like(x2)
    lib().emu_local_ncc_bwd(_p(x1), _p(x2), _p(stats), _p(_f(gscore)), _p(g1), _p(g2), *dims)
    return score, g1, g2


def sobel_fwd(x, weights):
    """sobel.cu's forward on the CPU: x [B, 1, H, W], 1-D blur weights [k] -> [B, 2, H, W]."""
    x, w = _f(x), _f(weights)
    B, _, H, W = x.shape
    out = np.empty((B, 2, H, W), np.float32)
    lib().emu_sobel_fwd(_p(x), _p(out), ctypes.c_int(B), ctypes.c_int(H), ctypes.c_int(W), _p(w), ctypes.c_int(w.size))
    return out


def sobel_bwd(gout, weights):
    """sobel.cu's adjoint on the CPU: gout [B, 2, H, W] -> g_x [B, 1, H, W]."""
    gout, w = _f(gout), _f(weights)
    B, _, H, W = gout.shape
    g = np.empty((B, 1, H, W), np.float32)
    lib().emu_sobel_bwd(_p(gout), _p(g), ctypes.c_int(B), ctypes.c_int(H), ctypes.c_int(W), _p(w), ctypes.c_int(w.size))
    return g
