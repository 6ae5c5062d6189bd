"""ctypes front-end of tests/hostemu/libhostemu_jacobian.so: the per-pixel pose-Jacobian math of csrc/jacobian.cu
(jacobian_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_jacobian.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_jacobian.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "jacobian_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def jac_sens_pose(sens, dsrc, dG, dWd, Wd, rows, cols, drange=None, stop_grad=False):
    """jacobian.cu's math on the CPU: sens [B, H*W, 8 | 12] -> J [B, H*W, P]; drange [B, 2, P] selects the Trilinear form."""
    tri = drange is not None
    sens, dsrc, dG, dWd, Wd, rows, cols = (_f(a) for a in (sens, dsrc, dG, dWd, Wd, rows, cols))
    drange = _f(drange) if tri else None
    B, P, H, W = dsrc.shape[0], dsrc.shape[1], rows.size, cols.size
    J = np.empty((B, H * W, P), np.float32)
    lib().emu_jac_sens_pose(ctypes.c_int(int(tri)), _p(sens), _p(dsrc), _p(dG), _p(dWd), _p(Wd), _p(rows), _p(cols), _p(drange),
                            _p(J), ctypes.c_int(B), ctypes.c_int(H), ctypes.c_int(W), ctypes.c_int(P), ctypes.c_int(int(stop_grad)))
    return J
