"""ctypes front-end of tests/hostemu/libhostemu_deform_bproj.so: the density backprojection of csrc/deform.cu (deform_math.cuh +
polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra).  The library also carries emu_deform.py's forward and
backward (hostemu_deform_bproj.cpp includes hostemu_deform.cpp), which emu_deform.py itself serves."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_deform_bproj.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_deform_bproj.cpp"), os.path.join(_HERE, "hostemu_deform.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "polyrigid_math.cuh",
                                                                     "deform_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def deform_bproj(shape, src, tgt, raylen, U, n_points, amin, amax, gout, voxel_shift=0.5, eps=1e-8):
    """The volume's shape, deform_oracle.fwd's other arguments and gout (B, N) -> g_V (D0, D1, D2) fp32: the gradient of
    sum(gout * image) with respect to the density, summed over the poses."""
    src, tgt, raylen, gout = map(_c, (src, tgt, raylen, gout))
    U = _c(U)
    field = np.ascontiguousarray(np.concatenate([np.moveaxis(U, 1, -1), np.zeros(U.shape[:1] + U.shape[2:] + (1,), np.float32)], -1))
    B, N = tgt.shape[:2]
    Bf, g0, g1, g2 = field.shape[:4]
    g_vol = np.empty(tuple(shape), np.float32)
    lib().emu_deform_bproj(*map(ctypes.c_int, shape), _p(src), _p(tgt), _p(raylen), _p(field), ctypes.c_int(Bf),
                           *map(ctypes.c_int, (g0, g1, g2)), _p(gout), _p(g_vol), ctypes.c_int(B), ctypes.c_long(N),
                           ctypes.c_float(voxel_shift), ctypes.c_float(eps), ctypes.c_int(n_points), ctypes.c_float(amin),
                           ctypes.c_float(amax))
    return g_vol
