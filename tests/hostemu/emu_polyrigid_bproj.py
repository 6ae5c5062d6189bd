"""ctypes front-end of tests/hostemu/libhostemu_polyrigid_bproj.so: the density backprojection of csrc/polyrigid.cu
(polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra).  The library also carries emu_polyrigid.py's forward and
backward (hostemu_polyrigid_bproj.cpp includes hostemu_polyrigid.cpp), which emu_polyrigid.py itself serves."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_polyrigid_bproj.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_polyrigid_bproj.cpp"), os.path.join(_HERE, "hostemu_polyrigid.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "polyrigid_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def polyrigid_bproj(shape, src, tgt, raylen, M, weights, n_points, amin, amax, gout, voxel_shift=0.5, eps=1e-8):
    """The volume's shape, polyrigid_oracle.fwd's other arguments and gout (B, N) -> g_V (D0, D1, D2) fp32: the gradient of
    sum(gout * image) with respect to the density, summed over the poses."""
    src, tgt, raylen, M, weights, gout = map(_c, (src, tgt, raylen, M, weights, gout))
    B, N = tgt.shape[:2]
    Bm, K = M.shape[:2]
    g_vol = np.empty(tuple(shape), np.float32)
    lib().emu_polyrigid_bproj(*map(ctypes.c_int, shape), _p(src), _p(tgt), _p(raylen), _p(M), ctypes.c_int(Bm), ctypes.c_int(K),
                              _p(weights), *map(ctypes.c_int, weights.shape[1:]), _p(gout), _p(g_vol), ctypes.c_int(B),
                              ctypes.c_long(N), ctypes.c_float(voxel_shift), ctypes.c_float(eps), ctypes.c_int(n_points),
                              ctypes.c_float(amin), ctypes.c_float(amax))
    return g_vol
