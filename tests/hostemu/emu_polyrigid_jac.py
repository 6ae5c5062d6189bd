"""ctypes front-end of tests/hostemu/libhostemu_polyrigid_jac.so: the per-pixel motion Jacobian of csrc/polyrigid.cu
(polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra).  The library also carries emu_polyrigid.py's forward and
backward (hostemu_polyrigid_jac.cpp includes hostemu_polyrigid.cpp), which emu_polyrigid.py itself serves."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_polyrigid_jac.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_polyrigid_jac.cpp"), os.path.join(_HERE, "hostemu_polyrigid.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "polyrigid_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def polyrigid_jac(vol, src, tgt, raylen, M, weights, T, H, W, n_points, amin, amax, packed=False, voxel_shift=0.5, eps=1e-8):
    """The per-pixel motion Jacobian of b200drr_polyrigid_jac on a full H x W grid (tgt (B, H*W, 3)), T (Bm, K, 6, 3, 4) ->
    dict(img (B, H*W), J (B, K, H*W, 6), rects (B, K, 4) int32)."""
    vol, src, tgt, raylen, M, weights, T = map(_c, (vol, src, tgt, raylen, M, weights, T))
    B = tgt.shape[0]
    Bm, K = M.shape[:2]
    assert tgt.shape[1] == H * W and T.shape[:2] == (Bm, K)
    img = np.empty((B, H * W), np.float32)
    J = np.empty((B, K, H * W, 6), np.float32)
    rects = np.empty((B, K, 4), np.int32)
    lib().emu_polyrigid_jac(_p(vol), *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), _p(raylen), _p(M), ctypes.c_int(Bm),
                            ctypes.c_int(K), _p(weights), *map(ctypes.c_int, weights.shape[1:]), _p(T), _p(img), _p(J), _p(rects),
                            ctypes.c_int(B), ctypes.c_int(H), ctypes.c_int(W), ctypes.c_float(voxel_shift), ctypes.c_float(eps),
                            ctypes.c_int(n_points), ctypes.c_float(amin), ctypes.c_float(amax), ctypes.c_int(int(packed)))
    return dict(img=img, J=J, rects=rects)
