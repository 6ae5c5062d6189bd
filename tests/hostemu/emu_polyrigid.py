"""ctypes front-end of tests/hostemu/libhostemu_polyrigid.so: the blended-rigid march of csrc/polyrigid.cu (polyrigid_math.cuh +
ray_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_polyrigid.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_polyrigid.cpp")] + [
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


def polyrigid(vol, src, tgt, raylen, M, weights, n_points, amin, amax, gout=None, packed=False, voxel_shift=0.5, eps=1e-8):
    """The arguments of polyrigid_oracle.fwd / bwd -> dict(out (B, N)) and, with gout, g_src, g_tgt, g_raylen, g_M, g_alphamin,
    g_alphamax as polyrigid_oracle.bwd returns them."""
    vol, src, tgt, raylen, M, weights = map(_c, (vol, src, tgt, raylen, M, weights))
    B, N = tgt.shape[:2]
    Bm, K = M.shape[:2]
    out = np.empty((B, N), np.float32)
    grads = gout is not None
    gout = _c(gout) if grads else None
    g_src = np.empty((B, 3), np.float32) if grads else None
    g_tgt = np.empty((B, N, 3), np.float32) if grads else None
    g_raylen = np.empty((B, N), np.float32) if grads else None
    g_M = np.empty((Bm, K, 3, 4), np.float32) if grads else None
    g_alpha = np.empty(2, np.float32) if grads else None
    lib().emu_polyrigid(_p(vol), *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), _p(raylen), _p(M), ctypes.c_int(Bm), ctypes.c_int(K),
                        _p(weights), *map(ctypes.c_int, weights.shape[1:]), _p(gout), _p(out), _p(g_src), _p(g_tgt), _p(g_raylen),
                        _p(g_M), _p(g_alpha), ctypes.c_int(B), ctypes.c_long(N), ctypes.c_float(voxel_shift), ctypes.c_float(eps),
                        ctypes.c_int(n_points), ctypes.c_float(amin), ctypes.c_float(amax), ctypes.c_int(int(packed)))
    res = dict(out=out)
    if grads:
        res.update(g_src=g_src, g_tgt=g_tgt, g_raylen=g_raylen, g_M=g_M, g_alphamin=float(g_alpha[0]), g_alphamax=float(g_alpha[1]))
    return res


def trilinear(vol, src, tgt, raylen, n_points, amin, amax, voxel_shift=0.5, eps=1e-8):
    """The Trilinear renderer's forward (trilinear_ray_fwd) on the same rays -> (B, N)."""
    vol, src, tgt, raylen = map(_c, (vol, src, tgt, raylen))
    B, N = tgt.shape[:2]
    out = np.empty((B, N), np.float32)
    lib().emu_polyrigid_trilinear(_p(vol), *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), _p(raylen), _p(out), ctypes.c_int(B),
                                  ctypes.c_long(N), ctypes.c_float(voxel_shift), ctypes.c_float(eps), ctypes.c_int(n_points),
                                  ctypes.c_float(amin), ctypes.c_float(amax))
    return out
