"""ctypes front-end of tests/hostemu/libhostemu_deform.so: the deformable march of csrc/deform.cu (deform_math.cuh +
polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_deform.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_deform.cpp")] + [
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
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def deform(vol, src, tgt, raylen, U, n_points, amin, amax, gout=None, packed=False, scatter=True, voxel_shift=0.5, eps=1e-8):
    """The arguments of deform_oracle.fwd / bwd -> dict(out (B, N)) and, with gout, g_src, g_tgt, g_raylen, g_U (None without
    scatter), g_alphamin, g_alphamax as deform_oracle.bwd returns them, and flushes (B, N): how often each ray added its field
    registers to g_U."""
    vol, src, tgt, raylen, U = map(_c, (vol, src, tgt, raylen, U))
    field = np.ascontiguousarray(np.concatenate([np.moveaxis(U, 1, -1), np.zeros(U.shape[:1] + U.shape[2:] + (1,), np.float32)], -1))
    B, N = tgt.shape[:2]
    Bf, g0, g1, g2 = field.shape[:4]
    out = np.empty((B, N), np.float32)
    grads = gout is not None
    gout = _c(gout) if grads else None
    g_src = np.empty((B, 3), np.float32) if grads else None
    g_tgt = np.empty((B, N, 3), np.float32) if grads else None
    g_raylen = np.empty((B, N), np.float32) if grads else None
    g_field = np.empty_like(field) if grads and scatter else None
    g_alpha = np.empty(2, np.float32) if grads else None
    flushes = np.zeros((B, N), np.int32) if grads else None
    lib().emu_deform(_p(vol), *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), _p(raylen), _p(field), ctypes.c_int(Bf),
                     *map(ctypes.c_int, (g0, g1, g2)), _p(gout), _p(out), _p(g_src), _p(g_tgt), _p(g_raylen), _p(g_field), _p(g_alpha),
                     _p(flushes), ctypes.c_int(B), ctypes.c_long(N), ctypes.c_float(voxel_shift), ctypes.c_float(eps),
                     ctypes.c_int(n_points), ctypes.c_float(amin), ctypes.c_float(amax), ctypes.c_int(int(packed)))
    res = dict(out=out)
    if grads:
        res.update(g_src=g_src, g_tgt=g_tgt, g_raylen=g_raylen, g_alphamin=float(g_alpha[0]), g_alphamax=float(g_alpha[1]),
                   flushes=flushes, g_U=None if g_field is None else np.ascontiguousarray(np.moveaxis(g_field[..., :3], -1, 1)),
                   lane3=None if g_field is None else g_field[..., 3])
    return res
