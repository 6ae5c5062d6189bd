"""ctypes front-end of tests/hostemu/libhostemu_brick_sens.so: the brick decomposition of the training step's sensitivities walk
(csrc/siddon_brick.cu, SENS mode; brick.cuh + ray_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_brick_sens.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_brick_sens.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "brick.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
        _lib.emu_siddon_sens_brick.restype = ctypes.c_long
    return _lib


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def siddon_sens_brick(vol, src, tgt, raylen, gout, brick=(24, 32, 32), voxel_shift=0.5, eps=1e-8):
    """Training step through the brick decomposition: dict(img, sens, g_source, g_target, g_raylen, pairs), shaped like
    tests/hostemu/emu.py's siddon_sens."""
    vol, src, tgt, raylen, gout = _f(vol), _f(src), _f(tgt), _f(raylen), _f(gout)
    B, N = tgt.shape[0], tgt.shape[1]
    out, sens = np.empty((B, 1, N), np.float32), np.empty((B, N, 8), np.float32)
    g_src, g_tgt, g_len = np.empty((B, 1, 3), np.float32), np.empty((B, N, 3), np.float32), np.empty((B, 1, N), np.float32)
    pairs = lib().emu_siddon_sens_brick(_p(vol), *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), _p(raylen), _p(gout), _p(out),
                                        _p(sens), _p(g_src), _p(g_tgt), _p(g_len), ctypes.c_int(B), ctypes.c_long(N),
                                        ctypes.c_float(voxel_shift), ctypes.c_float(eps), *map(ctypes.c_int, brick))
    return dict(img=out, sens=sens, g_source=g_src, g_target=g_tgt, g_raylen=g_len, pairs=int(pairs))
