"""ctypes front-end of tests/hostemu/libhostemu_svf.so: the scaling-and-squaring step of csrc/svf.cu (svf_math.cuh +
deform_math.cuh + polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra).  Fields here are (Bf, g0, g1, g2, 3) in
voxel units, as tests/svf_oracle.py takes them."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_svf.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_svf.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "polyrigid_math.cuh",
                                                                     "deform_math.cuh", "svf_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _pad(u):
    u = np.asarray(u, np.float32)
    return np.ascontiguousarray(np.concatenate([u, np.zeros(u.shape[:-1] + (1,), np.float32)], -1))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _args(field, D, s):
    Bf, g0, g1, g2 = field.shape[:4]
    return (*map(ctypes.c_int, (Bf, g0, g1, g2, *D)), ctypes.c_float(s))


def square(u, s, D):
    """One squaring step of u (Bf, g0, g1, g2, 3) -> (u' (Bf, g0, g1, g2, 3), lane 3 of the kernel's output)."""
    field = _pad(u)
    out = np.full_like(field, np.nan)
    lib().emu_svf_square(_p(field), _p(out), *_args(field, D, s))
    return out[..., :3], out[..., 3]


def square_bwd(u, gp, s, D):
    """The step's adjoint at u for the upstream gradient gp -> (g (Bf, g0, g1, g2, 3), lane 3 of the kernel's output)."""
    field, g = _pad(u), _pad(gp)
    gin = np.full_like(field, np.nan)
    lib().emu_svf_square_bwd(_p(field), _p(g), _p(gin), *_args(field, D, s))
    return gin[..., :3], gin[..., 3]


def exp(v, steps, D):
    """exp(v) by `steps` emulated squarings -> the displacement (Bf, g0, g1, g2, 3)."""
    u = np.asarray(v, np.float32)
    for k in range(steps):
        u = square(u, 2.0**-steps if k == 0 else 1.0, D)[0]
    return u
