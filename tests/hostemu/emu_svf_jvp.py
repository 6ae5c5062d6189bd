"""ctypes front-end of tests/hostemu/libhostemu_svf_jvp.so: the tangent of one scaling-and-squaring step of csrc/svf.cu
(svf_math.cuh + deform_math.cuh + polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra).  Fields here are
(Bf, g0, g1, g2, 3) in voxel units, as tests/svf_oracle.py takes them."""
import ctypes
import os
import subprocess

import numpy as np

from hostemu.emu_svf import _args, _p, _pad

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_svf_jvp.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_svf_jvp.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "polyrigid_math.cuh",
                                                                     "deform_math.cuh", "svf_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def square_jvp(u, t, s, D, primal=True):
    """The tangent of one squaring step at u along t, both (Bf, g0, g1, g2, 3) -> (t' (Bf, g0, g1, g2, 3), lane 3 of the kernel's
    tangent output, u' (Bf, g0, g1, g2, 4) with its lane 3, or None with primal=False: the kernel's out left NULL)."""
    field, tan = _pad(u), _pad(t)
    tout = np.full_like(field, np.nan)
    out = np.full_like(field, np.nan) if primal else None
    lib().emu_svf_square_jvp(_p(field), _p(tan), _p(tout), None if out is None else _p(out), *_args(field, D, s))
    return tout[..., :3], tout[..., 3], out


def exp_jvp(v, t, steps, D):
    """exp(v) and its tangent along t by `steps` emulated tangent squarings, the primal carried through `out` -> both
    (Bf, g0, g1, g2, 3)."""
    u, t = np.asarray(v, np.float32), np.asarray(t, np.float32)
    for k in range(steps):
        t, _, out = square_jvp(u, t, 2.0**-steps if k == 0 else 1.0, D)
        u = out[..., :3]
    return u, t
