"""ctypes front-end of tests/hostemu/libhostemu_log_euclidean_jac.so: the P-tangent squaring step of csrc/svf.cu and the Jacobian
march of csrc/deform.cu (svf_math.cuh + deform_math.cuh + polyrigid_math.cuh + ray_math.cuh) compiled for the CPU (test infra).
Fields here are (Bf, g0, g1, g2, 3) and tangents (Bf, g0, g1, g2, P, 3), voxel units."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_log_euclidean_jac.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_log_euclidean_jac.cpp"), os.path.join(_HERE, "hostemu_deform.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "polyrigid_math.cuh",
                                                                     "deform_math.cuh", "svf_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _pad(a):
    a = np.asarray(a, np.float32)
    return np.ascontiguousarray(np.concatenate([a, np.zeros(a.shape[:-1] + (1,), np.float32)], -1))


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _i(*v):
    return [ctypes.c_int(int(x)) for x in v]


def square_tangents(u, T, s, D, primal=True):
    """One P-tangent squaring step at u (Bf, g0, g1, g2, 3) along T (Bf, g0, g1, g2, P, 3) -> (T' (..., P, 3), lane 3 of T',
    u' (Bf, g0, g1, g2, 4) or None with primal=False)."""
    field, tan = _pad(u), _pad(T)
    tout = np.full_like(tan, np.nan)
    out = np.full_like(field, np.nan) if primal else None
    Bf, g0, g1, g2, P = tan.shape[:5]
    lib().emu_svf_square_tangents(_p(field), _p(tan), _p(tout), _p(out), *_i(Bf, P, g0, g1, g2, *D), ctypes.c_float(s))
    return tout[..., :3], tout[..., 3], out


def deform_jac(vol, src, tgt, raylen, U, T, K, H, W, n_points, amin, amax, packed=False, voxel_shift=0.5, eps=1e-8):
    """U (Bf, g0, g1, g2, 3) and T (Bf, g0, g1, g2, 6K, 3) in voxel units; rays as deform_oracle takes them, on a full H x W grid
    -> dict(img (B, H*W), J (B, K, H*W, 6), rects (B, K, 4), flushes (B, H*W))."""
    vol, src, tgt, raylen = (np.ascontiguousarray(x, np.float32) for x in (vol, src, tgt, raylen))
    field, tan = _pad(U), _pad(T)
    Bf, g0, g1, g2 = field.shape[:4]
    B = tgt.shape[0]
    img = np.empty((B, H * W), np.float32)
    J = np.empty((B, K, H * W, 6), np.float32)
    rects = np.empty((B, K, 4), np.int32)
    flushes = np.empty((B, H * W), np.int32)
    lib().emu_deform_jac(_p(vol), *_i(*vol.shape), _p(src), _p(tgt), _p(raylen), _p(field), _p(tan), *_i(Bf, g0, g1, g2, K), _p(img),
                         _p(J), _p(rects), _p(flushes), *_i(B, H, W), ctypes.c_float(voxel_shift), ctypes.c_float(eps),
                         ctypes.c_int(n_points), ctypes.c_float(amin), ctypes.c_float(amax), ctypes.c_int(int(packed)))
    return dict(img=img, J=J, rects=rects, flushes=flushes)
