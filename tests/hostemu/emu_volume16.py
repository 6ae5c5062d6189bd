"""ctypes front-end of tests/hostemu/libhostemu_volume16.so: the 16-bit voxel reads of the Siddon kernels (common.cuh, ray_math.cuh,
brick.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_volume16.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None

VOL_TYPES = {"float32": 0, "float16": 1, "bfloat16": 2}


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_volume16.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "brick.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
        _lib.emu_siddon_walks16.restype = ctypes.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def vox16_to_f32(bits, bf16: bool):
    """uint16 bit patterns -> float32 through the kernels' conversion function."""
    bits = np.ascontiguousarray(bits, dtype=np.uint16)
    out = np.empty(bits.shape, np.float32)
    lib().emu_vox16_to_f32(_p(bits), _p(out), ctypes.c_long(bits.size), ctypes.c_int(int(bf16)))
    return out


def siddon_walks(vol, vol_type, src, tgt, brick=(24, 32, 32), voxel_shift=0.5, eps=1e-8):
    """vol: float32 array (vol_type 'float32') or uint16 bit patterns ('float16' / 'bfloat16').  Returns dict(lean (B, N),
    sens (B, N, 7) = (S, A, C), brick_fwd, brick_sens) of the whole-volume walks and of the brick decomposition."""
    vol = np.ascontiguousarray(vol, dtype=np.float32 if vol_type == "float32" else np.uint16)
    src, tgt = np.ascontiguousarray(src, np.float32), np.ascontiguousarray(tgt, np.float32)
    B, N = tgt.shape[0], tgt.shape[1]
    lean, bfwd = np.empty((B, N), np.float32), np.empty((B, N), np.float32)
    sens, bsens = np.empty((B, N, 7), np.float32), np.empty((B, N, 7), np.float32)
    rc = lib().emu_siddon_walks16(_p(vol), VOL_TYPES[vol_type], *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), ctypes.c_int(B),
                                  ctypes.c_long(N), ctypes.c_float(voxel_shift), ctypes.c_float(eps), *map(ctypes.c_int, brick),
                                  _p(lean), _p(sens), _p(bfwd), _p(bsens))
    assert rc == 0
    return dict(lean=lean, sens=sens, brick_fwd=bfwd, brick_sens=bsens)
