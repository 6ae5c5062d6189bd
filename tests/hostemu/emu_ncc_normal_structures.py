"""ctypes front-end of tests/hostemu/libhostemu_ncc_normal_structures.so: the block-sparse normal equations and the structure
footprints of csrc/ncc_normal_structures.cu (ncc_normal_structures_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_ncc_normal_structures.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_ncc_normal_structures.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "structures_math.cuh",
                                                                     "ncc_normal_math.cuh", "ncc_normal_structures_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def footprints(src, G, rows, cols, box, S, voxel_shift=0.5):
    """src (B*S, 3), G (B*S, 3, 4), rows (H,), cols (W,), box (S, 6) -> rects (B*S, 4) int32."""
    src, G, rows, cols = (np.ascontiguousarray(a, np.float32) for a in (src, G, rows, cols))
    box = np.ascontiguousarray(box, np.int32)
    BS = G.shape[0]
    rects = np.empty((BS, 4), np.int32)
    lib().emu_structure_footprints(_p(src), _p(G), _p(rows), _p(cols), _p(box), _p(rects), ctypes.c_int(BS // S), ctypes.c_int(S),
                                   ctypes.c_int(rows.size), ctypes.c_int(cols.size), ctypes.c_float(voxel_shift))
    return rects


def ncc_normal_structures(x, t, J, strides, rects, K, S, eps=1e-5, weight=1.0):
    """x (B, H, W), t (1 or B, H, W); J a flat fp32 array addressed by the element strides (pose, structure, pixel, parameter);
    rects (B, S, 4) -> (A (B, 6K, 6K), g (B, 6K)) float64, weight times the sums."""
    x = np.ascontiguousarray(x, np.float32)
    t = np.ascontiguousarray(t, np.float32)
    J = np.ascontiguousarray(J, np.float32).reshape(-1)
    rects = np.ascontiguousarray(rects, np.int32)
    B, H, W = x.shape
    P = 6 * K
    A = np.zeros((B, P, P), np.float64)
    g = np.zeros((B, P), np.float64)
    lib().emu_ncc_normal_structures(_p(x), _p(t), ctypes.c_int(t.shape[0]), _p(J), *(ctypes.c_long(int(s)) for s in strides),
                                    _p(rects), ctypes.c_int(B), ctypes.c_int(K), ctypes.c_int(S), ctypes.c_int(H), ctypes.c_int(W),
                                    ctypes.c_double(eps), ctypes.c_double(weight), _p(A), _p(g))
    return A, g
