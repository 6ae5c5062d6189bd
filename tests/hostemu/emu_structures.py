"""ctypes front-end of tests/hostemu/libhostemu_structures.so: the piecewise-rigid render of csrc/structures.cu (the gated box walk,
the footprint culling, the label boxes; structures_math.cuh + ray_math.cuh) compiled for the CPU (test infra)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_structures.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_structures.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "structures_math.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def structures(vol, labels, src, G, Wd, rows, cols, slot_of_label, box, S, sens=True, cull=True, voxel_shift=0.5, eps=1e-8):
    """src (B*S, 3), G / Wd (B*S, 3, 4), rows (H,), cols (W,), slot_of_label (256,), box (S, 6) -> dict(out (B*S, H*W),
    sens (B*S, H*W, 8) or None, rect (B*S, 4))."""
    vol, labels = _c(vol, np.float32), _c(labels, np.uint8)
    src, G, Wd, rows, cols = (_c(a, np.float32) for a in (src, G, Wd, rows, cols))
    slot_of_label, box = _c(slot_of_label, np.int32), _c(box, np.int32)
    BS, H, W = G.shape[0], rows.size, cols.size
    out = np.empty((BS, H * W), np.float32)
    sn = np.empty((BS, H * W, 8), np.float32) if sens else None
    rect = np.empty((BS, 4), np.int32)
    lib().emu_structures(_p(vol), _p(labels), *map(ctypes.c_int, vol.shape), _p(src), _p(G), _p(Wd), _p(rows), _p(cols),
                         _p(slot_of_label), _p(box), _p(out), _p(sn), _p(rect), ctypes.c_int(BS // S), ctypes.c_int(S),
                         ctypes.c_int(H), ctypes.c_int(W), ctypes.c_float(voxel_shift), ctypes.c_float(eps), ctypes.c_int(int(cull)))
    return dict(out=out, sens=sn, rect=rect)


def label_boxes(labels):
    labels = _c(labels, np.uint8)
    boxes = np.empty((256, 6), np.int32)
    lib().emu_label_boxes(_p(labels), *map(ctypes.c_int, labels.shape), _p(boxes))
    return boxes
