"""The per-ray frame record of the brick kernel's sensitivities mode (csrc/brick.cuh, SensFrameRec) on the CPU: a pair started from
the record that brick_prep_kernel writes (with 1/d from the ray table and s from the pose, as the kernel reads them) must give
bit for bit what brick_pair_sens gives on the freshly built ray -- the image term S, the coefficients A and C and the ray length."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu")
_SO = os.path.join(_HERE, "libhostemu_brick_sens_frame.so")
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def _load():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_brick_sens_frame.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "brick.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
        _lib.emu_brick_sens_frame_pairs.restype = ctypes.c_long
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _pairs(vol, src, tgt, raylen, brick, max_pairs=400_000, shift=0.5, eps=1e-8):
    """(fresh, framed), each [pairs][8] = S, A[3], C[3], L."""
    vol, src, tgt, raylen = (np.ascontiguousarray(x, dtype=np.float32) for x in (vol, src, tgt, raylen))
    B, N = tgt.shape[0], tgt.shape[1]
    fresh, framed = np.empty((max_pairs, 8), np.float32), np.empty((max_pairs, 8), np.float32)
    n = _load().emu_brick_sens_frame_pairs(_p(vol), *map(ctypes.c_int, vol.shape), _p(src), _p(tgt), _p(raylen), ctypes.c_int(B),
                                          ctypes.c_long(N), ctypes.c_float(shift), ctypes.c_float(eps), *map(ctypes.c_int, brick),
                                          _p(fresh), _p(framed), ctypes.c_long(max_pairs))
    assert 0 < n <= max_pairs
    return fresh[:n], framed[:n]


def _bit_equal(fresh, framed):
    assert np.array_equal(fresh.view(np.uint32), framed.view(np.uint32)), np.argwhere(fresh != framed)[:5]
    assert np.abs(fresh[:, 1:7]).max() > 0  # the pairs walked something


@pytest.mark.parametrize("brick", [(3, 4, 4), (5, 2, 7)])
def test_framed_pair_is_bit_equal_on_exact_ties(brick):
    """The dyadic geometry of test_brick_sens_cpu.py: rays through voxel edges and corners and through brick edges and corners."""
    rng = np.random.default_rng(0)
    for _ in range(6):
        dims = tuple(int(x) for x in rng.integers(8, 40, 3))
        vol = rng.random(dims).astype(np.float32)
        n = 300
        d = rng.choice([32.0, 64.0, 128.0], size=(n, 3)) * rng.choice([-1.0, 1.0], size=(n, 3))
        through = np.stack([rng.integers(0, dims[a] + 1, n).astype(np.float64) for a in range(3)], 1) - 0.5
        through += rng.choice([0.0, 0.0, 0.25, 0.5], size=(n, 1)) * rng.choice([0.0, 1.0], size=(n, 3))
        src = through - d * rng.integers(1, 4, size=(n, 1)) * 0.25
        s, t = src.astype(np.float32).reshape(n, 1, 3), (src + 2.0 * d).astype(np.float32).reshape(n, 1, 3)
        l = np.linalg.norm(t - s, axis=-1).reshape(n, 1).astype(np.float32)
        _bit_equal(*_pairs(vol, s.reshape(n, 3), t, l, brick))


def test_framed_pair_is_bit_equal_on_the_bench_rays():
    """512^3 -> 256^2, pose 1 of the bench's pose set, detector rows 45-70, production 24 x 32 x 32 bricks."""
    import torch
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import convert
    D, H = 512, 256
    x = torch.linspace(-1, 1, D)
    vol = torch.exp(-((x[:, None, None] - 0.1) ** 2 + (x[None, :, None] + 0.2) ** 2 + x[None, None, :] ** 2) / 0.3).numpy()
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H))
    rot, xyz = synthetic.make_poses(2, seed=0)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot[1:], xyz[1:], parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1)
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
    rows = slice(45 * H, 71 * H)
    _bit_equal(*_pairs(vol, src.reshape(1, 3).numpy(), tgt[:, rows].numpy(), raylen[:, rows].numpy(), (24, 32, 32)))


def test_framed_pair_is_bit_equal_with_the_source_inside_the_volume():
    """Every ray starts inside the volume: the frame's entry alpha is negative and the entry voxel is not on a face."""
    rng = np.random.default_rng(1)
    dims = (40, 36, 44)
    vol = rng.random(dims).astype(np.float32)
    B, n = 3, 400
    src = (rng.random((B, 3)) * 0.6 + 0.2) * np.array(dims) - 0.5
    d = rng.normal(size=(B, n, 3))
    d *= 80.0 / np.linalg.norm(d, axis=-1, keepdims=True)
    tgt = (src[:, None, :] + d).astype(np.float32)
    l = np.linalg.norm(d, axis=-1).astype(np.float32)
    _bit_equal(*_pairs(vol, src.astype(np.float32), tgt, l, (5, 2, 7)))
