"""Seeded cases of the deformable render tests (test_deform_cpu.py, test_gpu_deform.py).  Rays are in voxel-index space and fields
in voxel-index units, as the kernels and deform_oracle take them; the volumes, ray geometries and the SURVEY 8c tolerance rule are
trilinear_cases.py's."""
import numpy as np

import trilinear_cases as tc

DIMS = (37, 45, 29)
N_POINTS = 90


def smooth_field(rng, Bf, grid, amp):
    """(Bf, 3, *grid) smooth displacements of about `amp` voxels: a few random low-frequency sinusoids per component."""
    axes = np.meshgrid(*[(np.arange(g) + 0.5) / g for g in grid], indexing="ij")
    U = np.zeros((Bf, 3) + tuple(grid))
    for b in range(Bf):
        for c in range(3):
            for _ in range(3):
                k, ph = rng.normal(size=3) * 2.5, rng.random() * 2 * np.pi
                U[b, c] += np.sin(sum(ki * np.pi * a for ki, a in zip(k, axes)) + ph) / 3
    return (amp * U).astype(np.float32)


def _case(name, per_pose, grid, geometry, seed, H=9, W=11, B=2, dims=DIMS, ragged=False, amp=2.5, out_and_back=False):
    rng = np.random.default_rng(seed)
    if geometry == "axis":
        src, tgt, raylen = tc.axis(dims, H, W)
        B = src.shape[0]
    else:
        src, tgt, raylen = getattr(tc, geometry)(dims, H, W, B, seed=seed)
    U = smooth_field(rng, B if per_pose else 1, grid, amp)
    if out_and_back:   # along axis 0 the field swings by +-0.9 D0 across the lattice: samples leave the padded volume and come back
        i = (np.arange(grid[0]) + 0.5) / grid[0]
        U[:, 0] += (0.9 * dims[0] * np.sin(2 * np.pi * i))[None, :, None, None].astype(np.float32)
    N = H * W
    if ragged:     # an arbitrary ray set, not a detector grid
        keep = np.sort(rng.permutation(N)[: N - 13])
        tgt, raylen, H, W = tgt[:, keep], raylen[:, keep], 0, 0
    amin, amax = tc.range_of(dims, src, tgt)
    if geometry == "inside":
        amin = 0.0
    gout = rng.normal(size=raylen.shape).astype(np.float32)
    return dict(name=name, vol=tc.volume(dims), src=src, tgt=np.ascontiguousarray(tgt), raylen=np.ascontiguousarray(raylen), U=U,
                n_points=N_POINTS, amin=float(amin), amax=float(amax), H=H, W=W, gout=gout,
                kinks=tc.axis_kinks(H, W) if geometry == "axis" else None)


CASES = {
    "shared": lambda: _case("shared", False, (8, 8, 8), "miss", 1),
    "per_pose": lambda: _case("per_pose", True, (7, 9, 5), "miss", 2),             # lattice does not divide the volume
    "fine_lattice": lambda: _case("fine_lattice", False, (30, 37, 23), "miss", 3),   # ~one node per voxel
    "per_pose_ragged": lambda: _case("per_pose_ragged", True, (5, 6, 7), "miss", 4, ragged=True),
    "out_and_back": lambda: _case("out_and_back", False, (8, 8, 8), "miss", 5, out_and_back=True),
    "source_inside": lambda: _case("source_inside", True, (8, 8, 8), "inside", 6),
    "axis_parallel": lambda: _case("axis_parallel", False, (8, 8, 8), "axis", 7),
}


def args(c):
    """The positional arguments deform_oracle.fwd takes."""
    return (c["vol"], c["src"], c["tgt"], c["raylen"], c["U"], c["n_points"], c["amin"], c["amax"])


def pack(U):
    """(Bf, 3, g0, g1, g2) -> the kernels' layout (Bf, g0, g1, g2, 4), lane 3 zero."""
    U = np.asarray(U, np.float32)
    return np.ascontiguousarray(np.concatenate([np.moveaxis(U, 1, -1), np.zeros(U.shape[:1] + U.shape[2:] + (1,), np.float32)], -1))
