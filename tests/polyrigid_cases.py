"""Seeded cases of the blended-rigid (skinned) render tests (test_polyrigid_cpu.py, test_gpu_polyrigid.py).  Rays are in voxel-index
space as the kernels and polyrigid_oracle take them; the volumes, ray geometries and the SURVEY 8c tolerance rule are
trilinear_cases.py's."""
import numpy as np

import trilinear_cases as tc

DIMS = (37, 45, 29)
N_POINTS = 90


def rigid(rng, angle, shift, centre):
    """A 3 x 4 rigid map of voxel space: rotation by `angle` rad about a random axis through `centre`, then a translation of length
    `shift` voxels."""
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(angle) * Kx + (1 - np.cos(angle)) * Kx @ Kx
    t = rng.normal(size=3)
    t = shift * t / np.linalg.norm(t)
    return np.concatenate([R, (centre - R @ centre + t)[:, None]], axis=1)


def lattice(rng, K, grid, dims, total=0.9):
    """(K, *grid) smooth weights in [0, 1] with sum_k <= total: Gaussian bumps at random centres, normalised where they overlap."""
    axes = np.meshgrid(*[(np.arange(g) + 0.5) / g for g in grid], indexing="ij")
    bumps = []
    for _ in range(K):
        c = 0.2 + 0.6 * rng.random(3)
        s = 0.12 + 0.15 * rng.random()
        bumps.append(np.exp(-sum((a - ci) ** 2 for a, ci in zip(axes, c)) / (2 * s * s)))
    w = np.stack(bumps)
    w *= total / np.maximum(w.sum(0, keepdims=True), 1.0)
    return w.astype(np.float32)


def _maps(rng, Bm, K, dims, angle=0.12, shift=2.5):
    centre = (np.asarray(dims, np.float64) - 1) / 2
    return np.stack([[rigid(rng, angle, shift, centre + rng.normal(size=3) * 4) for _ in range(K)] for _ in range(Bm)]).astype(np.float32)


def _case(name, K, per_pose, grid, geometry, seed, H=9, W=11, B=2, dims=DIMS, ragged=False, push_out=False):
    rng = np.random.default_rng(seed)
    if geometry == "axis":
        src, tgt, raylen = tc.axis(dims, H, W)
        B = src.shape[0]
    else:
        src, tgt, raylen = getattr(tc, geometry)(dims, H, W, B, seed=seed)
    M = _maps(rng, B if per_pose else 1, K, dims)
    if push_out:   # structure 0 is pulled from far outside: most of what it covers samples the zero padding
        M[:, 0, :, 3] += np.float32(0.8) * np.asarray(dims, np.float32)
    N = H * W
    if ragged:     # an arbitrary ray set, not a detector grid
        keep = np.sort(rng.permutation(N)[: N - 13])
        tgt, raylen, H, W = tgt[:, keep], raylen[:, keep], 0, 0
    amin, amax = tc.range_of(dims, src, tgt)
    if geometry == "inside":
        amin = 0.0
    gout = rng.normal(size=raylen.shape).astype(np.float32)
    return dict(name=name, vol=tc.volume(dims), src=src, tgt=np.ascontiguousarray(tgt), raylen=np.ascontiguousarray(raylen), M=M,
                weights=lattice(rng, K, grid, dims), n_points=N_POINTS, amin=float(amin), amax=float(amax), H=H, W=W, gout=gout,
                kinks=tc.axis_kinks(H, W) if geometry == "axis" else None)


CASES = {
    "k1_shared": lambda: _case("k1_shared", 1, False, (8, 8, 8), "miss", 1),
    "k3_per_pose": lambda: _case("k3_per_pose", 3, True, (7, 9, 5), "miss", 2),            # lattice does not divide the volume
    "k8_shared": lambda: _case("k8_shared", 8, False, (6, 6, 6), "miss", 3),
    "k8_per_pose_ragged": lambda: _case("k8_per_pose_ragged", 8, True, (5, 6, 7), "miss", 4, ragged=True),
    "pushed_out": lambda: _case("pushed_out", 3, False, (8, 8, 8), "miss", 5, push_out=True),
    "source_inside": lambda: _case("source_inside", 3, True, (8, 8, 8), "inside", 6),
    "axis_parallel": lambda: _case("axis_parallel", 3, False, (8, 8, 8), "axis", 7),
}


def args(c):
    """The positional arguments polyrigid_oracle.fwd takes."""
    return (c["vol"], c["src"], c["tgt"], c["raylen"], c["M"], c["weights"], c["n_points"], c["amin"], c["amax"])
