"""The named ray geometries of the trilinear oracle tests (tests/trilinear_cases.py) are what their names say, and every bound the
SURVEY 8c rule derives on them stays finite and below trilinear_cases.TOL_CAP.  Oracle only: runs without a GPU."""
import numpy as np
import pytest

import trilinear_cases as tc
from oracle import oracle

DIMS_A, H_A, W_A, B_A = tc.SHAPE_A


def test_detector_sides_are_not_multiples_of_the_tiles():
    for dims, H, W, _ in tc.PARTIAL_TILE_SHAPES:
        assert H % 16 and W % 16, (dims, H, W)
    assert DIMS_A[0] % 2 and DIMS_A[2] % 2     # odd volume sides
    assert min(tc.SHAPE_THIN[0]) == 2 and min(tc.SHAPE_SLIVER[0]) == 1


def test_miss_rays_give_exact_zeros_and_share_their_poses_with_hits():
    src, tgt, raylen = tc.miss(DIMS_A, H_A, W_A, B_A, seed=1)
    vol = np.random.default_rng(0).random(DIMS_A, dtype=np.float32) + 0.5      # no zero voxel anywhere
    amin, amax = tc.range_of(DIMS_A, src, tgt)
    img = oracle.trilinear_fwd(vol, src[:, None], tgt, raylen[:, None], n_points=77, alphamin=amin, alphamax=amax,
                               dtype=np.float64).reshape(B_A, -1)
    lo, hi = tc.entry_exit(DIMS_A, src, tgt, padded=True)
    missed = ~(lo < hi)
    for b in range(B_A):
        assert 0.2 * missed[b].size < missed[b].sum() < 0.8 * missed[b].size
        assert (img[b][missed[b]] == 0.0).all()
        assert (img[b][~missed[b]] > 0.0).mean() > 0.95


def test_inside_sources_enter_before_alpha_zero():
    src, tgt, _ = tc.inside(DIMS_A, H_A, W_A, B_A, seed=2)
    assert ((src >= 0) & (src <= np.asarray(DIMS_A) - 1)).all()
    lo, hi = tc.entry_exit(DIMS_A, src, tgt)
    assert (lo < 0).all() and (hi > 0).all()


@pytest.mark.parametrize("shift", [0.5, 0.0])
@pytest.mark.parametrize("shape", [tc.SHAPE_A, tc.SHAPE_THIN, tc.SHAPE_SLIVER])
def test_axis_parallel_rays_lie_where_their_names_say(shape, shift):
    dims, H, W, _ = shape
    planes = tc.axis_planes(dims, shift)
    src, tgt, _ = tc.axis(dims, H, W, shift)
    assert src.shape[0] == len(planes) and (-0.5 in planes) and float(dims[0] - 1) in planes
    for b, p in enumerate(planes):
        pix0 = tc.pix(src[b, 0], shift)
        assert pix0 == np.float32(p)                                   # the intended integer plane / half-cell, exactly
        assert (p == int(p)) or (-1.0 < p < 0.0)
        rows = tgt[b].reshape(H, W, 3)
        for h in range(H):
            k = tc.axis_row_kind(h)
            if k == 0:
                assert (rows[h, :, 0] - src[b, 0] == 0.0).all()         # exactly zero direction along axis 0 (the slab axis)
                assert rows[h, W // 2, 2] - src[b, 2] == 0.0           # ... and along axis 2 in the centre column
                assert tc.pix(src[b, 2], shift) == np.floor(tc.pix(src[b, 2], shift))   # at an integer pix2
            elif k == 1:
                assert (rows[h, :, 0] == np.nextafter(src[b, 0], np.float32(-np.inf))).all()
            else:
                assert (rows[h, :, 0] != src[b, 0]).all() or h == H // 2
    lo, hi = tc.entry_exit(dims, src, tgt, shift)
    assert (lo < hi).any(axis=1).all()                                  # every pose hits the volume


def _tolerances(vol, src, tgt, raylen, n_points, amin, amax, shift=0.5, kinks=None):
    """The bounds test_gpu_trilinear_oracle derives: image, g_volume, g_raylen with gout on every ray; end points and range
    partials with gout zeroed on the kink rays of the axis-parallel geometry."""
    B, N = tgt.shape[:2]
    gout = np.random.default_rng(5).random((B, 1, N), dtype=np.float32)
    args = (vol, src[:, None], tgt, raylen[:, None])
    fkw = dict(n_points=n_points, alphamin=amin, alphamax=amax, voxel_shift=shift)
    i64 = oracle.trilinear_fwd(*args, dtype=np.float64, **fkw)
    i32 = oracle.trilinear_fwd(*args, dtype=np.float32, **fkw)
    assert tc.relerr(i32, i64) < 1e-4
    g64 = oracle.trilinear_bwd(*args, gout, dtype=np.float64, **fkw)
    g32 = oracle.trilinear_bwd(*args, gout, dtype=np.float32, **fkw)
    out = {k: tc.tol(g32[k], g64[k], 1e-4) for k in ("g_volume", "g_raylen")}
    if kinks is not None:
        gout = gout * ~kinks.reshape(1, 1, N)
        g64 = oracle.trilinear_bwd(*args, gout, dtype=np.float64, want_vol=False, **fkw)
        g32 = oracle.trilinear_bwd(*args, gout, dtype=np.float32, want_vol=False, **fkw)
    out.update({k: tc.tol(g32[k], g64[k], 1e-3) for k in ("g_target", "g_source")})
    ga32 = tc.alpha_partials_f32(vol, src, tgt, raylen, gout, **fkw)
    scale = tc.alpha_scale(g64["g_raylen"], raylen, amin, amax)
    out["g_alpha"] = tc.tol(ga32, [g64["g_alphamin"], g64["g_alphamax"]], 1e-3, scale)
    return out


@pytest.mark.parametrize("name", ["inside", "miss", "axis", "axis_shift0", "near_identical"])
def test_8c_tolerances_are_finite_and_capped(name):
    """The bound of every gradient the GPU test compares, derived on the named geometry from the oracle's own fp32 run."""
    dims, H, W, B = tc.SHAPE_A
    shift = 0.0 if name == "axis_shift0" else 0.5
    if name == "near_identical":
        dims, H, W, B = (32, 32, 32), 48, 48, 4
        src, tgt, raylen = tc.near_identical(dims, H, W, B)
    elif name.startswith("axis"):
        src, tgt, raylen = tc.axis(dims, H, W, shift)
    else:
        src, tgt, raylen = getattr(tc, name)(dims, H, W, B, seed=3)
    vol = tc.volume(dims)
    amin, amax = tc.range_of(dims, src, tgt, shift)
    kinks = tc.axis_kinks(H, W) if name.startswith("axis") else None
    for P in (77,) if name == "near_identical" else (2, 77):   # the contention case runs at 77 samples
        t = _tolerances(vol, src, tgt, raylen, P, amin, amax, shift, kinks)
        assert all(np.isfinite(v) and v <= tc.TOL_CAP for v in t.values()), t
