"""The named ray geometries and ray classes of the Siddon oracle tests (tests/siddon_cases.py): each geometry is what its name says,
the classes cover every ray on which the oracle's own fp32 and fp64 disagree while leaving out few rays, exact ties have an exact
reference, and the host emulation of the kernels' walk pins the tie convention.  Oracle and host emulation only: no GPU."""
import functools

import numpy as np
import pytest

import siddon_cases as sc
import trilinear_cases as tc
from conftest import relerr
from oracle import oracle

DIMS_A4, H_A, W_A, B_A = sc.SHAPE_A4


@functools.lru_cache(maxsize=None)
def _geometry(name):
    """-> (dims, src, tgt, raylen, shift, eps) of a named case."""
    kind, _, arg = name.partition(":")
    shift = 0.0 if arg.endswith("s0") else 0.5
    if kind in ("inside", "miss"):
        dims, H, W, B = tc.SHAPE_A if arg == "" else tc.SHAPE_THIN
        return (dims,) + getattr(tc, kind)(dims, H, W, B, seed=2) + (0.5, 1e-8)
    if kind == "cone":   # the pose-in cones of test_gpu_siddon_oracle.py, as the ray tensors the GPU test gives every kernel
        geom, shape = arg.split("/")
        dims, H, W, B = dict(A4=sc.SHAPE_A4, brick=sc.SHAPE_BRICK_ROUTE, sliver=tc.SHAPE_SLIVER)[shape]
        src, G, Wd, rows, cols, t64, l64, _ = sc.cone_pose(geom, dims, H, W, B)
        return dims, src, t64.astype(np.float32), l64.astype(np.float32), 0.5, 1e-8
    if kind == "near_identical":
        dims, H, W, B = sc.SHAPE_NEAR
        return (dims,) + tc.near_identical(dims, H, W, B, seed=2) + (0.5, 1e-8)
    if kind == "axis":
        dims, H, W, _ = tc.SHAPE_SLIVER if arg.startswith("sliver") else tc.SHAPE_A
        return (dims,) + tc.axis(dims, H, W, shift) + (shift, 1e-8)
    if kind == "planar":
        dims, H, W, _ = tc.SHAPE_THIN if arg.startswith("thin") else sc.SHAPE_A4
        face = float(arg.split("/")[1])
        return (dims,) + sc.planar_axis(dims, H, W, face, shift) + (shift, 1e-8)
    if kind == "lattice":
        dims = sc.LATTICE_DIMS[int(arg)]
        return (dims,) + sc.lattice_ties(dims, 512, seed=int(arg))[:3] + (0.5, 0.0)
    if kind == "lattice_rays":
        dims = sc.LATTICE_DIMS[int(arg)]
        return (dims,) + sc.lattice_rays(dims, 1000, seed=int(arg)) + (0.5, 0.0)
    raise KeyError(name)


ORDINARY = ["inside", "miss", "inside:thin", "miss:thin", "near_identical", "cone:rotated/A4", "cone:inside/A4", "cone:rotated/sliver"]
BRICK_ROUTE = "cone:rotated/brick"   # 384 x 352 x 384 voxels, sources ~1000 voxels out: see the fraction test
PLANAR = [f"planar:A4/{f}" for f in sc.planar_faces(DIMS_A4)] + [f"planar:thin/{f}" for f in sc.planar_faces(tc.SHAPE_THIN[0])]
EDGES = ["axis:A", "axis:A/s0", "axis:sliver", "axis:sliver/s0"] + PLANAR + [p + "/s0" for p in PLANAR[:2]]
TIES = [f"lattice:{i}" for i in range(3)] + [f"lattice_rays:{i}" for i in range(3)]


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """fp64 and fp32 oracle on a named case with gout = 1: images (B, N), g_target (B, N, 3), g_raylen (B, N), g_volume, and the
    per-ray source gradients (each ray run as its own pose), plus the ray classes."""
    dims, src, tgt, raylen, shift, eps = _geometry(name)
    vol = tc.volume(dims)
    B, N = tgt.shape[:2]
    out = {}
    kw = dict(voxel_shift=shift, eps=eps)
    srcr = np.repeat(src, N, axis=0)                    # (B*N, 3): per-ray source gradients
    for dt in (np.float64, np.float32):
        img = oracle.siddon_fwd(vol, src[:, None], tgt, raylen[:, None], dtype=dt, **kw).reshape(B, N)
        g = oracle.siddon_bwd(vol, src[:, None], tgt, raylen[:, None], np.ones((B, 1, N)), dtype=dt, **kw)
        gr = oracle.siddon_bwd(vol, srcr[:, None], tgt.reshape(B * N, 1, 3), raylen.reshape(B * N, 1, 1), np.ones((B * N, 1, 1)),
                               dtype=dt, want_vol=False, **kw)
        out[dt] = dict(img=img, g_target=g["g_target"].reshape(B, N, 3), g_raylen=g["g_raylen"].reshape(B, N),
                       g_volume=g["g_volume"], g_src_ray=gr["g_source"].reshape(B, N, 3))
    return vol, out[np.float64], out[np.float32], sc.classify(dims, src, tgt, shift, eps)


def _disagree(a, b, ref):
    """Per-ray error over the reference's max-abs: (B, N)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    e = np.abs(a - b)
    if e.ndim == 3:
        e = e.max(-1)
    return e / max(np.abs(ref).max(), 1e-30)


# ---- the geometries -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shift", [0.5, 0.0])
@pytest.mark.parametrize("shape", [sc.SHAPE_A4, tc.SHAPE_THIN])
def test_planar_axis_rows_lie_in_the_named_faces_and_the_grid_is_affine(shape, shift):
    dims, H, W, _ = shape
    faces = sc.planar_faces(dims)
    assert -0.5 in faces and (dims[0] < 16 or 15.5 in faces) and (dims[0] < 24 or 23.5 in faces)
    for face in faces:
        src, tgt, _ = sc.planar_axis(dims, H, W, face, shift)
        t = tgt[0].reshape(H, W, 3).astype(np.float64)
        s = src[0].astype(np.float64)
        assert tc.pix(src[0, 0], shift) == np.float32(face)
        f2 = tc.pix(src[0, 2], shift)
        assert f2 - np.floor(f2) == 0.5 and -0.5 <= f2 <= dims[2] - 0.5          # axis-2 face inside the volume
        assert (t[H // 2, :, 0] - s[0] == 0.0).all() and (t[:, W // 2, 2] - s[2] == 0.0).all()
        assert (np.abs(t[..., 0] - s[0])[np.arange(H) != H // 2] > 0).all()
        # affine in (h, w): the grid rebuilt from pixels (0,0), (0,W-1), (H-1,0) matches every pixel to fp32 rounding
        hh, ww = np.meshgrid(np.arange(H) / (H - 1), np.arange(W) / (W - 1), indexing="ij")
        rebuilt = t[0, 0] + hh[..., None] * (t[H - 1, 0] - t[0, 0]) + ww[..., None] * (t[0, W - 1] - t[0, 0])
        assert np.abs(rebuilt - t).max() <= 4 * np.spacing(np.float32(np.abs(t).max()))
        _pose_rays_exact_in_fp32(*sc.grid_matrices(src, tgt, H, W), tgt)
        cls = sc.classify(dims, src, tgt, shift)
        on = cls["on_face"].reshape(H, W)
        assert on[H // 2].sum() >= W // 2 and on[:, W // 2].sum() >= H // 2   # the face row and column hit the volume
        assert not cls["near_face"].any()


def _pose_rays_exact_in_fp32(G, Wd, rows, cols, tgt):
    """G (cols[w], rows[h], 1, 1) evaluated in fp32 in two orders of operations, with every product and partial sum rounded,
    equals the fp32 ray targets: the pose-in kernels generate exactly these rays."""
    G = np.asarray(G, np.float32)
    H, W = len(rows), len(cols)
    c = np.asarray(cols, np.float32)[None, None, :, None]
    r = np.asarray(rows, np.float32)[None, :, None, None]
    g = [G[:, None, None, :, k] for k in range(4)]
    one = (g[0] * c + g[1] * r) + (g[2] + g[3])
    two = ((g[3] + g[2]) + g[1] * r) + g[0] * c
    for t in (one, two):
        assert t.dtype == np.float32 and (t.reshape(len(G), H * W, 3) == tgt).all()


@pytest.mark.parametrize("kind", ["rotated", "inside"])
@pytest.mark.parametrize("shape", [sc.SHAPE_A4, sc.SHAPE_BRICK_ROUTE, tc.SHAPE_SLIVER])
def test_cone_pose_matrices_are_exact_in_fp32(shape, kind):
    dims, H, W, B = shape
    src, G, Wd, rows, cols, t64, l64, _ = sc.cone_pose(kind, dims, H, W, B)
    _pose_rays_exact_in_fp32(G, Wd, rows, cols, t64.astype(np.float32))
    assert (t64.astype(np.float32) == t64).all()


@pytest.mark.parametrize("dims", sc.LATTICE_DIMS + ((128, 64, 64), (512, 512, 256)))
def test_lattice_ties_are_exact_affine_and_tie_on_two_and_three_axes(dims):
    i = 1
    src, tgt, raylen, G, Wd, rows, cols = sc.lattice_ties(dims, 512, seed=i)
    _pose_rays_exact_in_fp32(G, Wd, rows, cols, tgt)
    d = tgt.astype(np.float64) - src[:, None, :].astype(np.float64)
    assert set(np.abs(d).ravel()) <= set(sc.LATTICE_D)                   # power-of-two components, eps = 0
    t64, l64, _ = sc.pose_rays(G, Wd, rows, cols)
    assert (t64 == tgt).all() and np.allclose(l64, raylen, rtol=1e-6)      # the pose matrices give the same rays, exactly
    assert (tgt[:, 0] + tgt[:, 3] == tgt[:, 1] + tgt[:, 2]).all()          # 2 x 2 affine
    assert ((4 * src) == np.round(4 * src)).all()                          # quarter-voxel lattice (shift 0.5: x = pix)
    ties2 = ties3 = 0
    for b in range(len(src)):
        for n in range(4):
            al = {}
            for a in range(3):
                p32 = ((np.arange(dims[a] + 1, dtype=np.float32) - np.float32(0.5)) - src[b, a]) / np.float32(d[b, n, a])
                p64 = ((np.arange(dims[a] + 1) - 0.5) - np.float64(src[b, a])) / d[b, n, a]
                assert (p32.astype(np.float64) == p64).all()                     # every plane alpha exact in fp32
                x = src[b].astype(np.float64)[None, :] + p64[:, None] * d[b, n][None, :]
                inb = np.all((x >= -0.5) & (x <= np.asarray(dims) - 0.5), axis=1)
                al[a] = set(p64[inb])
            ties2 += len((al[0] & al[1]) | (al[0] & al[2]) | (al[1] & al[2]))
            ties3 += len(al[0] & al[1] & al[2])
    assert ties2 >= 200 and ties3 >= 20, (ties2, ties3)


# ---- the classes cover what the oracle cannot resolve, and little else -------------------------------------------------------------
@pytest.mark.parametrize("name", ORDINARY + EDGES + [BRICK_ROUTE])
def test_classes_cover_every_ray_the_oracle_disagrees_with_itself_on(name):
    """Every ray on which the oracle's fp32 and fp64 differ by more than 1e-5 of the maximum is excluded: near-face for images,
    g_raylen and g_volume; near-face or near-tie for end-point gradients.  How many rays that excludes: the next test."""
    dims, src, tgt, raylen, shift, eps = _geometry(name)
    vol, r64, r32, cls = _oracle(name)
    ex_img, ex_end = sc.excluded(cls, "image"), sc.excluded(cls, "g_target")
    for k in ("img", "g_raylen"):
        bad = _disagree(r32[k], r64[k], r64[k]) > 1e-5
        assert not (bad & ~ex_img).any(), (k, np.argwhere(bad & ~ex_img)[:5])
    for k in ("g_target", "g_src_ray"):
        bad = _disagree(r32[k], r64[k], r64[k]) > 1e-5
        assert not (bad & ~ex_end).any(), (k, np.argwhere(bad & ~ex_end)[:5])
    # g_volume with gout zeroed on near-face rays
    B, N = tgt.shape[:2]
    g = (~ex_img).astype(np.float64).reshape(B, 1, N)
    gv = [oracle.siddon_bwd(vol, src[:, None], tgt, raylen[:, None], g, dtype=dt, voxel_shift=shift, eps=eps)["g_volume"]
          for dt in (np.float64, np.float32)]
    assert relerr(gv[1], gv[0]) < 5e-4      # the fp32 accumulation of the scatter (1.2e-4 on the brick-route volume)
    if name in ORDINARY + [BRICK_ROUTE]:
        assert not cls["near_face"].any()


@pytest.mark.parametrize("name", ORDINARY + [BRICK_ROUTE])
def test_excluded_fraction(name):
    """The end-point gradients' excluded class stays within 2 % of the rays on the ordinary geometries and within 30 % on the
    brick-route volume, where sources ~1000 voxels out put the fp32 position error of a crossing near 1e-4 voxel and ~1100
    crossings per ray make close pairs common: there the oracle itself disagrees with its fp64 on 2 % of the rays.  The GPU test
    still pins every excluded ray, against the un-cut walk."""
    _, r64, r32, cls = _oracle(name)
    ex = sc.excluded(cls, "g_target")
    bound = 0.3 if name == BRICK_ROUTE else 0.02
    bad = _disagree(r32["g_target"], r64["g_target"], r64["g_target"]) > 1e-5
    print(f"{name}: excluded {ex.mean():.4f}, oracle fp32 unresolved {bad.mean():.4f}")
    assert ex.mean() <= bound, ex.mean()


@pytest.mark.parametrize("name", ORDINARY + EDGES + TIES)
def test_per_ray_telescoping_identities(name):
    """sum_a dI/dt_a d_a = -I (ray length held fixed) and sum_a (dI/ds_a + dI/dt_a) d_a = 0 (the whole line is integrated, quirk
    Q1), per ray, for the fp64 oracle: any order of tied crossings satisfies both."""
    dims, src, tgt, raylen, shift, eps = _geometry(name)
    _, r64, _, _ = _oracle(name)
    d = tgt.astype(np.float64) - src[:, None, :].astype(np.float64) + eps
    scale = np.abs(r64["img"]).max()
    e1 = np.abs((r64["g_target"] * d).sum(-1) + r64["img"]) / scale
    e2 = np.abs(((r64["g_target"] + r64["g_src_ray"]) * d).sum(-1)) / scale
    assert e1.max() < 1e-9 and e2.max() < 1e-9, (e1.max(), e2.max())


# ---- exact ties: an exact reference for the image, g_raylen and g_volume; the kernels' convention by consistency ----------------
@pytest.mark.parametrize("name", TIES)
def test_lattice_oracle_is_exact_and_the_emulated_walk_matches_it(name):
    """fp32 and fp64 oracles agree per ray to 1e-6.  The host emulation of the kernels' walk -- un-cut, cut into slabs and major-axis
    pieces, cut into bricks, and the two-walk backward -- matches the oracle's image, g_raylen and g_volume, and every cut matches
    the un-cut walk per ray, end-point gradients included (the tie convention: lowest axis first)."""
    from hostemu import emu, emu_brick_sens
    dims, src, tgt, raylen, shift, eps = _geometry(name)
    vol, r64, r32, _ = _oracle(name)
    B, N = tgt.shape[:2]
    for k in ("img", "g_raylen", "g_target", "g_src_ray"):
        assert _disagree(r32[k], r64[k], r64[k]).max() < 1e-6, k
    assert relerr(r32["g_volume"], r64["g_volume"]) < 1e-6
    args = (vol, src[:, None], tgt, raylen[:, None], np.ones((B, 1, N), np.float32))
    whole = emu.siddon_sens(*args, eps=eps, slab=0)
    assert _disagree(whole["img"].reshape(B, N), r64["img"], r64["img"]).max() < 1e-6
    assert _disagree(whole["g_raylen"].reshape(B, N), r64["g_raylen"], r64["g_raylen"]).max() < 1e-6
    cuts = [emu.siddon_sens(*args, eps=eps, slab=s) for s in (-4, 3, 16)]
    cuts.append(emu_brick_sens.siddon_sens_brick(*args, eps=eps, brick=(3, 4, 4)))
    cuts.append(emu_brick_sens.siddon_sens_brick(*args, eps=eps, brick=(24, 32, 32)))
    for c in cuts:
        for k in ("img", "g_target", "g_raylen"):
            ref = whole[k].reshape(B, N, -1)
            assert _disagree(c[k].reshape(B, N, -1), ref, ref).max() < 1e-6, k
        assert relerr(c["g_source"], whole["g_source"]) < 1e-6
    bwd = emu.siddon_bwd(*args, eps=eps)
    assert relerr(bwd["g_volume"], r64["g_volume"]) < 1e-6
    assert _disagree(bwd["g_raylen"].reshape(B, N), r64["g_raylen"], r64["g_raylen"]).max() < 1e-6
    ref = whole["g_target"]
    assert _disagree(bwd["g_target"], ref, ref).max() < 1e-6               # two-walk backward: the same tie convention
