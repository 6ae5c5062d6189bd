"""Named ray geometries, ray classes and the tolerance rule of the Siddon oracle tests (test_gpu_siddon_oracle.py); what each
geometry claims to be, and that the classes cover every ray the oracle cannot resolve in fp32, is checked on the CPU by
test_siddon_cases_cpu.py.  Shares the volumes, geometries and the SURVEY 8c rule of trilinear_cases.py.  Rays are in voxel-index
space: src (B, 3), tgt (B, N, 3), raylen (B, N), all fp32 numpy; N = H * W in row-major detector order.

Siddon's image is continuous in the geometry except on rays that run in a voxel face; its end-point gradients jump wherever two
plane crossings of different axes swap order (a crossing coefficient moves from one axis to the other).  So rays are classed from
the geometry alone, in fp64:
  on-face    a direction component is exactly 0 and the source lies exactly on a voxel face of that axis: well defined (the
             +eps tilt of the direction picks the side) and compared like every other ray;
  near-face  the ray runs within FACE_TOL voxel of a face without being on it: fp32 round-off picks the side, so its image and
             every gradient are ill-conditioned;
  near-tie   two crossings of different axes lie closer along the ray than their fp32 position error (classify), exact
             ties included: the image is continuous there but the end-point gradients are a convention of the walk's order."""
import numpy as np

import trilinear_cases as tc
from trilinear_cases import TOL_CAP, inside, miss, near_identical, volume  # noqa: F401  (the shared geometries and cap)

FACE_TOL = 1e-3      # voxels: a near-face ray runs this close to a face along its whole path through the volume
# crossing position error bound: TIE_ULPS x 2^-24 of the crossing's distance from the source plus TIE_ULPS_PLANE x 2^-24 of the
# plane coordinate over the axis' share of the direction.  A small pair that still covers, with some margin, every ray on which
# the oracle's own fp32 and fp64 end-point gradients differ, on every geometry of test_siddon_cases_cpu.py (rotated poses of the
# brick-route volume included)
TIE_ULPS = 4.0
TIE_ULPS_PLANE = 3.0
LATTICE_D = (32.0, 64.0, 128.0)   # |direction components| of the lattice geometry: every plane alpha is a dyadic rational

# (dims, H, W, B): a twin of trilinear_cases.SHAPE_A that the brick kernels take (D2 % 4 == 0, a partial 24 x 32 x 32 brick on
# every axis), a volume large enough for the sensitivities walk's brick route (>= 2048 bricks), and the scatter-contention cube
SHAPE_A4 = ((97, 130, 60), 37, 53, 3)
SHAPE_BRICK_ROUTE = ((384, 352, 384), 45, 61, 4)
SHAPE_NEAR = ((32, 32, 32), 128, 128, 16)
LATTICE_DIMS = ((16, 32, 8), (32, 16, 64), (8, 8, 8))


def siddon_tol(err32, floor):
    """The SURVEY 8c rule on the well-conditioned rays: max(floor, 2 x the oracle's own fp32-vs-fp64 error there), capped at
    TOL_CAP.  err32 is that error, measured per ray over the rays the comparison keeps."""
    t = max(floor, 2.0 * float(err32))
    assert np.isfinite(err32) and t <= TOL_CAP, (t, floor)
    return t


def per_ray_err(got, ref, keep=None, scale=None):
    """Largest per-ray error over the kept rays, relative to the reference's max-abs over them (or `scale`).  got / ref are
    (B, N) or (B, N, k)."""
    g = np.asarray(got, np.float64)
    r = np.asarray(ref, np.float64)
    B, N = r.shape[:2]
    g, r = g.reshape(B * N, -1), r.reshape(B * N, -1)
    if keep is not None:
        k = np.asarray(keep, bool).reshape(B * N)
        g, r = g[k], r[k]
    if r.size == 0:
        return 0.0
    s = np.abs(r).max() if scale is None else scale
    return float(np.abs(g - r).max() / max(float(s), 1e-30))


# ---- geometries ---------------------------------------------------------------------------------------------------------------------
def planar_faces(dims):
    """Voxel faces (in pix = x + shift - 0.5) on axis 0 for planar_axis: an interior face 7.5, the 16-plane slab face 15.5, the
    24-voxel brick face 23.5, the lower face -0.5 and the upper face D0 - 0.5; only those the volume has are kept.  A ray in a
    face samples the voxel on the side of the +eps tilt of its direction, and the oracle's fp32 nearest lookup (round half to
    even at the face's midpoints) lands on that side only where face + 0.5 is even, so only such faces are named: on the others
    the fp32 oracle is no reference for the fp64 one (the upper face of an odd-sided volume is one)."""
    D0 = dims[0]
    return [f for f in dict.fromkeys((7.5, 15.5, 23.5, -0.5, D0 - 0.5)) if -0.5 <= f <= D0 - 0.5 and (f + 0.5) % 2 == 0]


def planar_axis(dims, H, W, face, shift=0.5):
    """One pose: the detector is perpendicular to axis 1 and affine in (h, w) (the brick kernels rebuild it from three corners); its
    row H // 2 has targets with the source's axis-0 coordinate, its column W // 2 the source's axis-2 coordinate.  The source lies
    on the face pix0 = `face` and on an axis-2 face near the volume's middle, so row H // 2 lies in a voxel face of axis 0, column
    W // 2 in one of axis 2, and their pixel on a voxel edge; every other ray is oblique.  Every coordinate and step is a multiple
    of 2^-6 with a few significant bits, so t(h, w) = t(0, 0) + h dv + w du is exact in fp32 whatever the order of operations: the
    pose-in kernels, given the matrices of the same grid (grid_matrices), generate exactly these targets.
    -> src (1, 3), tgt (1, H*W, 3), raylen (1, H*W)."""
    D = np.asarray(dims, np.float64)
    f2 = 2.0 * np.floor((D[2] - 1) / 4) + 1.5                     # face + 0.5 even (planar_faces)
    s = np.array([face + 0.5 - shift, -0.5 * D[1] - 9.375, f2 + 0.5 - shift])
    h = np.arange(H, dtype=np.float64)[:, None] - H // 2
    w = np.arange(W, dtype=np.float64)[None, :] - W // 2
    step0 = _q(1.6 * np.sqrt(2.0) * max(D[0], 4.0) / H, 6)          # rows span ~2.3 D0 on axis 0, columns ~2.3 D2 on axis 2
    step2 = _q(1.6 * np.sqrt(2.0) * D[2] / W, 6)
    t = np.empty((H, W, 3))
    t[..., 0] = s[0] + step0 * h + 0.0 * w
    t[..., 1] = 1.5 * D[1] + 10.765625 + 0.015625 * h + 0.0078125 * w   # a slight tilt: rows do not share one axis-1 direction
    t[..., 2] = s[2] + step2 * w + 0.0 * h
    return tc._finish([s], [t.reshape(H * W, 3)])


def _q(x, bits):
    """x rounded to a multiple of 2^-bits."""
    return np.round(np.asarray(x, np.float64) * 2.0 ** bits) / 2.0 ** bits


def grid_matrices(src, tgt, H, W):
    """Pose-in matrices of an affine H x W grid with rows = h, cols = w: G from pixels (0,0), (0,W-1), (H-1,0)."""
    t = np.asarray(tgt, np.float64).reshape(len(src), H, W, 3)
    du, dv = (t[:, 0, -1] - t[:, 0, 0]) / max(W - 1, 1), (t[:, -1, 0] - t[:, 0, 0]) / max(H - 1, 1)
    z = np.zeros_like(du)
    G = np.stack([du, dv, t[:, 0, 0], z], -1).astype(np.float32)
    Wd = np.stack([du, dv, t[:, 0, 0] - np.asarray(src, np.float64), z], -1).astype(np.float32)
    return G, Wd, np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32)


def _lattice_steps():
    """(a, b, c) with a, a + b, a + c, a + b + c all in +-LATTICE_D: one direction component of a 2 x 2 affine detector
    (d(h, w) = a + h b + w c) whose four rays all have power-of-two components."""
    S = [s * v for v in LATTICE_D for s in (1.0, -1.0)]
    return [(a, y - a, z - a) for a in S for y in S for z in S if (y + z - a) in S]


def lattice_ties(dims, B, seed=0, shift=0.5):
    """Exact ties: power-of-two dims, B poses with sources on the quarter-voxel lattice in and around the volume and a 2 x 2 affine
    detector whose four direction vectors have components +-32 / 64 / 128.  With eps = 0 every plane alpha, every midpoint and
    every grid_sample coordinate is exact in fp32, and many rays pass exactly through voxel edges and corners (crossings of two
    and three axes at one alpha).  -> src (B, 3), tgt (B, 4, 3), raylen (B, 4), and the pose matrices of the same rays
    (G, Wd (B, 3, 4), rows, cols (2,)): target = G (cols[w], rows[h], 1, 1), target - source = Wd (cols[w], rows[h], 1, 1)."""
    assert all(d & (d - 1) == 0 for d in dims), dims
    rng = np.random.default_rng(seed)
    steps = np.array(_lattice_steps())
    D = np.asarray(dims, np.float64)
    pix = np.floor(rng.uniform(-1.0, D[None, :], size=(B, 3)) * 4.0) / 4.0
    s = pix + 0.5 - shift
    abc = steps[rng.integers(0, len(steps), size=(B, 3))]          # (B, axis, (a, b, c))
    a, bv, cu = abc[..., 0], abc[..., 1], abc[..., 2]
    hw = np.array([(0, 0), (0, 1), (1, 0), (1, 1)], np.float64)   # row-major (h, w)
    d = a[:, None, :] + hw[None, :, 0:1] * bv[:, None, :] + hw[None, :, 1:2] * cu[:, None, :]
    src, tgt, raylen = tc._finish(s, s[:, None, :] + d)
    z = np.zeros((B, 3))
    G = np.stack([cu, bv, s + a, z], -1).astype(np.float32)        # p = (cols[w], rows[h], 1, 1) with cols = rows = (0, 1)
    Wd = np.stack([cu, bv, a, z], -1).astype(np.float32)
    axes = np.array([0.0, 1.0], np.float32)
    return src, tgt, raylen, G, Wd, axes, axes


def lattice_rays(dims, n, seed=0, shift=0.5):
    """The ray-set form of lattice_ties: one ray per pose (src (n, 3), tgt (n, 1, 3), raylen (n, 1)), each through a lattice
    point of the volume (as test_brick_sens_cpu.py), so nearly every ray passes through a voxel edge or corner."""
    rng = np.random.default_rng(seed)
    D = np.asarray(dims, np.float64)
    d = rng.choice(LATTICE_D, size=(n, 3)) * rng.choice([-1.0, 1.0], size=(n, 3))
    through = np.floor(rng.uniform(0.0, D + 1.0, size=(n, 3))) - 0.5            # a voxel corner (pix), inside the closed box
    through += rng.choice([0.0, 0.0, 0.25, 0.5], size=(n, 1)) * rng.choice([0.0, 1.0], size=(n, 3))
    s = through - d * rng.integers(1, 4, size=(n, 1)) * 0.25 + 0.5 - shift
    src, tgt, raylen = tc._finish(s, (s + 2.0 * d)[:, None, :])
    return src, tgt, raylen


def pose_matrices(src, centre, u, v, H, W):
    """Pose-in inputs of a cone detector (trilinear_cases._cone): target = G (cols[w], rows[h], 1, 1), target - source = Wd (...),
    rows / cols ~ linspace(-1, 1).  -> G, Wd (B, 3, 4), rows (H,), cols (W,) fp32, and the fp64 targets / ray lengths they define.
    G's entries are multiples of 2^-4 below 2^11 and rows / cols multiples of 2^-6 in [-1, 1], so G p is exact in fp32 in any
    order of operations: the pose-in kernels generate exactly the fp32 targets the ray-tensor kernels are given, and the un-cut
    walk on those ray tensors is a reference for their per-ray gradients on near-tie rays."""
    src, centre, u, v = (np.asarray(x, np.float64) for x in (src, centre, u, v))
    u, v, centre = _q(u, 4), _q(v, 4), _q(centre, 4)
    assert np.abs(centre).max() + np.abs(u).max() + np.abs(v).max() < 2.0 ** 11
    z = np.zeros_like(src)
    G = np.stack([u, v, centre, z], -1).astype(np.float32)
    Wd = np.stack([u, v, centre - src, z], -1).astype(np.float32)
    rows, cols = (_q(np.linspace(-1.0, 1.0, n), 6).astype(np.float32) for n in (H, W))
    return (G, Wd, rows, cols) + pose_rays(G, Wd, rows, cols)


def pose_rays(G, Wd, rows, cols):
    """fp64 targets (B, H*W, 3), ray lengths (B, H*W) and the detector coordinates p (H*W, 4) of pose-in matrices."""
    H, W = len(rows), len(cols)
    p = np.stack(np.broadcast_arrays(np.asarray(cols, np.float64)[None, :], np.asarray(rows, np.float64)[:, None],
                                     np.ones((1, 1)), np.ones((1, 1))), -1).reshape(H * W, 4)
    tgt = np.einsum("bij,nj->bni", np.asarray(G, np.float64), p)
    dl = np.einsum("bij,nj->bni", np.asarray(Wd, np.float64), p)
    return tgt, np.linalg.norm(dl, axis=-1), p


def cone_pose(geom, dims, H, W, B, seed=2):
    """Pose-in twins of trilinear_cases.inside / miss / near_identical-like cones: (src fp32 (B, 3), G, Wd, rows, cols,
    tgt64, raylen64, p)."""
    rng = np.random.default_rng(seed)
    D = np.asarray(dims, np.float64)
    diag, centre = float(np.linalg.norm(D)), (D - 1) / 2
    srcs, cs, us, vs = [], [], [], []
    for _ in range(B):
        d, u, v = tc._frame(rng)
        if geom == "inside":
            s = (0.25 + 0.5 * rng.random(3)) * (D - 1)
            c, u, v = s + 1.5 * diag * d, 0.9 * diag * u, 0.7 * diag * v
        else:   # "rotated": source outside, the volume filling most of the detector
            s = centre - 1.6 * diag * d
            c, u, v = centre + 0.6 * diag * d, 0.45 * diag * u, 0.4 * diag * v
        srcs.append(s)
        cs.append(c)
        us.append(u)
        vs.append(v)
    src = np.asarray(srcs, np.float32)
    return (src,) + pose_matrices(src, cs, us, vs, H, W)


# ---- ray classes ------------------------------------------------------------------------------------------------------------------
def _box_range(s, d, dims, shift, skip=None):
    """alpha interval over which the line lies in the closed box of the voxel faces (x in [-shift, D - shift]) on every axis but
    `skip`; (B, N) each, empty where lo > hi."""
    lo = np.full(d.shape[:2], -np.inf)
    hi = np.full(d.shape[:2], np.inf)
    for a in range(3):
        if a == skip:
            continue
        with np.errstate(divide="ignore", invalid="ignore"):
            a0 = (-shift - s[..., a]) / d[..., a]
            a1 = (dims[a] - shift - s[..., a]) / d[..., a]
        inside = (s[..., a] >= -shift) & (s[..., a] <= dims[a] - shift)
        par = d[..., a] == 0
        lo = np.where(par, np.where(inside, lo, np.inf), np.maximum(lo, np.minimum(a0, a1)))
        hi = np.where(par, np.where(inside, hi, -np.inf), np.minimum(hi, np.maximum(a0, a1)))
    return lo, hi


def classify(dims, src, tgt, shift=0.5, eps=1e-8, chunk=4096):
    """Ray classes from the geometry alone, in fp64 of the fp32 inputs (module docstring).  -> dict of (B, N) bool arrays
    on_face, near_face, near_tie, and min_gap (B, N): the smallest distance along the ray, in voxels, between consecutive
    crossings of different axes inside the volume, over its bound (near_tie = min_gap < 1)."""
    dims = tuple(int(x) for x in dims)
    s = np.asarray(src, np.float64).reshape(-1, 1, 3)
    t = np.asarray(tgt, np.float64)
    B, N = t.shape[:2]
    s = np.broadcast_to(s, (B, 1, 3))
    draw = t - s                                          # exact: fp32 differences fit in fp64
    d = draw + eps
    on_face = np.zeros((B, N), bool)
    near_face = np.zeros((B, N), bool)
    for a in range(3):
        p = s[..., a] + shift - 0.5                        # pix of the source on axis a
        f = np.clip(np.round(p - 0.5) + 0.5, -0.5, dims[a] - 0.5)   # nearest voxel face
        lo, hi = _box_range(s, d, dims, shift, skip=a)
        hits = lo <= hi
        reach = np.where(hits, np.maximum(np.abs(np.where(hits, lo, 0)), np.abs(np.where(hits, hi, 0))), 0.0)
        drift = np.abs(p - f) + np.abs(d[..., a]) * reach   # how far from the face the ray gets inside the volume
        exact = (draw[..., a] == 0) & (p == f)
        on_face |= exact & hits
        near_face |= (drift < FACE_TOL) & hits & ~exact
    min_gap = np.full(B * N, np.inf)
    sf, df = np.broadcast_to(s, (B, N, 3)).reshape(-1, 3), d.reshape(-1, 3)
    nd = np.linalg.norm(df, axis=1)
    M = sum(dims) + 3
    for r0 in range(0, B * N, chunk):
        sl = slice(r0, min(B * N, r0 + chunk))
        ss, dd, nn = sf[sl], df[sl], nd[sl]
        R = len(ss)
        alpha = np.empty((R, M))
        err = np.empty((R, M))
        axis = np.empty((R, M), np.int8)
        k = 0
        for a in range(3):
            plane = np.arange(dims[a] + 1, dtype=np.float64) - shift
            with np.errstate(divide="ignore", invalid="ignore"):
                al = (plane[None, :] - ss[:, a:a + 1]) / dd[:, a:a + 1]
                # fp32 position error of this crossing along the ray: alpha = (plane - s) / d carries three roundings (the
                # numerator's, the direction's, the quotient's), each relative to alpha, so the crossing moves by a few 2^-24 of
                # its distance from the source; the sample coordinate of a segment between two crossings is rounded at the
                # scale of the plane's own coordinate, which moves it along the ray by that over the axis' share of the direction
                e = 2.0 ** -24 * (TIE_ULPS * np.abs(al) * nn[:, None]
                                  + TIE_ULPS_PLANE * (np.abs(plane)[None, :] + 1.0) * (nn / np.abs(dd[:, a]))[:, None])
            n = dims[a] + 1
            alpha[:, k:k + n], err[:, k:k + n], axis[:, k:k + n] = al, e, a
            k += n
        # only crossings on the closed volume box change the sampled voxel (with a margin: one just outside ties with a face)
        x = ss[:, None, :] + np.where(np.isfinite(alpha), alpha, 0.0)[..., None] * dd[:, None, :]
        inbox = np.isfinite(alpha) & np.all((x >= -shift - FACE_TOL) & (x <= np.asarray(dims) - shift + FACE_TOL), axis=-1)
        alpha = np.where(inbox, alpha, np.inf)
        order = np.argsort(alpha, axis=1, kind="stable")
        al = np.take_along_axis(alpha, order, 1)
        ax = np.take_along_axis(axis, order, 1)
        er = np.take_along_axis(err, order, 1)
        # consecutive crossings suffice: between two crossings of different axes lies a consecutive pair of different axes
        valid = np.isfinite(al[:, 1:]) & (ax[:, 1:] != ax[:, :-1])
        gap = (al[:, 1:] - np.where(np.isfinite(al[:, :-1]), al[:, :-1], 0.0)) * nn[:, None]
        with np.errstate(invalid="ignore", divide="ignore"):
            ratio = np.where(valid, gap / (er[:, 1:] + er[:, :-1]), np.inf)
        min_gap[sl] = ratio.min(axis=1)
    min_gap = min_gap.reshape(B, N)
    return dict(on_face=on_face, near_face=near_face, near_tie=min_gap < 1.0, min_gap=min_gap)


def excluded(cls, quantity):
    """Rays a comparison with the fp64 oracle leaves out: near-face for images, g_raylen and g_volume; near-face and near-tie for
    end-point gradients."""
    ex = cls["near_face"].copy()
    if quantity in ("g_target", "g_source", "sens"):
        ex |= cls["near_tie"]
    return ex
