"""Named ray geometries and the SURVEY 8c tolerance rule of the trilinear oracle tests (test_gpu_trilinear_oracle.py); what each
geometry claims to be is checked on the CPU by test_trilinear_cases_cpu.py.  Rays are in voxel-index space (what the kernels
and the oracle take): src (B, 3), tgt (B, N, 3), raylen (B, N), all fp32 numpy; N = H * W in row-major detector order."""
import numpy as np

from conftest import relerr

TOL_CAP = 5e-3   # no tolerance derived by the 8c rule may exceed this: a degenerate case must not quietly loosen a bound

# (dims, H, W, B): detector sides that are not multiples of the 16-pixel tiles, odd volume sides
SHAPE_A = ((97, 130, 61), 37, 53, 3)
SHAPE_THIN = ((2, 180, 160), 45, 67, 2)
SHAPE_SLIVER = ((1, 64, 48), 29, 35, 2)
PARTIAL_TILE_SHAPES = (SHAPE_A, SHAPE_THIN, SHAPE_SLIVER, ((256, 256, 256), 200, 200, 4))


def tol(f32, f64, floor, scale=None):
    """SURVEY 8c: max(floor, 2 x the oracle's own fp32-vs-fp64 error); capped so a degenerate case fails instead.  Errors are
    max-abs over the reference's max-abs, or over `scale` where given (alpha_scale)."""
    err = relerr(f32, f64) if scale is None else np.abs(np.subtract(f32, f64)).max() / scale
    t = max(floor, 2.0 * err)
    assert np.isfinite(err) and t <= TOL_CAP, (t, floor)
    return t


def alpha_scale(g_raylen, raylen, amin, amax):
    """Size of the terms the range partials sum: d/d alphamin = sum_rays g L [-sum V / (P-1) + step sum (1-lin) G.dp], and the
    first term alone is g_raylen L / (amax - amin) per ray.  The partials themselves nearly cancel (the image changes with the
    range only through the samples at its ends), so errors are measured against this scale, not against their own size."""
    s = np.abs(np.asarray(g_raylen, np.float64).reshape(-1) * np.asarray(raylen, np.float64).reshape(-1)).sum() / (amax - amin)
    return max(float(s), 1e-30)   # no sampled value at all: any difference from the reference then fails


def volume(dims):
    """The smooth test volume (synthetic "smooth": two Gaussian blobs) tapered by sin^2 to zero at its faces, so that the zero
    padding adds no edge either: end-point gradients of rays that graze a face stay as well conditioned as the interior."""
    from diffdrr_b200 import synthetic
    vol = synthetic.make_volume(dims, "smooth", seed=4).astype(np.float64)
    for a, n in enumerate(dims):
        w = np.sin(np.pi * (np.arange(n) + 1.0) / (n + 1.0)) ** 2
        vol *= w.reshape([-1 if i == a else 1 for i in range(3)])
    return vol.astype(np.float32)


def alpha_partials_f32(vol, src, tgt, raylen, gout, chunk=256, mask=None, **kw):
    """The oracle's fp32 d/d(alphamin, alphamax), summed per pose over chunks of `chunk` rays and then in fp64 -- the reduction
    structure of the kernels (a block sum per CTA, atomics across CTAs) -- instead of one serial fp32 sum over every ray of the
    batch, whose round-off grows with the ray count and says nothing about the per-ray math."""
    from oracle import oracle
    B, N = tgt.shape[:2]
    gout = gout.reshape(B, -1, N)   # (B, C, N) with a label mask (mask_to_channels), else C = 1
    ga = np.zeros(2)
    for b in range(B):
        for n0 in range(0, N, chunk):
            sl = slice(n0, min(N, n0 + chunk))
            rays = (src[b:b + 1, None], tgt[b:b + 1, sl], raylen[b:b + 1, None, sl], gout[b:b + 1, :, sl])
            if mask is None:
                g = oracle.trilinear_bwd(vol, *rays, dtype=np.float32, want_vol=False, **kw)
            else:
                g = oracle.trilinear_bwd_mask(vol, mask, *rays, dtype=np.float32, want_vol=False, **kw)
            ga += (g["g_alphamin"], g["g_alphamax"])
    return ga


def _cone(src, centre, u, v, H, W):
    """Targets of an H x W detector centred on `centre` spanned by the half-extents u (columns) and v (rows)."""
    su = np.linspace(-1.0, 1.0, W)
    sv = np.linspace(-1.0, 1.0, H)
    tgt = centre[None, None, :] + sv[:, None, None] * v[None, None, :] + su[None, :, None] * u[None, None, :]
    return tgt.reshape(H * W, 3)


def _finish(src, tgt):
    src = np.asarray(src, np.float32)
    tgt = np.asarray(tgt, np.float32)
    raylen = np.linalg.norm(tgt.astype(np.float64) - src[:, None, :].astype(np.float64), axis=-1).astype(np.float32)
    return src, tgt, raylen


def _frame(rng):
    d = rng.normal(size=3)
    d /= np.linalg.norm(d)
    u = np.cross(d, [0.3, 0.5, 0.8])
    u /= np.linalg.norm(u)
    return d, u, np.cross(d, u)


def inside(dims, H, W, B, seed=0):
    """Sources inside the volume (entry alpha < 0 on every ray), detector 1.5 volume diagonals away in a random direction."""
    rng = np.random.default_rng(seed)
    D = np.asarray(dims, np.float64)
    diag = float(np.linalg.norm(D))
    srcs, tgts = [], []
    for _ in range(B):
        s = (0.25 + 0.5 * rng.random(3)) * (D - 1)
        d, u, v = _frame(rng)
        srcs.append(s)
        tgts.append(_cone(s, s + 1.5 * diag * d, 0.9 * diag * u, 0.7 * diag * v, H, W))
    return _finish(srcs, tgts)


def miss(dims, H, W, B, seed=0):
    """Sources outside, a detector wider than the projection of the volume: hits and misses in every pose."""
    rng = np.random.default_rng(seed)
    D = np.asarray(dims, np.float64)
    diag = float(np.linalg.norm(D))
    centre = (D - 1) / 2
    srcs, tgts = [], []
    for _ in range(B):
        d, u, v = _frame(rng)
        s = centre - 2.0 * diag * d
        srcs.append(s)
        tgts.append(_cone(s, centre + 2.0 * diag * d, 1.2 * diag * u, 1.0 * diag * v, H, W))
    return _finish(srcs, tgts)


def near_identical(dims, H, W, B, seed=0):
    """B poses within 1e-3 voxel of each other, rays through the volume clear of its edges: the voxels they cross receive thousands of
    red_adds each from the volume-gradient scatter."""
    rng = np.random.default_rng(seed)
    D = np.asarray(dims, np.float64)
    centre = (D - 1) / 2
    d = np.array([0.31, 0.87, 0.38])
    d /= np.linalg.norm(d)
    u = np.cross(d, [0.0, 0.0, 1.0])
    u /= np.linalg.norm(u)
    v = np.cross(d, u)
    srcs, tgts = [], []
    for _ in range(B):
        s = centre - 4.0 * D.max() * d + 1e-3 * rng.standard_normal(3)
        srcs.append(s)
        tgts.append(_cone(s, centre + 2.0 * D.max() * d, 0.45 * D.max() * u, 0.45 * D.max() * v, H, W))
    return _finish(srcs, tgts)


def axis_planes(dims, shift=0.5):
    """pix0 of the axis-parallel poses: an integer plane on a 16- and 8-plane slab face (15), another integer plane (7), the upper
    face D0-1 (its far corner is out of bounds) and the zero-padding half-cell -0.5; only those inside [-1, D0) are kept."""
    D0 = dims[0]
    return [p for p in dict.fromkeys((15.0, 7.0, float(D0 - 1), -0.5)) if -1.0 < p < D0]


def axis_row_kind(h):
    """Row class of the axis-parallel detector: 0 = exactly zero direction along axis 0, 1 = one ulp of pix0 below,
    2 = oblique (ordinary rays sharing the pose)."""
    return h % 3


def axis(dims, H, W, shift=0.5):
    """One pose per entry of axis_planes: the source sits on the plane pix0 = p (x0 = p + 0.5 - shift), rays run along axis 1
    towards a detector beyond the volume.  Rows by axis_row_kind; the centre column also has zero direction along axis 2, at an
    integer pix2, so its rays are parallel to axis 1 with corner weights exactly 0 or 1 on two axes."""
    D = np.asarray(dims, np.float64)
    planes = axis_planes(dims, shift)
    z_src = float(np.floor((D[2] - 1) / 2))
    srcs, tgts = [], []
    for p in planes:
        x0 = np.float32(p + 0.5 - shift)
        s = np.array([x0, -0.5 * D[1] - 7.123, z_src + 0.5 - shift], np.float64)
        t = np.empty((H, W, 3), np.float64)
        # off-grid, per-column axis-1 end points: the samples of different rays do not all meet the pix1 = integer planes at once
        t[:, :, 1] = 1.5 * D[1] + 9.377 + 0.0137 * np.arange(W)[None, :]
        t[:, :, 2] = s[2] + np.linspace(-0.8, 0.8, W)[None, :] * D[2]
        t[:, W // 2, 2] = s[2]
        for h in range(H):
            k = axis_row_kind(h)
            t[h, :, 0] = x0 if k == 0 else np.nextafter(x0, np.float32(-np.inf)) if k == 1 else x0 + (h - H / 2) * 0.37
        srcs.append(s)
        tgts.append(t.reshape(H * W, 3))
    return _finish(srcs, tgts)


def axis_kinks(H, W):
    """(H*W,) bool: the axis-parallel rays that run on an integer plane of pix0 (row kinds 0 and 1) or pix2 (the centre column).
    There the interpolant has a kink, and its derivative -- hence the end-point gradients and range partials -- is a
    one-sided sub-gradient whose side the reference's own fp32 / fp64 normalisation round-off picks (the tie convention
    DESIGN.md "Pinned" excludes).  Image, g_volume and g_raylen are continuous there and are compared on every ray."""
    k = np.array([axis_row_kind(h) for h in range(H)])
    kink = np.repeat((k != 2)[:, None], W, axis=1)
    kink[:, W // 2] = True
    return kink.reshape(H * W)


def pix(x, shift=0.5):
    """The kernels' continuous voxel coordinate (align_corners=False): pix = x + shift - 0.5."""
    return np.float32(x) + np.float32(shift - 0.5)


def entry_exit(dims, src, tgt, shift=0.5, eps=1e-8, padded=False):
    """Unclamped per-ray entry / exit alphas in fp64: of the slab test of reference renderers.py:124-140 (planes x = -shift and
    dims + 1 - shift), or with padded=True of the region pix in (-1, D) where the interpolant can be non-zero."""
    s = src[:, None, :].astype(np.float64)
    d = tgt.astype(np.float64) - s + eps
    lo, hi = (-0.5 - shift, np.asarray(dims, np.float64) + 0.5 - shift) if padded else (-shift, np.asarray(dims, np.float64) + 1.0 - shift)
    with np.errstate(divide="ignore", invalid="ignore"):
        a0 = (lo - s) / d
        a1 = (hi - s) / d
    return np.minimum(a0, a1).max(-1), np.maximum(a0, a1).min(-1)


def range_of(dims, src, tgt, shift=0.5, eps=1e-8):
    """Batch-global sampling range [alphamin, alphamax] as the module computes it (fp32, clamped to [0, 1])."""
    from oracle import oracle
    return oracle.alpha_minmax(dims, src[:, None, :], tgt, shift, eps, np.float32)
