"""Blended-rigid (skinned) DRRs (`DRR.render_polyrigid`; DESIGN.md 6h): the volume under K rigid motions blended by smooth weights.

The rays and samples are the Trilinear renderer's.  Every sample x (voxel-index coordinates) reads the density at
    y = x + sum_k w_k(x) (M_k [x; 1] - x),        M_k = A^-1 X_k^-1 A,
X_k the world motion of structure k (meaning as in render_structures), A = drr.affine, w_k a coarse weight lattice over the volume
with sum_k w_k <= 1 (the rest of the weight stays on the identity).  M is formed here with torch ops, so autograd carries the
kernel's g_M (include/b200drr.h: b200drr_polyrigid_bwd) on to whatever parameterises the motions.

A density passed as `density=` may require grad (fp32): its gradient is the forward's transpose in the density, a backprojection
along the blended samples (b200drr_polyrigid_bproj; DESIGN.md 6o), for reconstruction under articulated motion.
"""
from __future__ import annotations

import weakref

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .deform import _check_density, _check_renderer, _launch_args, _marches, _rendered_density
from .renderers import _ptr, _stream, _vol_entry  # noqa: F401  (_vol_entry: the tests call the entry points through this module)
from .structures import _batch_size, _label_tuple, _motion_matrices, _rigid_inverse, _translation, twist_matrix

MAX_STRUCTURES = 8
_weights_cache = None   # (key, weak reference to the mask, lattice) of the last polyrigid_weights call


def _gaussian_1d(sigma, device):
    radius = max(1, int(3.0 * sigma + 0.5))
    x = torch.arange(-radius, radius + 1, dtype=torch.float32, device=device)
    k = torch.exp(-0.5 * (x / sigma) ** 2)
    return k / k.sum()


def polyrigid_weights(mask, labels, grid=(64, 64, 64), sigma=6.0, spacing=(1.0, 1.0, 1.0)):
    """Blend weights for render_polyrigid from a label volume: -> (K, g0, g1, g2) fp32 on the mask's device, in [0, 1], sum_k <= 1.

    Channel k is the occupancy of labels[k] in `mask` (D0, D1, D2) averaged onto the lattice, smoothed by a Gaussian of `sigma`
    mm (`spacing` = voxel size in mm per axis; zero beyond the volume), and the channels are scaled down together wherever they
    sum above 1.  Set-up code in plain torch; the result of the last call is kept and returned again while the mask tensor is
    unchanged.  Any lattice of the same form may be passed to render_polyrigid instead."""
    global _weights_cache
    labels = _label_tuple(labels)
    grid = tuple(int(g) for g in grid)
    spacing = tuple(float(s) for s in spacing)
    if mask.dim() != 3 or len(grid) != 3 or min(grid) < 1 or len(spacing) != 3 or not sigma > 0:
        raise ValueError(f"polyrigid_weights needs a 3-D label volume, a 3-D lattice and sigma > 0, got mask {tuple(mask.shape)}, "
                         f"grid {grid}, sigma {sigma}")
    key = (mask.data_ptr(), mask._version, mask.device, tuple(mask.shape), labels, grid, float(sigma), spacing)
    if _weights_cache is not None and _weights_cache[0] == key and _weights_cache[1]() is mask:
        return _weights_cache[2]
    with torch.no_grad():
        occ = torch.stack([(mask == lab).float() for lab in labels])[None]                  # (1, K, D0, D1, D2)
        w = torch.nn.functional.adaptive_avg_pool3d(occ, grid)[0]                           # (K, g0, g1, g2)
        for a in range(3):
            cell_mm = spacing[a] * mask.shape[a] / grid[a]
            k = _gaussian_1d(max(float(sigma) / cell_mm, 1e-3), mask.device)
            w = w.movedim(1 + a, -1)
            shape = w.shape
            w = torch.nn.functional.conv1d(w.reshape(-1, 1, shape[-1]), k[None, None], padding=k.numel() // 2).reshape(shape)
            w = w.movedim(-1, 1 + a)
        w = (w / w.sum(0, keepdim=True).clamp_min(1.0)).clamp_(0.0, 1.0).contiguous()
    _weights_cache = (key, weakref.ref(mask), w)
    return w


def _packed_weights(drr, weights):
    """The kernels' copy of the lattice (channel-last, K padded to 4 or 8), cached per lattice tensor on `drr`.  Building it is the
    one place the lattice's values are read on the host: weights outside [0, 1] or summing above 1 are refused here."""
    key = (weights.data_ptr(), weights._version, weights.device, tuple(weights.shape))
    cached = getattr(drr, "_polyrigid_cache", None)
    if cached is not None and cached[0] == key and cached[1]() is weights:
        return cached[2]
    K, g0, g1, g2 = weights.shape
    with torch.no_grad():
        w = weights.detach().contiguous()
        lo, hi, total = torch.stack([w.min(), w.max(), w.sum(0).max()]).tolist()   # one device-to-host copy per lattice
        if not (lo >= 0.0 and hi <= 1.0 and total <= 1.0 + 1e-5):
            raise ValueError(f"render_polyrigid needs blend weights in [0, 1] that sum to at most 1 over the structures; got values "
                             f"in [{lo:g}, {hi:g}] and a largest sum of {total:g}")
        lib = _lib.load()
        packed = torch.empty(int(lib.b200drr_polyrigid_weight_floats(K, g0, g1, g2)), dtype=torch.float32, device=w.device)
        with torch.cuda.device(w.device):
            _lib.check(lib.b200drr_polyrigid_pack_weights(_ptr(w), K, g0, g1, g2, _ptr(packed), _stream()),
                       "b200drr_polyrigid_pack_weights")
    object.__setattr__(drr, "_polyrigid_cache", (key, weakref.ref(weights), packed))
    return packed


def check_supported(drr, args, parameterization, motions, weights, kwargs, density=None):
    """Refuse, before any launch, what the blended-rigid render does not cover: -> (motion matrices, B, K).  density: the volume
    rendered in place of drr.density (render_polyrigid's density=), or None."""
    _check_renderer(drr, "render_polyrigid", "the blended motion", kwargs)
    if not torch.is_tensor(weights) or weights.dim() != 4 or weights.dtype != torch.float32:
        got = f"{weights.dtype} {tuple(weights.shape)}" if torch.is_tensor(weights) else type(weights).__name__
        raise ValueError(f"weights must be an fp32 lattice (K, g0, g1, g2), got {got}")
    K = weights.shape[0]
    if K > MAX_STRUCTURES:
        raise NotImplementedError(f"render_polyrigid blends at most {MAX_STRUCTURES} structures, got {K}")
    if weights.requires_grad:
        raise NotImplementedError("render_polyrigid produces no gradient for the blend weights: they must not require grad")
    B = _batch_size(args, parameterization)
    X = _motion_matrices(motions, K, B)
    vol, no_grad = _rendered_density(drr, density, "render_polyrigid",
                                     "render_polyrigid produces no volume gradient: the density must not require grad")
    _check_density(vol, "render_polyrigid", no_grad)
    if X.device != vol.device or weights.device != vol.device:
        raise ValueError(f"motions and weights must be on the density's device {vol.device}, not {X.device} and {weights.device}")
    return X, B, K


class _PolyrigidFunction(torch.autograd.Function):
    """out (B, 1, N) for rays in voxel-index space, the maps M (Bm, K, 3, 4) and the range alpha_range = [alphamin, alphamax]; the
    density comes from its packed-corner copy when there is one, fp32 or 16-bit, through the entry point that takes it."""

    @staticmethod
    def forward(ctx, volume, packed, source, target, img, M, alpha_range, wpacked, lattice, voxel_shift, eps, n_points, grid):
        vol = volume.contiguous()
        fn, head, name, (src, tgt, raylen), (H, W) = _launch_args("b200drr_polyrigid_fwd", vol, packed, source, target, img, grid)
        B, N = tgt.shape[0], tgt.shape[1]
        M = M.contiguous().float()
        arange = alpha_range.detach().to(device=vol.device, dtype=torch.float32).contiguous()
        out = torch.empty(B, N, dtype=torch.float32, device=vol.device)
        tail = (B, N, H, W, voxel_shift, eps, n_points, _ptr(arange), _stream())
        geom = (*vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(M), M.shape[0], M.shape[1], _ptr(wpacked), *lattice)
        with torch.cuda.device(vol.device):
            _lib.check(fn(*head, *geom, _ptr(out), *tail), name)
        ctx.save_for_backward(vol, packed, src, tgt, raylen, M, arange, wpacked)
        ctx.consts = (lattice, voxel_shift, eps, n_points, H, W, source.shape, img.shape)
        return out.view(B, 1, N)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        vol, packed, src, tgt, raylen, M, arange, wpacked = ctx.saved_tensors
        lattice, voxel_shift, eps, n_points, H, W, source_shape, img_shape = ctx.consts
        B, N = tgt.shape[0], tgt.shape[1]
        dev = vol.device
        gout = gout.reshape(B, N).contiguous().float()
        lib = _lib.load()
        g_vol = None
        if ctx.needs_input_grad[0]:   # the forward's transpose in the density: a backprojection, no density read
            g_vol = torch.empty(vol.shape, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.b200drr_polyrigid_bproj(*vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(M), M.shape[0],
                                                       M.shape[1], _ptr(wpacked), *lattice, _ptr(gout), _ptr(g_vol), B, N, H, W,
                                                       voxel_shift, eps, n_points, _ptr(arange), _stream()), "b200drr_polyrigid_bproj")
        if not any(ctx.needs_input_grad[2:7]):   # a reconstruction step: the density is the only input that wants a gradient
            return g_vol, None, None, None, None, None, None, None, None, None, None, None, None
        g_src = torch.empty(B, 3, dtype=torch.float32, device=dev)
        g_tgt = torch.empty(B, N, 3, dtype=torch.float32, device=dev)
        g_raylen = torch.empty(B, N, dtype=torch.float32, device=dev)
        g_M = torch.empty_like(M)
        g_range = torch.empty(2, dtype=torch.float32, device=dev)
        scratch = torch.empty(int(lib.b200drr_polyrigid_scratch_floats(B, N, H, W, M.shape[1])), dtype=torch.float32, device=dev)
        fn, head, name, _, _ = _launch_args("b200drr_polyrigid_bwd", vol, packed, src, tgt, raylen, (H, W))
        with torch.cuda.device(dev):
            _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(M), M.shape[0], M.shape[1], _ptr(wpacked),
                          *lattice, _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_raylen), _ptr(g_M), _ptr(g_range), _ptr(scratch),
                          B, N, H, W, voxel_shift, eps, n_points, _ptr(arange), _stream()), name)
        return (g_vol, None, g_src.view(source_shape), g_tgt, g_raylen.view(img_shape), g_M, g_range, None, None, None, None, None,
                None)


def voxel_maps(drr, X):
    """World motions X (..., K, 4, 4) -> the kernels' maps M = A^-1 X^-1 A (..., K, 3, 4), fp32; the product is taken in float64
    so that identity motions give an exact identity rotation block (and a translation of float64 round-off)."""
    A = drr._affine.reshape(4, 4).double()
    Ainv = torch.linalg.inv_ex(A).inverse   # not the module's fp32 inverse: A^-1 A must be the identity to float64 round-off
    return (Ainv @ _rigid_inverse(X.double()) @ A)[..., :3, :].float()


def render_polyrigid(drr, *args, motions, weights, parameterization=None, convention=None, degrees=False, calibration=None,
                     n_points=500, alphamin=None, alphamax=None, blend="linear", steps=10, density=None, **kwargs):
    """See DRR.render_polyrigid."""
    if blend not in ("linear", "log_euclidean"):
        raise ValueError(f"blend must be 'linear' or 'log_euclidean', got {blend!r}")
    if blend == "log_euclidean":
        from . import svf

        svf.check_steps(steps)
    X, B, K = check_supported(drr, args, parameterization, motions, weights, kwargs, density=density)
    vol, r = drr.density if density is None else density, drr.renderer
    wpacked = _packed_weights(drr, weights)
    if blend == "log_euclidean":   # the lattice check above is the linear blend's; the packed copy is not used
        return svf.render_log_euclidean(drr, args, X, B, weights, steps, parameterization, convention, degrees, calibration,
                                        n_points, alphamin, alphamax, vol)
    source, marches = _marches(drr, args, B, parameterization, convention, degrees, calibration, alphamin, alphamax, vol=vol)
    M = voxel_maps(drr, X)
    M = M if M.dim() == 4 else M[None]
    packed = r._packed_volume(vol)
    outs = [_PolyrigidFunction.apply(vol, packed, source, tgt, lens, M, alpha_range, wpacked, tuple(weights.shape[1:]),
                                     float(r.voxel_shift), float(r.eps), int(n_points), grid) for tgt, lens, alpha_range, grid in marches]
    out = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)   # serial patches with a range each, as DRR.render
    return drr.reshape_transform(out, batch_size=B)


def polyrigid_pivots(drr, weights):
    """(K, 3) float64 world points: the weight-weighted centroid of each channel's lattice nodes, the centre about which
    polyrigid_jacobian and PolyrigidLevenbergMarquardt turn structure k.  Node i of axis a sits at voxel coordinate
    (i + 1/2) D_a / g_a - 1/2 (render_polyrigid's lattice convention), mapped to world by drr.affine.  A channel whose weights are
    all zero gets the volume's centre.  Torch ops only, no host sync."""
    K, g = weights.shape[0], weights.shape[1:]
    D = drr.density.shape
    w = weights.detach().double()
    axes = [(torch.arange(g[a], dtype=torch.float64, device=w.device) + 0.5) * (D[a] / g[a]) - 0.5 for a in range(3)]
    total = w.sum((1, 2, 3))
    centroid = torch.stack([(w.sum(tuple(b + 1 for b in range(3) if b != a)) * axes[a]).sum(-1) for a in range(3)], -1)
    centre = torch.stack([torch.full((), (d - 1) / 2, dtype=torch.float64, device=w.device) for d in D])   # no host-to-device copy
    p = torch.where((total > 0)[:, None], centroid / torch.where(total > 0, total, 1.0)[:, None], centre)
    A = drr._affine.reshape(4, 4).double()
    return p @ A[:3, :3].mT + A[:3, 3]


def polyrigid_tangents(drr, X, pivots):
    """T (Bm, K, 6, 3, 4) fp32: the derivatives dM_k / d xi_ki at xi = 0 of the voxel maps M_k = A^-1 X_k(xi)^-1 A (voxel_maps) under
    the left increment X_k(xi) = T(c_k) exp(xi_k^) T(-c_k) X_k about pivot c_k (structures.apply_increments).  X (K, 4, 4) -> Bm = 1,
    or (B, K, 4, 4); pivots (K, 3) float64.  X_k(xi)^-1 = X_k^-1 T(c_k) exp(-xi_k^) T(-c_k), and the derivative is linear in the
    generator: T_i = -(A^-1 X_k^-1 T(c_k) E_i T(-c_k) A)[:3], E_i = twist_matrix(e_i), in closed form in float64."""
    A = drr._affine.reshape(4, 4).double()
    Ainv = torch.linalg.inv_ex(A).inverse
    X = X.detach().double()
    X = X if X.dim() == 4 else X[None]
    E = twist_matrix(torch.eye(6, dtype=torch.float64, device=X.device))                  # (6, 4, 4)
    left = Ainv @ _rigid_inverse(X) @ _translation(pivots)                                 # (Bm, K, 4, 4)
    right = _translation(-pivots) @ A                                                      # (K, 4, 4)
    T = -(left[:, :, None] @ E @ right[None, :, None])                                     # (Bm, K, 6, 4, 4)
    return T[..., :3, :].float().contiguous()


def polyrigid_jacobian(drr, *args, motions, weights, parameterization=None, convention=None, degrees=False, calibration=None,
                       n_points=500, alphamin=None, alphamax=None, return_footprints=False, blend="linear", steps=10, **kwargs):
    """See DRR.polyrigid_jacobian."""
    if blend not in ("linear", "log_euclidean"):
        raise ValueError(f"blend must be 'linear' or 'log_euclidean', got {blend!r}")
    if blend == "log_euclidean":
        from . import svf

        svf.check_steps(steps)
    det = drr.detector
    if det.n_subsample is not None or drr.patch_size is not None:
        raise NotImplementedError("polyrigid_jacobian covers the full detector only, not p_subsample or patch_size: the Jacobian "
                                  "kernel marches full H x W grids")
    X, B, K = check_supported(drr, args, parameterization, motions, weights, kwargs)
    if blend == "log_euclidean":
        return _log_euclidean_jacobian(drr, args, X, B, K, weights, steps, parameterization, convention, degrees, calibration,
                                       n_points, alphamin, alphamax, return_footprints)
    vol, r = drr.density, drr.renderer
    H, W = det.height, det.width
    with torch.no_grad():
        wpacked = _packed_weights(drr, weights)
        source, [(target, raylen, arange, grid)] = _marches(drr, args, B, parameterization, convention, degrees, calibration,
                                                            alphamin, alphamax)
        M = voxel_maps(drr, X)
        M = (M if M.dim() == 4 else M[None]).contiguous()
        T = polyrigid_tangents(drr, X, polyrigid_pivots(drr, weights))
        packed = r._packed_volume(vol)
        volc = vol.contiguous()
        fn, head, name, (src, tgt, raylen), _ = _launch_args("b200drr_polyrigid_jac", volc, packed, source, target, raylen, grid)
        img = torch.empty(B, H * W, dtype=torch.float32, device=vol.device)
        J = torch.empty(B, K, H * W, 6, dtype=torch.float32, device=vol.device)
        rects = torch.empty(B, K, 4, dtype=torch.int32, device=vol.device)
        with torch.cuda.device(vol.device):
            _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(M), M.shape[0], K, _ptr(wpacked),
                          *weights.shape[1:], _ptr(T), _ptr(img), _ptr(J), _ptr(rects), B, H, W, float(r.voxel_shift), float(r.eps),
                          int(n_points), _ptr(arange), _stream()), name)
    img = drr.reshape_transform(img.view(B, 1, H * W), batch_size=B)
    J = J.view(B, K, H, W, 6)
    return (img, J, rects) if return_footprints else (img, J)


def _log_euclidean_jacobian(drr, args, X, B, K, weights, steps, parameterization, convention, degrees, calibration, n_points, alphamin,
                            alphamax, return_footprints):
    """polyrigid_jacobian(blend="log_euclidean") after its checks (DESIGN.md 6p): the velocity and its 6K tangents, the squarings
    of the velocity (svf.square_chain, as render_polyrigid takes them) and of the tangents over its levels
    (svf.square_chain_tangents), then one b200drr_deform_jac march of exp(v) contracting the 6K tangents of exp(v)."""
    from . import svf

    vol, r = drr.density, drr.renderer
    H, W = drr.detector.height, drr.detector.width
    dims = tuple(vol.shape)
    with torch.no_grad():
        _packed_weights(drr, weights)   # render_polyrigid's lattice check
        levels, U = svf.square_chain(svf.polyrigid_velocity(drr, X, weights), steps, dims)
        T = svf.square_chain_tangents(levels, svf.velocity_tangents(drr, X, weights, polyrigid_pivots(drr, weights)), dims)
        del levels
        source, [(target, raylen, arange, grid)] = _marches(drr, args, B, parameterization, convention, degrees, calibration,
                                                            alphamin, alphamax)
        packed = r._packed_volume(vol)
        volc = vol.contiguous()
        fn, head, name, (src, tgt, raylen), _ = _launch_args("b200drr_deform_jac", volc, packed, source, target, raylen, grid)
        img = torch.empty(B, H * W, dtype=torch.float32, device=vol.device)
        J = torch.empty(B, K, H * W, 6, dtype=torch.float32, device=vol.device)
        rects = torch.empty(B, K, 4, dtype=torch.int32, device=vol.device)
        with torch.cuda.device(vol.device):
            _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(U), U.shape[0], *U.shape[1:4], _ptr(T), 6 * K, K,
                          _ptr(img), _ptr(J), _ptr(rects), B, H, W, float(r.voxel_shift), float(r.eps), int(n_points), _ptr(arange),
                          _stream()), name)
    img = drr.reshape_transform(img.view(B, 1, H * W), batch_size=B)
    J = J.view(B, K, H, W, 6)
    return (img, J, rects) if return_footprints else (img, J)
