"""Stationary velocity fields (DESIGN.md 6m): the group exponential of a velocity on the deformable render's lattice, by scaling
and squaring on the GPU, and the log-Euclidean blend of `DRR.render_polyrigid(blend="log_euclidean")` built on it.

exp(v) ~ (id + v / 2^N)^(2^N): N composition steps u' = u + u o (id + u), the first one taking u_0 = v / 2^N.  Every step is one
launch of b200drr_svf_square (include/b200drr.h), its lookup clamped to the lattice's node range, and the backward runs the
steps' adjoints (b200drr_svf_square_bwd) in reverse.  The field is render_deformed's lattice (node i of axis a at voxel coordinate
(i + 1/2) D_a / g_a - 1/2), so the exponential's output goes straight into render_deformed's march.
"""
from __future__ import annotations

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .deform import render_voxel_field, voxel_field
from .pose import _hat
from .renderers import _ptr, _stream
from .structures import _rigid_inverse

MAX_STEPS = 16


def _aligned(t):
    """t contiguous and 16-byte aligned (the kernels read float4 nodes)."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _scale(k, steps):
    """Step k's s: 1 / 2^steps on the first step (it folds v / 2^steps in), 1 on the others."""
    return 2.0**-steps if k == 0 else 1.0


def square_chain(U, steps, dims):
    """The kernels' field U (Bf, g0, g1, g2, 4), voxel units -> (levels, exp(U)): `steps` squaring launches on a volume of shape
    dims, levels the inputs of the steps (levels[0] is U).  No autograd."""
    levels = [_aligned(U)]
    lib = _lib.load()
    with torch.cuda.device(U.device):
        for k in range(steps):
            out = torch.empty_like(levels[0])
            _lib.check(lib.b200drr_svf_square(_ptr(levels[-1]), _ptr(out), U.shape[0], *U.shape[1:4], *dims, _scale(k, steps),
                                              _stream()), "b200drr_svf_square")
            levels.append(out)
    return levels[:-1], levels[-1]


def square_chain_bwd(levels, g, dims):
    """The adjoint of square_chain: an upstream gradient g on exp(U) -> the gradient on U, the steps' adjoints in reverse over
    square_chain's levels.  No autograd."""
    steps = len(levels)
    g = _aligned(g)
    lib = _lib.load()
    with torch.cuda.device(g.device):
        for k in reversed(range(steps)):
            gin = torch.empty_like(levels[0])
            _lib.check(lib.b200drr_svf_square_bwd(_ptr(levels[k]), _ptr(g), _ptr(gin), g.shape[0], *g.shape[1:4], *dims,
                                                  _scale(k, steps), _stream()), "b200drr_svf_square_bwd")
            g = gin
    return g


def square_chain_jvp(levels, T, dims, steps=None):
    """The tangent T (voxel units, U's layout) pushed through the squarings, one b200drr_svf_square_jvp per step -> (exp(U) or
    None, the tangent of exp(U)).  levels: square_chain's levels, read as they are (steps = len(levels), exp(U) not returned); or,
    with `steps` given, [U] alone: each launch then also writes the next level, b200drr_svf_square's bits, so the primal and the
    tangent share the `steps` launches and exp(U) is returned.  The exact transpose of square_chain_bwd over the same levels.  No
    autograd."""
    carry = steps is not None
    levels, steps = [_aligned(levels[0])] if carry else list(levels), steps if carry else len(levels)
    T = _aligned(T)
    lib = _lib.load()
    with torch.cuda.device(T.device):
        for k in range(steps):
            tout = torch.empty_like(levels[0])
            out = torch.empty_like(levels[0]) if carry else None
            _lib.check(lib.b200drr_svf_square_jvp(_ptr(levels[k]), _ptr(T), _ptr(tout), _ptr(out), T.shape[0], *T.shape[1:4], *dims,
                                                  _scale(k, steps), _stream()), "b200drr_svf_square_jvp")
            if carry:
                levels.append(out)
            T = tout
    return (levels[-1] if carry else None), T


class _SquaringFunction(torch.autograd.Function):
    """The kernels' field U (Bf, g0, g1, g2, 4), voxel units -> exp(U) in the same layout, by `steps` squaring launches on a volume
    of shape dims (square_chain).  Saves the input of every step (steps fields of U's size) for the backward (square_chain_bwd)."""

    @staticmethod
    def forward(ctx, U, steps, dims):
        levels, out = square_chain(U, steps, dims)
        ctx.save_for_backward(*levels)
        ctx.consts = dims
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return square_chain_bwd(ctx.saved_tensors, g, ctx.consts), None, None


def check_steps(steps):
    if isinstance(steps, bool) or not isinstance(steps, int) or not 1 <= steps <= MAX_STEPS:
        raise ValueError(f"steps must be an int in 1..{MAX_STEPS} (the number of squarings), got {steps!r}")


def check_velocity(drr, velocity, steps):
    """exp_velocity's refusals, before any launch."""
    check_steps(steps)
    if not torch.is_tensor(velocity) or velocity.dtype != torch.float32 or velocity.dim() not in (4, 5) or \
            velocity.shape[-4] != 3 or min(velocity.shape[-3:]) < 1 or (velocity.dim() == 5 and velocity.shape[0] < 1):
        got = f"{velocity.dtype} {tuple(velocity.shape)}" if torch.is_tensor(velocity) else type(velocity).__name__
        raise ValueError(f"velocity must be an fp32 velocity lattice (3, g0, g1, g2) or (B, 3, g0, g1, g2), got {got}")
    g0, g1, g2 = velocity.shape[-3:]
    if 4 * g0 * g1 * g2 >= 2**31 - 1:
        raise NotImplementedError(f"exp_velocity takes a lattice below 2^31 floats per pose (4 channels), got {(g0, g1, g2)}")
    if not velocity.is_cuda:
        raise _lib.B200DRRError(f"diffdrr_b200 runs on CUDA devices only (velocity is on {velocity.device}); there is no CPU "
                                "fallback")
    if velocity.device != drr.density.device:
        raise ValueError(f"velocity must be on the density's device {drr.density.device}, not {velocity.device}")


def _world(drr, phi, dim):
    """The kernels' field (Bf, g0, g1, g2, 4), voxel units -> world mm (Bf, 3, g0, g1, g2), or (3, g0, g1, g2) for dim 4."""
    lin = drr._affine.reshape(4, 4)[:3, :3]
    u = torch.einsum("ij,bxyzj->bixyz", lin, phi[..., :3])
    return u if dim == 5 else u[0]


def exp_velocity(drr, velocity, steps=10):
    """The pull-back displacement of exp(v) for a stationary velocity field v, by scaling and squaring on the GPU (DESIGN.md 6m).

    velocity: fp32 (3, g0, g1, g2) or (B, 3, g0, g1, g2) on the density's device, world mm, on render_deformed's lattice (node i
    of axis a at voxel coordinate (i + 1/2) D_a / g_a - 1/2 of drr.density).  -> the displacement u of phi = exp(v) = id + u,
    world mm, the same shape: pass it as drr.render_deformed(..., field=u).  phi is the composition of 2^steps copies of
    id + v / 2^steps, each step's lookup trilinear with lattice coordinates clamped to the node range; the error against the
    exact flow falls 4x per step (steps = 10 by default; 1..16).  A zero velocity gives an exactly zero field.

    Differentiable in the velocity (b200drr_svf_square_bwd; the gradient repeats to fp32 reordering).  Autograd keeps the input
    of every step, `steps` fields of Bf * g0 * g1 * g2 * 16 bytes (4.2 MB per 64^3 field and step).  A velocity that is not
    fp32, of the wrong rank or channel count, on the CPU or another device, or a steps outside 1..16 raises before any launch."""
    check_velocity(drr, velocity, steps)
    phi = _SquaringFunction.apply(voxel_field(drr, velocity), steps, tuple(drr.density.shape))
    return _world(drr, phi, velocity.dim())


def exp_velocity_jvp(drr, velocity, tangent, steps=10):
    """exp_velocity and its directional derivative along a velocity tangent (DESIGN.md 6n) -> (u, du), both world mm in the
    velocity's shape: u = exp_velocity(drr, velocity, steps), bit for bit, and du = d/de exp_velocity(drr, velocity + e tangent,
    steps) at e = 0.  One b200drr_svf_square_jvp launch per step carries the primal and the tangent together.  tangent: a tensor
    of the velocity's shape, dtype and device.  No autograd: the results do not require grad.  The refusals are exp_velocity's
    and DRR.deformed_jvp's tangent checks, before any launch."""
    from .deform import _check_tangent

    check_velocity(drr, velocity, steps)
    _check_tangent(velocity, tangent)
    with torch.no_grad():
        phi, dphi = square_chain_jvp([voxel_field(drr, velocity)], voxel_field(drr, tangent), tuple(drr.density.shape), steps=steps)
        return _world(drr, phi, velocity.dim()), _world(drr, dphi, velocity.dim())


def se3_log_matrix(X):
    """Rigid matrices X (..., 4, 4) -> their logarithms (..., 4, 4) [hat(w) V(w)^-1 t; 0 0], float64 (V as pose._se3_V).  The
    rotation part is w = theta / (2 sin theta) vee(R - R^T), theta = atan2(|vee(R - R^T)| / 2, (tr R - 1) / 2), with the series
    1 + theta^2 / 6 for theta / sin theta near 0: finite with the correct derivative at the identity, where registration starts.
    Rotations by less than pi."""
    X = X.double()
    R, t = X[..., :3, :3], X[..., :3, 3]
    vee = torch.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
    c = 0.5 * (R[..., 0, 0] + R[..., 1, 1] + R[..., 2, 2] - 1.0)
    theta = torch.atan2(0.5 * torch.linalg.vector_norm(vee, dim=-1), c)
    small = theta < 1e-4
    f = torch.where(small, 1.0 + theta * theta / 6.0, theta / torch.where(small, torch.ones_like(theta), torch.sin(theta)))
    w = 0.5 * f[..., None] * vee
    # V(w)^-1 = I - W / 2 + e W^2, e = 1 / theta^2 - (1 + cos theta) / (2 theta sin theta) (series 1/12 + theta^2 / 720): closed
    # form, so no solve that synchronises with the host (CUDA-graph capture)
    ts = torch.where(small, torch.ones_like(theta), theta)
    e = torch.where(small, 1.0 / 12.0 + theta * theta / 720.0, 1.0 / (ts * ts) - (1.0 + torch.cos(ts)) / (2.0 * ts * torch.sin(ts)))
    W = _hat(w)
    Vinv = torch.eye(3, dtype=W.dtype, device=W.device) - 0.5 * W + e[..., None, None] * (W @ W)
    top = torch.cat([W, Vinv @ t[..., None]], -1)
    return torch.cat([top, torch.zeros_like(top[..., :1, :])], -2)


def polyrigid_velocity(drr, X, weights):
    """The log-Euclidean velocity of world motions X (K, 4, 4) or (B, K, 4, 4) blended by the lattice weights (K, g0, g1, g2) ->
    the kernels' field (Bm, g0, g1, g2, 4), voxel units: v(x) = sum_k w_k(x) L_k [x; 1] at every node x, L_k = A^-1 log(X_k^-1) A
    = log(M_k) for voxel_maps' M_k, formed in float64.  Torch ops, so autograd carries the field's gradient on to the motions."""
    A = drr._affine.reshape(4, 4).double()
    Ainv = torch.linalg.inv_ex(A).inverse
    L = (Ainv @ se3_log_matrix(_rigid_inverse(X.double())) @ A)[..., :3, :].float()   # (..., K, 3, 4)
    L = L if L.dim() == 4 else L[None]
    K, g = weights.shape[0], tuple(weights.shape[1:])
    D = drr.density.shape
    W = weights.reshape(K, -1)
    axes = [((torch.arange(g[a], dtype=torch.float64, device=W.device) + 0.5) * (D[a] / g[a]) - 0.5).float() for a in range(3)]
    xh = torch.nn.functional.pad(torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3), (0, 1), value=1.0)
    Lw = torch.matmul(W.T, L.reshape(L.shape[0], K, 12)).view(L.shape[0], -1, 3, 4)   # sum_k w_k(x) L_k per node: (Bm, n, 3, 4)
    v = (Lw * xh[:, None, :]).sum(-1)
    return torch.nn.functional.pad(v.view(L.shape[0], *g, 3), (0, 1)).contiguous()


def square_chain_tangents(levels, T, dims):
    """P tangents T (Bm, g0, g1, g2, P, 4), voxel units, node-major, pushed through the squarings over square_chain's levels (read
    as they are, so the primal is not recomputed), one b200drr_svf_square_tangents per step -> the P tangents of exp(U) in the
    same layout.  Slice p is square_chain_jvp(levels, T[..., p, :], dims)[1] bit for bit.  Two tangent fields live at a time.  No
    autograd."""
    steps = len(levels)
    T = _aligned(T)
    Bm, P = T.shape[0], T.shape[4]
    lib = _lib.load()
    with torch.cuda.device(T.device):
        spare = torch.empty_like(T)
        for k in range(steps):
            _lib.check(lib.b200drr_svf_square_tangents(_ptr(levels[k]), _ptr(T), _ptr(spare), None, Bm, P, *T.shape[1:4], *dims,
                                                       _scale(k, steps), _stream()), "b200drr_svf_square_tangents")
            T, spare = spare, T
    return T


def se3_log_tangents(Y, dY):
    """The derivative of se3_log_matrix at Y (..., 4, 4) along dY (the same shape), float64, by forward-mode AD through its closed
    form (torch.func.jvp): finite at the identity, where registration starts, and no host sync."""
    return torch.func.jvp(se3_log_matrix, (Y.double(),), (dY.double(),))[1]


def velocity_tangents(drr, X, weights, pivots):
    """The derivatives of polyrigid_velocity along the 6K motion increments (DESIGN.md 6p) -> (Bm, g0, g1, g2, 6K, 4) fp32, voxel
    units, node-major, lane 3 zero: tangent p = 6k + i at node x is w_k(x) (dL_k / d xi_ki) [x; 1] with
    dL_k / d xi_ki = A^-1 Dlog|_{X_k^-1}[-X_k^-1 T(c_k) E_i T(-c_k)] A, the left increment X_k(xi) = T(c_k) exp(xi^) T(-c_k) X_k about
    the pivot c_k of polyrigid_tangents (its inner matrix).  X (K, 4, 4) or (B, K, 4, 4); pivots (K, 3) float64.  Dlog in float64."""
    from .structures import _translation, twist_matrix

    A = drr._affine.reshape(4, 4).double()
    Ainv = torch.linalg.inv_ex(A).inverse
    Xinv = _rigid_inverse(X.detach().double())
    Xinv = Xinv if Xinv.dim() == 4 else Xinv[None]                                          # (Bm, K, 4, 4)
    E = twist_matrix(torch.eye(6, dtype=torch.float64, device=Xinv.device))                 # (6, 4, 4)
    dXinv = -(Xinv @ _translation(pivots))[:, :, None] @ E @ _translation(-pivots)[None, :, None]   # (Bm, K, 6, 4, 4)
    dL = Ainv @ se3_log_tangents(Xinv[:, :, None].expand_as(dXinv).contiguous(), dXinv) @ A
    dL = dL[..., :3, :].float()                                                             # (Bm, K, 6, 3, 4)
    Bm, K = dL.shape[:2]
    g = tuple(weights.shape[1:])
    D = drr.density.shape
    axes = [((torch.arange(g[a], dtype=torch.float64, device=dL.device) + 0.5) * (D[a] / g[a]) - 0.5).float() for a in range(3)]
    xh = torch.nn.functional.pad(torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3), (0, 1), value=1.0)
    t = torch.einsum("bkirc,nc->bnkir", dL, xh) * weights.reshape(K, -1).T[None, :, :, None, None]
    return torch.nn.functional.pad(t.reshape(Bm, *g, 6 * K, 3), (0, 1)).contiguous()


def render_log_euclidean(drr, args, X, B, weights, steps, parameterization, convention, degrees, calibration, n_points, alphamin,
                         alphamax, vol):
    """render_polyrigid(blend="log_euclidean") after its checks: exp of polyrigid_velocity, marched by render_deformed through the
    density vol (drr.density, or render_polyrigid's density=, whose gradient is then b200drr_deform_bproj's)."""
    U = _SquaringFunction.apply(polyrigid_velocity(drr, X, weights), steps, tuple(drr.density.shape))
    return render_voxel_field(drr, args, B, U, parameterization, convention, degrees, calibration, n_points, alphamin, alphamax,
                              vol)
