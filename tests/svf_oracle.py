"""fp64 reference of the scaling-and-squaring exponential (csrc/svf_math.cuh; DESIGN.md 6m), plain trilinear lookups with the
lattice coordinates clamped to the node range, written in torch so that autograd through it is the reference gradient too.

Fields are (Bf, g0, g1, g2, 3) in voxel-index units on a lattice over a volume of shape D: node i of axis a sits at voxel
coordinate (i + 1/2) D_a / g_a - 1/2, so a displacement u moves node i's lattice coordinate to i + u_a g_a / D_a."""
import numpy as np
import torch


def _t(a):
    return a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a), dtype=torch.float64)


def node_coords(g, D, dtype=torch.float64):
    """The voxel coordinates of the lattice nodes: (g0, g1, g2, 3)."""
    axes = [(torch.arange(g[a], dtype=dtype) + 0.5) * (D[a] / g[a]) - 0.5 for a in range(3)]
    return torch.stack(torch.meshgrid(*axes, indexing="ij"), -1)


def _cell(q, g):
    """Per axis of q (..., 3): clamped cell (i0, i1, f) and live (the clamp inactive)."""
    hi = torch.tensor([gi - 1 for gi in g], dtype=q.dtype)
    qc = torch.minimum(torch.clamp(q, min=0.0), hi)
    live = (q >= 0) & (q <= hi)
    i0 = torch.floor(qc.detach()).long()
    i0 = torch.minimum(i0, torch.tensor([max(gi - 2, 0) for gi in g]))
    i1 = torch.minimum(i0 + 1, torch.tensor([gi - 1 for gi in g]))
    return i0, i1, qc - i0.to(q.dtype), live


def _corners(i0, i1):
    for c in range(8):
        yield c, [(i1 if (c >> a) & 1 else i0)[..., a] for a in range(3)]


def lookup(u, q):
    """The clamped trilinear interpolant of u (Bf, g0, g1, g2, 3) at lattice coordinates q (Bf, ..., 3) -> (Bf, ..., 3)."""
    Bf, g = u.shape[0], tuple(u.shape[1:4])
    i0, i1, f, _ = _cell(q, g)
    flat = u.reshape(Bf, -1, 3)
    out = 0.0
    for c, idx in _corners(i0, i1):
        w = 1.0
        for a in range(3):
            w = w * (f[..., a] if (c >> a) & 1 else 1.0 - f[..., a])
        n = ((idx[0] * g[1] + idx[1]) * g[2] + idx[2]).reshape(Bf, -1)
        v = torch.gather(flat, 1, n[..., None].expand(-1, -1, 3)).reshape(q.shape)
        out = out + w[..., None] * v
    return out


def square(u, s, D):
    """One squaring step u'(x) = s u(x) + s U(x + s u(x)), U the clamped interpolant of u."""
    g = u.shape[1:4]
    sc = torch.tensor([g[a] / D[a] for a in range(3)], dtype=u.dtype)
    idx = torch.stack(torch.meshgrid(*[torch.arange(gi, dtype=u.dtype) for gi in g], indexing="ij"), -1)
    q = idx + s * u * sc
    return s * (u + lookup(u, q))


def scales(steps):
    return [2.0**-steps] + [1.0] * (steps - 1)


def exp(v, steps, D):
    """exp(v) by `steps` squarings: -> the displacement (the last level)."""
    u = _t(v)
    for s in scales(steps):
        u = square(u, s, D)
    return u


def square_bwd(u, gp, s, D):
    """The adjoint of square in closed form (svf_math.cuh's): node x gets s g'(x) + s^2 J_U(y)^T g'(x), J zero along a clamped
    axis, and each corner c of y's cell gets s w_c(y) g'(x)."""
    u, gp = _t(u), _t(gp)
    Bf, g = u.shape[0], tuple(u.shape[1:4])
    sc = torch.tensor([g[a] / D[a] for a in range(3)], dtype=u.dtype)
    idx = torch.stack(torch.meshgrid(*[torch.arange(gi, dtype=u.dtype) for gi in g], indexing="ij"), -1)
    q = idx + s * u * sc
    i0, i1, f, live = _cell(q, g)
    flat = u.reshape(Bf, -1, 3)
    out = (s * gp).reshape(Bf, -1, 3).clone()
    J = torch.zeros(q.shape + (3,), dtype=u.dtype)   # J[..., i, a] = dU_i / dy_a
    for c, cidx in _corners(i0, i1):
        w, dw = 1.0, [1.0, 1.0, 1.0]
        for a in range(3):
            fa = f[..., a] if (c >> a) & 1 else 1.0 - f[..., a]
            w = w * fa
            for b in range(3):
                dw[b] = dw[b] * (((1.0 if (c >> a) & 1 else -1.0) * torch.ones_like(fa)) if a == b else fa)
        n = ((cidx[0] * g[1] + cidx[1]) * g[2] + cidx[2]).reshape(Bf, -1)
        v = torch.gather(flat, 1, n[..., None].expand(-1, -1, 3)).reshape(q.shape)
        for a in range(3):
            J[..., a] += v * (dw[a] * sc[a] * live[..., a].to(u.dtype))[..., None]
        out.scatter_add_(1, n[..., None].expand(-1, -1, 3), (s * w[..., None] * gp).reshape(Bf, -1, 3))
    out += (s * s * torch.einsum("...ia,...i->...a", J, gp)).reshape(Bf, -1, 3)
    return out.reshape(u.shape)


def exp_bwd(v, g, steps, D):
    """The gradient of sum(g * exp(v)) with respect to v, by square_bwd through the levels in reverse."""
    levels = [_t(v)]
    for s in scales(steps)[:-1]:
        levels.append(square(levels[-1], s, D))
    g = _t(g)
    for u, s in zip(reversed(levels), reversed(scales(steps))):
        g = square_bwd(u, g, s, D)
    return g


def affine_identity(L, steps, x):
    """((I + L / 2^N)^(2^N) - I) [x; 1] for a (3, 4) voxel-space generator L at points x (..., 3): what trilinear scaling and
    squaring gives for v = L [x; 1] wherever every trajectory stays inside the lattice."""
    L = _t(L)
    E = torch.eye(4, dtype=torch.float64)
    E[:3] += L / 2.0**steps
    P = torch.linalg.matrix_power(E, 2**steps) - torch.eye(4, dtype=torch.float64)
    xh = torch.cat([_t(x), torch.ones(x.shape[:-1] + (1,), dtype=torch.float64)], -1)
    return xh @ P[:3].T


def jacobian_det(u, D):
    """det of the grad of phi = id + u at the interior nodes, by central differences in voxel units: (Bf, g0-2, g1-2, g2-2)."""
    u = _t(u)
    g = u.shape[1:4]
    h = [D[a] / g[a] for a in range(3)]
    cols = []
    for a in range(3):
        sl_p = [slice(1, -1)] * 3
        sl_m = [slice(1, -1)] * 3
        sl_p[a], sl_m[a] = slice(2, None), slice(None, -2)
        cols.append((u[(slice(None), *sl_p)] - u[(slice(None), *sl_m)]) / (2 * h[a]))
    Jm = torch.stack(cols, -1) + torch.eye(3, dtype=u.dtype)   # [..., i, a]
    return torch.linalg.det(Jm)
