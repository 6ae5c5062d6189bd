"""fp64 reference of the tangent of the scaling-and-squaring exponential (csrc/svf_math.cuh's svf_square_node_jvp; DESIGN.md 6n)
in closed form, on svf_oracle.py's fields (Bf, g0, g1, g2, 3) in voxel-index units: one step's tangent along t is
    t'(x) = s t(x) + s^2 J_U(y) t(x) + s sum_c w_c(y) t(c),      y = x + s u(x),
J_U the clamped interpolant's spatial gradient (zero along a clamped axis) and w_c the weights of y's clamped cell."""
import torch

import svf_oracle as so


def square_jvp(u, t, s, D):
    """The tangent of so.square at u along t, in closed form."""
    u, t = so._t(u), so._t(t)
    Bf, g = u.shape[0], tuple(u.shape[1:4])
    sc = torch.tensor([g[a] / D[a] for a in range(3)], dtype=u.dtype)
    idx = torch.stack(torch.meshgrid(*[torch.arange(gi, dtype=u.dtype) for gi in g], indexing="ij"), -1)
    q = idx + s * u * sc
    i0, i1, f, live = so._cell(q, g)
    flat = u.reshape(Bf, -1, 3)
    J = torch.zeros(q.shape + (3,), dtype=u.dtype)   # J[..., i, a] = dU_i / dy_a
    for c, cidx in so._corners(i0, i1):
        dw = [1.0, 1.0, 1.0]
        for a in range(3):
            fa = f[..., a] if (c >> a) & 1 else 1.0 - f[..., a]
            for b in range(3):
                dw[b] = dw[b] * (((1.0 if (c >> a) & 1 else -1.0) * torch.ones_like(fa)) if a == b else fa)
        n = ((cidx[0] * g[1] + cidx[1]) * g[2] + cidx[2]).reshape(Bf, -1)
        v = torch.gather(flat, 1, n[..., None].expand(-1, -1, 3)).reshape(q.shape)
        for a in range(3):
            J[..., a] += v * (dw[a] * sc[a] * live[..., a].to(u.dtype))[..., None]
    return s * t + s * s * torch.einsum("...ia,...a->...i", J, t) + s * so.lookup(t, q)


def exp_jvp(v, t, steps, D):
    """exp(v) and its tangent along t: square_jvp through the levels -> (exp(v), d exp(v))."""
    u, t = so._t(v), so._t(t)
    for s in so.scales(steps):
        u, t = so.square(u, s, D), square_jvp(u, t, s, D)
    return u, t
