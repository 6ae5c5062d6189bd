"""Reference implementation of the deformable trilinear render (DESIGN.md 6i) in numpy: a literal restatement of the model,
vectorised over every sample of every ray, with no sample-range skipping and no code shared with the kernels (the interpolant is
polyrigid_oracle's).  `dtype` selects the fp32 or the fp64 (ground truth) evaluation.  TEST INFRASTRUCTURE ONLY.

    x_m = s + alpha_m d,   d = t - s + eps,   alpha_m = alphamin + linspace(0, 1, P)[m] (alphamax - alphamin)
    y_m = x_m + u(x_m),      I = L step sum_m tri(V, y_m),   step = (alphamax - alphamin) / (P - 1)

Shapes: vol (D0, D1, D2); src (B, 3); tgt (B, N, 3); raylen (B, N); U (Bf, 3, g0, g1, g2) voxel-index displacements, Bf in {1, B}.
"""
import numpy as np

from polyrigid_oracle import _tri


def _march(vol, src, tgt, U, n_points, alphamin, alphamax, voxel_shift, eps, dtype):
    vol, src, tgt, U = (np.asarray(a, dtype) for a in (vol, src, tgt, U))
    B = tgt.shape[0]
    s = src[:, None, None, :]
    d = (tgt - src[:, None, :] + dtype(eps))[:, :, None, :]
    lin = np.linspace(0, 1, n_points, dtype=dtype)
    alpha = (lin * dtype(alphamax - alphamin) + dtype(alphamin))[None, None, :, None]
    x = s + alpha * d                                                   # (B, N, P, 3)
    kb = dtype(voxel_shift - 0.5)
    D = np.asarray(vol.shape, dtype)
    g = np.asarray(U.shape[2:], dtype)
    q = (x + kb + dtype(0.5)) * (g / D) - dtype(0.5)                    # lattice coordinates
    u, gu = zip(*[_tri(U[b if U.shape[0] > 1 else 0], q[b]) for b in range(B)])
    u, gu = np.stack(u), np.stack(gu) * (g / D)                         # (B, N, P, 3), (B, N, P, 3, 3): gu[..., c, a] = du_c/dx_a
    y = x + u
    V, G = _tri(vol[None], y + kb)
    return dict(lin=lin, alpha=alpha[..., 0], d=d[:, :, 0], q=q, y=y, gu=gu, V=V[..., 0], G=G[..., 0, :])


def fwd(vol, src, tgt, raylen, U, n_points, alphamin, alphamax, voxel_shift=0.5, eps=1e-8, dtype=np.float64):
    """-> image (B, N)."""
    dtype = np.dtype(dtype).type
    q = _march(vol, src, tgt, U, n_points, alphamin, alphamax, voxel_shift, eps, dtype)
    step = dtype(alphamax - alphamin) / dtype(n_points - 1)
    return np.asarray(raylen, dtype) * step * q["V"].sum(-1)


def _scatter(shape, p, vals):
    """Adjoint of _tri's value: sum over the points p (..., 3) of tri_weight(node, p) * vals (..., C) into an array (C, *shape)."""
    n = np.asarray(shape)
    fl = np.floor(p)
    f = p - fl
    i0 = fl.astype(np.int64)
    out = np.zeros((vals.shape[-1],) + tuple(shape), vals.dtype)
    for o0 in (0, 1):
        for o1 in (0, 1):
            for o2 in (0, 1):
                o = np.array([o0, o1, o2])
                idx = (i0 + o).reshape(-1, 3)
                w = np.where(o == 1, f, 1 - f).prod(-1).reshape(-1)
                inb = np.all((idx >= 0) & (idx < n), axis=-1)
                v = (w[:, None] * vals.reshape(-1, vals.shape[-1]))[inb]
                for c in range(vals.shape[-1]):
                    np.add.at(out[c], (idx[inb, 0], idx[inb, 1], idx[inb, 2]), v[:, c])
    return out


def bwd(vol, src, tgt, raylen, U, gout, n_points, alphamin, alphamax, voxel_shift=0.5, eps=1e-8, dtype=np.float64):
    """Gradients of sum(gout * image) for a FIXED sampling range, plus the partials w.r.t. the range: dict(g_src (B, 3),
    g_tgt (B, N, 3), g_raylen (B, N), g_U (Bf, 3, g0, g1, g2), g_alphamin, g_alphamax)."""
    dtype = np.dtype(dtype).type
    Bf = np.asarray(U).shape[0]
    q = _march(vol, src, tgt, U, n_points, alphamin, alphamax, voxel_shift, eps, dtype)
    L, gout = np.asarray(raylen, dtype), np.asarray(gout, dtype)
    B = L.shape[0]
    step = dtype(alphamax - alphamin) / dtype(n_points - 1)
    c = (gout * L * step)[..., None]                                    # (B, N, 1)
    G, alpha, lin = q["G"], q["alpha"], q["lin"]
    H = G + np.einsum("bnpca,bnpc->bnpa", q["gu"], G)                   # J^T G, J = 1 + grad u
    gsh = np.asarray(U).shape[2:]
    gU = np.stack([_scatter(gsh, q["q"][b], c[b][:, None, :] * G[b]) for b in range(B)])
    if Bf == 1:
        gU = gU.sum(0, keepdims=True)
    g_tgt = c * (alpha[..., None] * H).sum(2)
    g_src = (c * ((1 - alpha)[..., None] * H).sum(2)).sum(1)
    sumV = q["V"].sum(-1)
    Hd = (H * q["d"][:, :, None, :]).sum(-1)                            # (B, N, P)
    gLv = gout * L * sumV / dtype(n_points - 1)
    gLs = gout * L * step
    return dict(g_src=g_src, g_tgt=g_tgt, g_raylen=gout * step * sumV, g_U=gU,
                g_alphamin=float((-gLv + gLs * ((1 - lin) * Hd).sum(-1)).sum()),
                g_alphamax=float((gLv + gLs * (lin * Hd).sum(-1)).sum()))
