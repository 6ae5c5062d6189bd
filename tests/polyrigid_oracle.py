"""Reference implementation of the blended-rigid (skinned) trilinear render (DESIGN.md 6h) in numpy: a literal restatement of the
model, vectorised over every sample of every ray, with no sample-range skipping and no code shared with the kernels.  `dtype`
selects the fp32 or the fp64 (ground truth) evaluation.  TEST INFRASTRUCTURE ONLY.

    x_m = s + alpha_m d,   d = t - s + eps,   alpha_m = alphamin + linspace(0, 1, P)[m] (alphamax - alphamin)
    y_m = x_m + sum_k w_k(x_m) (M_k [x_m; 1] - x_m),      I = L step sum_m tri(V, y_m),   step = (alphamax - alphamin) / (P - 1)

Shapes: vol (D0, D1, D2); src (B, 3); tgt (B, N, 3); raylen (B, N); M (Bm, K, 3, 4) with Bm in {1, B}; weights (K, g0, g1, g2).
"""
import numpy as np


def _tri(arr, p):
    """Trilinear interpolant of arr (C, n0, n1, n2), zero outside, at array coordinates p (..., 3): -> value (..., C) and gradient
    w.r.t. p (..., C, 3)."""
    dt = p.dtype
    n = np.asarray(arr.shape[1:])
    fl = np.floor(p)
    f = p - fl
    i0 = fl.astype(np.int64)
    val = np.zeros(p.shape[:-1] + (arr.shape[0],), dt)
    grad = np.zeros(p.shape[:-1] + (arr.shape[0], 3), dt)
    for o0 in (0, 1):
        for o1 in (0, 1):
            for o2 in (0, 1):
                o = np.array([o0, o1, o2])
                idx = i0 + o
                inb = np.all((idx >= 0) & (idx < n), axis=-1)
                ic = np.clip(idx, 0, n - 1)
                v = np.where(inb[..., None], np.moveaxis(arr[:, ic[..., 0], ic[..., 1], ic[..., 2]], 0, -1), 0).astype(dt)
                wa = np.where(o == 1, f, 1 - f)                 # (..., 3) per-axis weights
                da = np.where(o == 1, 1.0, -1.0).astype(dt)     # their derivatives
                val += v * wa.prod(-1)[..., None]
                for a in range(3):
                    b, c = [x for x in range(3) if x != a]
                    grad[..., a] += v * (da[a] * wa[..., b] * wa[..., c])[..., None]
    return val, grad


def _march(vol, src, tgt, M, weights, n_points, alphamin, alphamax, voxel_shift, eps, dtype):
    vol, src, tgt, M, weights = (np.asarray(a, dtype) for a in (vol, src, tgt, M, weights))
    B = tgt.shape[0]
    M = np.broadcast_to(M, (B,) + M.shape[1:])
    s = src[:, None, None, :]
    d = (tgt - src[:, None, :] + dtype(eps))[:, :, None, :]
    lin = np.linspace(0, 1, n_points, dtype=dtype)
    alpha = (lin * dtype(alphamax - alphamin) + dtype(alphamin))[None, None, :, None]
    x = s + alpha * d                                                   # (B, N, P, 3)
    kb = dtype(voxel_shift - 0.5)
    D = np.asarray(vol.shape, dtype)
    g = np.asarray(weights.shape[1:], dtype)
    u = (x + kb + dtype(0.5)) * (g / D) - dtype(0.5)
    w, gw = _tri(weights, u)                                            # (B, N, P, K), (B, N, P, K, 3)
    gw = gw * (g / D)
    off = np.einsum("bkij,bnpj->bnpki", M[..., :3], x) + M[:, None, None, :, :, 3] - x[..., None, :]   # (B, N, P, K, 3)
    y = x + (w[..., None] * off).sum(-2)
    V, G = _tri(vol[None], y + kb)
    return dict(lin=lin, alpha=alpha[..., 0], d=d[:, :, 0], w=w, gw=gw, off=off, V=V[..., 0], G=G[..., 0, :], M=M)


def fwd(vol, src, tgt, raylen, M, weights, n_points, alphamin, alphamax, voxel_shift=0.5, eps=1e-8, dtype=np.float64):
    """-> image (B, N)."""
    dtype = np.dtype(dtype).type
    q = _march(vol, src, tgt, M, weights, n_points, alphamin, alphamax, voxel_shift, eps, dtype)
    step = dtype(alphamax - alphamin) / dtype(n_points - 1)
    return np.asarray(raylen, dtype) * step * q["V"].sum(-1)


def bwd(vol, src, tgt, raylen, M, weights, gout, n_points, alphamin, alphamax, voxel_shift=0.5, eps=1e-8, dtype=np.float64):
    """Gradients of sum(gout * image) for a FIXED sampling range, plus the partials w.r.t. the range: dict(g_src (B, 3),
    g_tgt (B, N, 3), g_raylen (B, N), g_M (Bm, K, 3, 4), g_alphamin, g_alphamax)."""
    dtype = np.dtype(dtype).type
    Bm = np.asarray(M).shape[0]
    q = _march(vol, src, tgt, M, weights, n_points, alphamin, alphamax, voxel_shift, eps, dtype)
    L, gout, src = np.asarray(raylen, dtype), np.asarray(gout, dtype), np.asarray(src, dtype)
    step = dtype(alphamax - alphamin) / dtype(n_points - 1)
    c = (gout * L * step)[..., None]                                    # (B, N, 1)
    G, w, alpha, lin = q["G"], q["w"], q["alpha"], q["lin"]
    R = q["M"][..., :3]                                                 # (B, K, 3, 3)
    RtG = np.einsum("bkij,bnpi->bnpkj", R, G)
    H = G + (w[..., None] * (RtG - G[..., None, :])).sum(-2) + (q["gw"] * (q["off"] * G[..., None, :]).sum(-1, keepdims=True)).sum(-2)
    wG = w[..., None] * G[..., None, :]                                 # (B, N, P, K, 3)
    A = c[..., None] * wG.sum(2)                                        # (B, N, K, 3)
    Bv = c[..., None] * (alpha[..., None, None] * wG).sum(2)
    gM = np.zeros(q["M"].shape, dtype)
    gM[..., :3] = np.einsum("bnki,bj->bkij", A, src) + np.einsum("bnki,bnj->bkij", Bv, q["d"])
    gM[..., 3] = A.sum(1)
    if Bm == 1:
        gM = gM.sum(0, keepdims=True)
    g_tgt = c * (alpha[..., None] * H).sum(2)
    g_src = (c * ((1 - alpha)[..., None] * H).sum(2)).sum(1)
    sumV = q["V"].sum(-1)
    Hd = (H * q["d"][:, :, None, :]).sum(-1)                            # (B, N, P)
    gLv = gout * L * sumV / dtype(n_points - 1)
    gLs = gout * L * step
    return dict(g_src=g_src, g_tgt=g_tgt, g_raylen=gout * step * sumV, g_M=gM,
                g_alphamin=float((-gLv + gLs * ((1 - lin) * Hd).sum(-1)).sum()),
                g_alphamax=float((gLv + gLs * (lin * Hd).sum(-1)).sum()))
