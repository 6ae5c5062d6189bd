"""fp64 reference of the log-Euclidean blended-rigid motion Jacobian (DESIGN.md 6p), in torch, built only on the library's
se3_log_matrix and the test suite's svf_oracle / deform_oracle.  The motions are voxel-space maps M_k = A^-1 X_k^-1 A with A = I
(world = voxel index), so the increment X_k(xi) = T(c_k) exp(xi^) T(-c_k) X_k acts as M_k(xi) = M_k T(c_k) exp(-xi^) T(-c_k).
TEST INFRASTRUCTURE ONLY.

Shapes: M (Bm, K, 4, 4); weights (K, g0, g1, g2); pivots (K, 3); xi (Bm, K, 6); fields (Bm, g0, g1, g2, 3) voxel units; tangents
(Bm, g0, g1, g2, 6K, 3), p = 6k + i."""
import numpy as np
import torch

import deform_oracle as do
import svf_oracle as so
from polyrigid_oracle import _tri
from diffdrr_b200.structures import twist_matrix
from diffdrr_b200.svf import se3_log_matrix


def _T(c):
    out = torch.eye(4, dtype=torch.float64).repeat(*c.shape[:-1], 1, 1)
    out[..., :3, 3] = c
    return out


def velocity(M, weights, pivots, xi, D):
    """v(x) = sum_k w_k(x) log(M_k(xi)) [x; 1] at the lattice nodes -> (Bm, g0, g1, g2, 3)."""
    Mx = M @ _T(pivots) @ torch.linalg.matrix_exp(-twist_matrix(xi)) @ _T(-pivots)
    L = se3_log_matrix(Mx)[..., :3, :]                                     # (Bm, K, 3, 4)
    g = tuple(weights.shape[1:])
    x = torch.nn.functional.pad(so.node_coords(g, D), (0, 1), value=1.0)   # (g0, g1, g2, 4)
    w = torch.as_tensor(np.asarray(weights), dtype=torch.float64)
    return torch.einsum("kxyz,bkrc,xyzc->bxyzr", w, L, x)


def tangents(M, weights, pivots, steps, D):
    """(exp(v), its derivatives along the 6K increments at xi = 0) by torch.func.jacfwd through svf_oracle.exp."""
    Bm, K = M.shape[:2]
    out, tans = [], []
    for b in range(Bm):
        f = lambda xi: so.exp(velocity(M[b:b + 1], weights, pivots, xi[None], D), steps, D)[0]   # noqa: E731
        xi0 = torch.zeros(K, 6, dtype=torch.float64)
        out.append(f(xi0))
        tans.append(torch.func.jacfwd(f)(xi0).reshape(*out[-1].shape, 6 * K).movedim(-1, -2))
    return torch.stack(out), torch.stack(tans)


def jacobian(c, U, T, K):
    """J (B, K, N, 6) = L step sum_m G_m . t_p(x_m) over deform_oracle's march of the field U (Bm, g0, g1, g2, 3) for the rays of
    case c, T its tangents (Bm, g0, g1, g2, 6K, 3); G and t_p are zero on the samples the kernel skips."""
    U, T = np.asarray(U, np.float64), np.asarray(T, np.float64)
    q = do._march(c["vol"], c["src"], c["tgt"], np.moveaxis(U, -1, 1), c["n_points"], c["amin"], c["amax"], 0.5, 1e-8, np.float64)
    B = q["q"].shape[0]
    Tc = np.moveaxis(T.reshape(*T.shape[:4], -1), -1, 1)                  # (Bm, 6K * 3, g0, g1, g2)
    t = np.stack([_tri(Tc[b if Tc.shape[0] > 1 else 0], q["q"][b])[0] for b in range(B)])   # (B, N, P, 6K * 3)
    t = t.reshape(*t.shape[:3], 6 * K, 3)
    step = (c["amax"] - c["amin"]) / (c["n_points"] - 1)
    J = np.asarray(c["raylen"], np.float64)[..., None] * step * np.einsum("bnma,bnmpa->bnp", q["G"], t)
    return np.moveaxis(J.reshape(B, -1, K, 6), 2, 1)


def image(c, U):
    return do.fwd(c["vol"], c["src"], c["tgt"], c["raylen"], np.moveaxis(np.asarray(U, np.float64), -1, 1), c["n_points"], c["amin"],
                  c["amax"])
