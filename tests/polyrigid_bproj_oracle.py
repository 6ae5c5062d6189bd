"""Reference of the blended-rigid render's transpose in the density (DESIGN.md 6o) in numpy, built on polyrigid_oracle's march and
deform_oracle's scatter: for a fixed camera and fixed maps the image is linear in V,
    I_n = L_n step sum_m tri(V, y_m),      y_m = x_m + sum_k w_k(x_m) (M_k [x_m; 1] - x_m),
so the gradient of sum_n gout_n I_n with respect to V is the backprojection
    g_V[corner] = sum over the poses, rays and samples of gout_n L_n step tri_weight(corner, y_m).
`dtype` selects the fp32 or the fp64 (ground truth) evaluation.  TEST INFRASTRUCTURE ONLY."""
import numpy as np

import deform_oracle as do
import polyrigid_oracle as po


def bproj(vol, src, tgt, raylen, M, weights, gout, n_points, alphamin, alphamax, voxel_shift=0.5, eps=1e-8, dtype=np.float64):
    """polyrigid_oracle.bwd's arguments -> g_V, the volume's shape, summed over the poses (shared or per-pose maps alike)."""
    dtype = np.dtype(dtype).type
    q = po._march(vol, src, tgt, M, weights, n_points, alphamin, alphamax, voxel_shift, eps, dtype)
    # _march's sample positions: x = s + alpha d, y = x + sum_k w_k off_k, as it forms them
    x = np.asarray(src, dtype)[:, None, None, :] + q["alpha"][..., None] * q["d"][:, :, None, :]
    y = x + (q["w"][..., None] * q["off"]).sum(-2) + dtype(voxel_shift - 0.5)      # volume array coordinates
    step = dtype(alphamax - alphamin) / dtype(n_points - 1)
    c = np.asarray(gout, dtype) * np.asarray(raylen, dtype) * step                  # (B, N)
    vals = np.broadcast_to(c[:, :, None, None], y.shape[:-1] + (1,))
    shape = np.asarray(vol).shape
    return sum(do._scatter(shape, y[b], np.ascontiguousarray(vals[b]))[0] for b in range(y.shape[0]))
