"""Reference of the deformable render's transpose in the density (DESIGN.md 6l) in numpy, built on deform_oracle's march and
scatter: for a fixed camera and field the image is linear in V,
    I_n = L_n step sum_m tri(V, y_m),      y_m = x_m + u(x_m),
so the gradient of sum_n gout_n I_n with respect to V is the backprojection
    g_V[corner] = sum over the poses, rays and samples of gout_n L_n step tri_weight(corner, y_m).
`dtype` selects the fp32 or the fp64 (ground truth) evaluation.  TEST INFRASTRUCTURE ONLY."""
import numpy as np

import deform_oracle as do


def bproj(vol, src, tgt, raylen, U, gout, n_points, alphamin, alphamax, voxel_shift=0.5, eps=1e-8, dtype=np.float64):
    """deform_oracle.bwd's arguments -> g_V, the volume's shape, summed over the poses (shared or per-pose fields alike)."""
    dtype = np.dtype(dtype).type
    q = do._march(vol, src, tgt, U, n_points, alphamin, alphamax, voxel_shift, eps, dtype)
    step = dtype(alphamax - alphamin) / dtype(n_points - 1)
    c = np.asarray(gout, dtype) * np.asarray(raylen, dtype) * step                  # (B, N)
    y = q["y"] + dtype(voxel_shift - 0.5)                                           # volume array coordinates
    vals = np.broadcast_to(c[:, :, None, None], y.shape[:-1] + (1,))
    shape = np.asarray(vol).shape
    return sum(do._scatter(shape, y[b], np.ascontiguousarray(vals[b]))[0] for b in range(y.shape[0]))
