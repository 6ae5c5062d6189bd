"""CPU checks of the per-pixel pose Jacobian (DRR.jacobian; csrc/jacobian.cu): the float64 tangents of every parameterization
against central differences, the kernels' per-pixel math (compiled for the host) against a NumPy statement of the chain rule and
against the adjoint of the pose-in backward's sums, argument validation of the new entry points, and the rejections that need
no device."""
import ctypes

import numpy as np
import pytest
import torch

from diffdrr_b200 import DRR, synthetic
from diffdrr_b200.drr import pose_in_matrices
from diffdrr_b200.jacobian import pose_in_tangents
from diffdrr_b200.pose import PARAMETERIZATIONS, RigidTransform, convert
from hostemu import emu_jacobian

_CALIB = torch.tensor([[[1.1, 0.02, 0.0, 3.0], [0.0, 0.9, 0.0, -2.0], [0.0, 0.0, 1.0, 0.5], [0.0, 0.0, 0.0, 1.0]]],
                      dtype=torch.float64)


def _drr(n=16, h=12, **kw):
    return DRR(synthetic.make_subject(synthetic.make_volume(n, "smooth")), **synthetic.detector_kwargs(h), **kw)


def _params(par, degrees, B=3, seed=1):
    rot, xyz = synthetic.make_poses(B, seed=seed)
    pose = RigidTransform(convert(rot, xyz, parameterization="euler_angles", convention="ZXY").matrix.double())
    rot, xyz = pose.convert(par, convention="ZXY", degrees=degrees)
    g = torch.Generator().manual_seed(seed)
    # off the manifold the convert() of the over-parameterised forms still has a derivative: test there too
    return rot + 0.01 * torch.randn(rot.shape, generator=g, dtype=rot.dtype), xyz


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("calibrated", [False, True])
@pytest.mark.parametrize("par,degrees", [(p, False) for p in PARAMETERIZATIONS if p != "matrix"] + [("euler_angles", True)])
def test_tangents_match_central_differences(par, degrees, calibrated, B):
    drr = _drr()
    det = drr.detector
    calib = _CALIB if calibrated else det._calibration
    rot, xyz = _params(par, degrees, B=B)
    dsrc, dG, dWd = pose_in_tangents(rot, xyz, par, "ZXY", degrees, det._reorient, calib, drr._affine_inverse)
    nr = rot.shape[1]
    assert dsrc.shape == (B, nr + 3, 3) and dG.shape == (B, nr + 3, 3, 4) and dWd.dtype == torch.float64

    def f(theta):
        P = convert(theta[:, :nr], theta[:, nr:], parameterization=par, convention="ZXY", degrees=degrees).matrix
        return torch.cat([t.flatten(1) for t in pose_in_matrices(P, det._reorient.double(), calib.double(),
                                                                    drr._affine_inverse.double())],
                         dim=1)

    theta, h = torch.cat([rot, xyz], dim=1), 1e-6
    fds, gots = [], []
    for k in range(nr + 3):
        e = torch.zeros_like(theta)
        e[:, k] = h
        fds.append((f(theta + e) - f(theta - e)) / (2 * h))
        gots.append(torch.cat([dsrc[:, k], dG[:, k].flatten(1), dWd[:, k].flatten(1)], dim=1))
    fd, got = torch.stack(fds, dim=1), torch.stack(gots, dim=1)  # relative to the largest derivative of the rotation / translation
    for sl in (slice(0, nr), slice(nr, nr + 3)):
        assert float((got[:, sl] - fd[:, sl]).abs().max() / fd[:, sl].abs().max()) < 1e-6, par


def _pixel_grid(H, W, rng):
    return np.sort(rng.uniform(-100, 100, H)).astype(np.float32), np.sort(rng.uniform(-100, 100, W)).astype(np.float32)


def _problem(tri, B=2, H=5, W=7, P=6, seed=0):
    rng = np.random.default_rng(seed)
    sens = rng.standard_normal((B, H * W, 12 if tri else 8)).astype(np.float32)
    if not tri:
        sens[..., 7] = 0.0
    else:
        sens[..., 9:] = 0.0
    rows, cols = _pixel_grid(H, W, rng)
    Wd = rng.standard_normal((B, 3, 4)).astype(np.float32)
    Wd[:, :, 3] += 900.0  # a source-to-detector offset dominates the world ray, as for a real C-arm
    tang = [rng.standard_normal(s).astype(np.float32) for s in ((B, P, 3), (B, P, 3, 4), (B, P, 3, 4))]
    drange = rng.standard_normal((B, 2, P)).astype(np.float32) if tri else None
    return sens, Wd, rows, cols, tang, drange


def _np_jacobian(sens, Wd, rows, cols, dsrc, dG, dWd, drange, stop_grad):
    """The chain rule of include/b200drr.h (b200drr_*_jac_sens_pose) in float64."""
    sens, Wd, dsrc, dG, dWd = (np.asarray(a, np.float64) for a in (sens, Wd, dsrc, dG, dWd))
    H, W = len(rows), len(cols)
    p = np.stack([np.tile(cols, H), np.repeat(rows, W), np.ones(H * W), np.ones(H * W)], axis=-1).astype(np.float64)
    dl = np.einsum("bij,nj->bni", Wd, p)
    J = np.einsum("bni,bkij,nj->bnk", sens[..., :3], dG, p) + np.einsum("bni,bki->bnk", sens[..., 4:7], dsrc)
    if not stop_grad:
        J += (sens[..., 3] / np.linalg.norm(dl, axis=-1))[..., None] * np.einsum("bni,bkij,nj->bnk", dl, dWd, p)
    if drange is not None:
        J += sens[..., 7, None] * drange[:, None, 0, :] + sens[..., 8, None] * drange[:, None, 1, :]
    return J


def _np_bwd_sums(sens, Wd, rows, cols, g, stop_grad, tri):
    """sens_bwd_pose_kernel / trilinear_sens_bwd_pose_kernel's per-pose sums in float64: (g_src, g_G, g_Wd, g_alpha_range per
    pose -- the kernel adds the last over the poses)."""
    sens, Wd, g = (np.asarray(a, np.float64) for a in (sens, Wd, g))
    H, W = len(rows), len(cols)
    p = np.stack([np.tile(cols, H), np.repeat(rows, W), np.ones(H * W), np.ones(H * W)], axis=-1).astype(np.float64)
    dl = np.einsum("bij,nj->bni", Wd, p)
    gl = np.zeros_like(g) if stop_grad else g * sens[..., 3] / np.linalg.norm(dl, axis=-1)
    g_G = np.einsum("bn,bni,nj->bij", g, sens[..., :3], p)
    g_Wd = np.einsum("bn,bni,nj->bij", gl, dl, p)
    g_src = np.einsum("bn,bni->bi", g, sens[..., 4:7])
    g_ar = np.einsum("bn,bni->bi", g, sens[..., 7:9]) if tri else None
    return g_src, g_G, g_Wd, g_ar


@pytest.mark.parametrize("tri,stop_grad,P", [(False, False, 6), (False, True, 6), (False, False, 16), (True, False, 7),
                                             (True, False, 1)])
def test_kernel_math_matches_numpy_and_the_adjoint_of_the_backward(tri, stop_grad, P):
    sens, Wd, rows, cols, (dsrc, dG, dWd), drange = _problem(tri, P=P)
    J = emu_jacobian.jac_sens_pose(sens, dsrc, dG, dWd, Wd, rows, cols, drange, stop_grad)
    ref = _np_jacobian(sens, Wd, rows, cols, dsrc, dG, dWd, drange, stop_grad)
    assert J.shape == ref.shape == (2, 35, P)
    assert np.abs(J - ref).max() / np.abs(ref).max() < 1e-5
    # adjoint identity: sum_n g_n J[n, k] == <the backward's reduced gradients, tangent k>
    g = np.random.default_rng(3).standard_normal(J.shape[:2])
    lhs = np.einsum("bn,bnk->bk", g, J.astype(np.float64))
    g_src, g_G, g_Wd, g_ar = _np_bwd_sums(sens, Wd, rows, cols, g, stop_grad, tri)
    rhs = (np.einsum("bi,bki->bk", g_src, dsrc) + np.einsum("bij,bkij->bk", g_G, dG) + np.einsum("bij,bkij->bk", g_Wd, dWd))
    if tri:
        rhs += np.einsum("bi,bik->bk", g_ar, drange)
    assert np.abs(lhs - rhs).max() / np.abs(rhs).max() < 1e-5


def test_entry_points_reject_bad_arguments_without_gpu():
    from diffdrr_b200 import _lib
    from diffdrr_b200 import build as b200build

    b200build.build()
    lib = _lib.load()
    buf = (ctypes.c_float * 64)()
    p, n = ctypes.cast(buf, ctypes.c_void_p), None
    ok = (p,) * 8
    assert lib.b200drr_siddon_jac_sens_pose(n, n, n, n, n, n, n, n, 1, 2, 2, 6, 0, n) == -1
    assert lib.b200drr_trilinear_jac_sens_pose(n, n, n, n, n, n, n, n, n, 1, 2, 2, 6, n) == -1
    for i in range(8):  # any single null pointer
        args = list(ok)
        args[i] = None
        assert lib.b200drr_siddon_jac_sens_pose(*args, 1, 2, 2, 6, 0, n) == -1
    for i in range(9):
        args = [p] * 9
        args[i] = None
        assert lib.b200drr_trilinear_jac_sens_pose(*args, 1, 2, 2, 6, n) == -1
    for B, H, W, P in ((1, 2, 2, 0), (1, 2, 2, 17), (1, 2, 2, -1), (0, 2, 2, 6), (65536, 2, 2, 6), (1, 0, 2, 6), (1, 2, -3, 6)):
        assert lib.b200drr_siddon_jac_sens_pose(*ok, B, H, W, P, 0, n) == -1, (B, H, W, P)
        assert lib.b200drr_trilinear_jac_sens_pose(*ok, p, B, H, W, P, n) == -1, (B, H, W, P)


def test_jacobian_rejects_unsupported_requests_before_any_launch():
    rot, xyz = synthetic.make_poses(2)
    kw = dict(parameterization="euler_angles", convention="ZXY")
    drr = _drr()
    with pytest.raises(ValueError, match="parameterization"):
        drr.jacobian(rot, xyz, parameterization=None)
    with pytest.raises(ValueError, match="parameterization"):
        drr.jacobian(convert(rot, xyz, **kw).matrix, parameterization="matrix")
    with pytest.raises(ValueError, match="one batch size"):
        drr.jacobian(rot[:1], xyz, **kw)
    with pytest.raises(NotImplementedError, match="sub-sampled"):
        _drr(p_subsample=0.5).jacobian(rot, xyz, **kw)
    with pytest.raises(NotImplementedError, match="patch_size"):
        _drr(patch_size=4).jacobian(rot, xyz, **kw)
    with pytest.raises(NotImplementedError, match="default options"):
        _drr(mode="bilinear").jacobian(rot, xyz, **kw)
    with pytest.raises(NotImplementedError, match="default options"):
        _drr(reducefn="max").jacobian(rot, xyz, **kw)
    with pytest.raises(NotImplementedError, match="default options"):
        _drr(renderer="trilinear", reducefn="max").jacobian(rot, xyz, **kw)
    with pytest.raises(NotImplementedError, match="fp64"):
        drr.to(torch.float64).jacobian(rot.double(), xyz.double(), **kw)
    from diffdrr_b200 import _lib
    with pytest.raises(_lib.B200DRRError, match="no CPU fallback"):
        _drr().jacobian(rot, xyz, **kw)
