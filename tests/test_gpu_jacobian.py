"""GPU tests of DRR.jacobian (csrc/jacobian.cu + the float64 pose tangents) and the Levenberg-Marquardt step built on it:
the image is the one drr(...) renders, sum_n g_n J[n] equals autograd's pose gradient of sum g * drr(...) through the existing,
golden-pinned backward (the adjoint identity), a float64 central difference agrees, unsupported requests raise, and LM reaches
the registration test's bounds."""
import numpy as np
import pytest
import torch

from gpu_common import DEV, relerr

pytestmark = pytest.mark.gpu

_KW = dict(convention="ZXY")


def _drr(D, H, renderer="siddon", dtype=torch.float32, kind="smooth", **kw):
    from diffdrr_b200 import DRR, synthetic
    drr = DRR(synthetic.make_subject(synthetic.make_volume(D, kind, seed=2)), **synthetic.detector_kwargs(H), renderer=renderer,
              **kw).to(DEV)
    if dtype != torch.float32:
        drr.density = drr.density.to(dtype)
    return drr


def _params(par, B, degrees=False, seed=3):
    from diffdrr_b200 import synthetic
    from diffdrr_b200.pose import RigidTransform, convert
    rot, xyz = synthetic.make_poses(B, seed=seed, rot_range=0.3, xyz_range=20.0)
    pose = RigidTransform(convert(rot.double(), xyz.double(), parameterization="euler_angles", convention="ZXY").matrix)
    rot, xyz = pose.convert(par, convention="ZXY", degrees=degrees)
    # a generic point: on the rotation manifold the SVD / eigh of rotation_9d / _10d have repeated values
    rot = rot + 0.01 * torch.randn(rot.shape, generator=torch.Generator().manual_seed(seed), dtype=rot.dtype)
    return rot.float().to(DEV).contiguous(), xyz.float().to(DEV).contiguous()


def _adjoint(drr, rot, xyz, par, degrees=False, calibration=None, n_points=500):
    """(lhs, rhs, img, img_ref): sum_n g J (+ the assembled Trilinear cross-pose range terms) and autograd's gradient."""
    kw = dict(parameterization=par, degrees=degrees, calibration=calibration, **_KW)
    tri = drr.renderer.__class__.__name__ == "Trilinear"
    if tri:
        kw["n_points"] = n_points
    img, J, (dmin, dmax, drange) = drr.jacobian(rot, xyz, return_range_terms=True, **kw)
    assert not img.requires_grad and not J.requires_grad and J.shape == (*img.shape, rot.shape[1] + 3)
    g = torch.randn(img.shape, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    lhs = torch.einsum("bchw,bchwk->bk", g.double(), J.double())
    if tri:  # pose c's parameters move every image through the range when c owns an extreme ray
        sm, sM = (g.double() * dmin.double()).flatten(1).sum(1), (g.double() * dmax.double()).flatten(1).sum(1)
        own = drange.double() * torch.stack([sm, sM], dim=1)[:, :, None]
        lhs = lhs + drange[:, 0].double() * sm.sum() + drange[:, 1].double() * sM.sum() - own.sum(1)
    r, x = rot.clone().requires_grad_(True), xyz.clone().requires_grad_(True)
    ref = drr(r, x, **kw)
    gr, gx = torch.autograd.grad((g * ref).sum(), (r, x))
    return lhs, torch.cat([gr, gx], dim=1).double(), img, ref.detach()


def _check(drr, rot, xyz, par, bound=1e-5, reruns=False, **kw):
    lhs, rhs, img, ref = _adjoint(drr, rot, xyz, par, **kw)
    assert relerr(img.cpu().numpy(), ref.cpu().numpy()) < 1e-6
    if reruns:  # the brick route sums the sensitivities with atomics: allow 3x the run-to-run spread of the gradient
        spread = max(relerr(_adjoint(drr, rot, xyz, par, **kw)[1].cpu().numpy(), rhs.cpu().numpy()) for _ in range(3))
        bound = max(bound, 3.0 * spread)
    err = relerr(lhs.cpu().numpy(), rhs.cpu().numpy())
    assert err < bound, f"adjoint identity: {err:.3e} (bound {bound:.1e})"


@pytest.mark.parametrize("stop_grad", [False, True])
@pytest.mark.parametrize("B", [1, 16])
def test_siddon_adjoint_identity_512(B, stop_grad):
    """512^3 -> 256^2: the major-axis pieces at one pose, the brick route at 16."""
    drr = _drr(512, 256, stop_gradients_through_grid_sample=stop_grad)
    rot, xyz = _params("euler_angles", B)
    _check(drr, rot, xyz, "euler_angles", reruns=B > 1)


_PARS = ["axis_angle", "euler_angles", "quaternion", "quaternion_adjugate", "rotation_6d", "rotation_9d", "rotation_10d",
         "se3_log_map"]


@pytest.mark.parametrize("par", _PARS)
def test_every_parameterization(par):
    drr = _drr(96, 64)
    rot, xyz = _params(par, 2)
    # the reference gradient of rotation_9d / _10d runs autograd through convert()'s fp32 SVD / eigh, which alone moved it by
    # 1.4e-5 to 4.8e-5 of its maximum on the H100; the float64 tangents are pinned to central differences on the CPU
    _check(drr, rot, xyz, par, bound=1e-4 if par in ("rotation_9d", "rotation_10d") else 1e-5)


def test_degrees_and_calibration():
    from diffdrr_b200.pose import RigidTransform
    drr = _drr(96, 64)
    rot, xyz = _params("euler_angles", 2, degrees=True)
    _check(drr, rot, xyz, "euler_angles", degrees=True)
    calib = torch.eye(4, device=DEV)
    calib[0, 0], calib[1, 1], calib[0, 3], calib[1, 3] = 1.05, 0.95, 2.0, -3.0
    rot, xyz = _params("euler_angles", 2)
    _check(drr, rot, xyz, "euler_angles", calibration=RigidTransform(calib))


@pytest.mark.parametrize("renderer", ["siddon", "trilinear"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_16bit_density(renderer, dtype):
    drr = _drr(96, 64, renderer=renderer, dtype=dtype)
    rot, xyz = _params("euler_angles", 2)
    _check(drr, rot, xyz, "euler_angles", n_points=77)


@pytest.mark.parametrize("n_points", [77, 500])
@pytest.mark.parametrize("B", [1, 4])
def test_trilinear_adjoint_identity(B, n_points):
    drr = _drr(128, 96, renderer="trilinear")
    rot, xyz = _params("euler_angles", B)
    _check(drr, rot, xyz, "euler_angles", n_points=n_points)


@pytest.mark.parametrize("renderer", ["siddon", "trilinear"])
def test_float64_central_difference(renderer):
    """Independent of every fp32 kernel: the fp64 reference-literal renderer, differenced along a random direction of theta."""
    drr = _drr(128, 64, renderer=renderer)
    rot, xyz = _params("euler_angles", 1)
    img, J = drr.jacobian(rot, xyz, parameterization="euler_angles", **_KW)
    gen = torch.Generator(device=DEV).manual_seed(11)
    # positive weights: a random-sign g cancels the sum down to the level of the kinks below
    g = 1.0 + torch.rand(img.shape, generator=gen, device=DEV).double()
    d = torch.randn(1, 6, generator=gen, device=DEV).double()
    d[:, 3:] *= 10.0  # mm next to radians
    d64 = drr.to(torch.float64)
    # both images are piecewise smooth in theta (kinks where a ray or a sample crosses a voxel face): a small step
    h = 1e-6
    with torch.no_grad():
        f = lambda t: (g * d64(rot.double() + t * d[:, :3], xyz.double() + t * d[:, 3:], parameterization="euler_angles",  # noqa: E731
                               **_KW)).sum()
        fd = float((f(h) - f(-h)) / (2 * h))
    an = float((g * (J.double() @ d[0])).sum())
    assert abs(an - fd) < 1e-3 * abs(fd), (an, fd)


def test_rejections_before_any_launch():
    from diffdrr_b200 import synthetic
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2))
    kw = dict(parameterization="euler_angles", **_KW)
    for bad in (dict(p_subsample=0.5), dict(patch_size=8), dict(mode="bilinear"), dict(reducefn="max"),
                dict(filter_intersections_outside_volume=True)):
        with pytest.raises(NotImplementedError):
            _drr(32, 16, **bad).jacobian(rot, xyz, **kw)
    with pytest.raises(ValueError):
        _drr(32, 16).jacobian(rot, xyz, parameterization=None)
    with pytest.raises(NotImplementedError, match="fp64"):
        _drr(32, 16).to(torch.float64).jacobian(rot.double(), xyz.double(), **kw)
    tri = _drr(32, 16, renderer="trilinear")
    tri.renderer.pack_corners = False
    with pytest.raises(NotImplementedError, match="packed"):
        tri.jacobian(rot, xyz, **kw)
    tri = _drr(32, 16, renderer="trilinear")
    tri.density.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="packed"):
        tri.jacobian(rot, xyz, **kw)


@pytest.mark.parametrize("renderer", ["siddon", "trilinear"])
def test_no_host_synchronisation(renderer):
    drr = _drr(64, 32, renderer=renderer)
    rot, xyz = _params("euler_angles", 2)
    kw = dict(parameterization="euler_angles", **_KW)
    drr.jacobian(rot, xyz, **kw)  # first call: caches, packing, module loads
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            drr.jacobian(rot, xyz, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def _lm_run(steps=30):
    """LM from the Adam registration test's start: (final 1 - NCC, rotation error, translation error, steps taken)."""
    from test_gpu_registration import _problem

    from diffdrr_b200 import LevenbergMarquardt
    drr, reg, ncc, target, true_rot, true_xyz = _problem()
    rot_id, xyz_id = id(reg.rotation), id(reg.translation)
    lm = LevenbergMarquardt(reg, target)
    history = []
    for it in range(steps):
        history.append(float(lm.step()))
        rot_err = float((reg.rotation.detach() - true_rot).abs().max())
        xyz_err = float((reg.translation.detach() - true_xyz).abs().max())
        if history[-1] < 1e-3 and rot_err < 0.02 and xyz_err < 2.0:
            break
    assert id(reg.rotation) == rot_id and id(reg.translation) == xyz_id  # updated in place: an optimizer can take over
    with torch.no_grad():
        final = float(1.0 - ncc(target, reg()).mean())
    assert np.isclose(final, history[-1], rtol=1e-3, atol=1e-6)  # step() returns the loss of the pose it leaves
    print(f"LM: {it + 1} steps, 1-NCC {final:.2e}, rotation error {rot_err:.2e} rad, translation error {xyz_err:.3f} mm; "
          f"loss history {['%.2e' % h for h in history]}")
    return final, rot_err, xyz_err, it + 1


def test_levenberg_marquardt_reaches_the_loss_and_translation_bounds():
    final, _, xyz_err, _ = _lm_run()
    assert final < 1e-3 and xyz_err < 2.0


@pytest.mark.xfail(strict=True, reason="within 30 steps LM reaches 1 - NCC ~1.5e-5 and ~0.5 mm but stops ~0.04 rad off in "
                                       "rotation, outside the Adam test's 0.02 rad (README)")
def test_levenberg_marquardt_reaches_all_registration_bounds():
    final, rot_err, xyz_err, steps = _lm_run()
    assert final < 1e-3 and rot_err < 0.02 and xyz_err < 2.0, \
        f"after {steps} LM steps: 1-NCC {final:.2e}, rotation error {rot_err:.3e} rad, translation error {xyz_err:.2f} mm"
