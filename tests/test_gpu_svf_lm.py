"""The tangent of the scaling-and-squaring exponential and diffeomorphic Levenberg-Marquardt on the GPU (DESIGN.md 6n):
b200drr_svf_square_jvp against the fp64 closed form of svf_jvp_oracle.py, its out against b200drr_svf_square bit for bit,
repeatable bits, the transpose relation with b200drr_svf_square_bwd; exp_velocity_jvp against fp64 torch.func.jvp;
DiffeomorphicLevenbergMarquardt's gradient against autograd through render_deformed(field=exp_velocity(V)), its product's symmetry,
no host sync, a non-increasing objective, the refusals, and the diffeomorphic registration scene of test_gpu_svf.py."""
import numpy as np
import pytest
import torch

import svf_jvp_oracle as sj
import svf_oracle as so
from conftest import relerr
from test_gpu_deform import _field, _scene
from test_gpu_svf import _velocity
from test_svf_cpu import CASES, SCALES, _case
from test_svf_jvp_cpu import _tangent
from diffdrr_b200 import (DRR, DiffeomorphicLevenbergMarquardt, NormalizedCrossCorrelation2d, _lib, exp_velocity, exp_velocity_jvp,
                          synthetic)
from diffdrr_b200.deform import voxel_field
from diffdrr_b200.registration import field_smoothness, ncc_z
from diffdrr_b200.renderers import _ptr, _stream
from diffdrr_b200.svf import square_chain

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
DIMS = (48, 56, 40)


def _pad(u):
    return torch.nn.functional.pad(torch.as_tensor(np.ascontiguousarray(u), dtype=torch.float32, device=DEV), (0, 1)).contiguous()


def _launch(name, field, *arrays, s, D):
    lib = _lib.load()
    _lib.check(getattr(lib, name)(_ptr(field), *map(_ptr, arrays), field.shape[0], *field.shape[1:4], *D, s, _stream()), name)


def _jvp(field, tan, s, D, primal=True):
    tout = torch.empty_like(field)
    out = torch.empty_like(field) if primal else None
    _launch("b200drr_svf_square_jvp", field, tan, tout, out, s=s, D=D)
    return tout, out


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_matches_fp64_reference_and_its_out_is_the_step(name, s):
    D, u, _ = _case(name)
    t = _tangent(name)
    field, tan = _pad(u), _pad(t)
    tout, out = _jvp(field, tan, s, D)
    ref = sj.square_jvp(u, t, s, D).numpy()
    assert torch.all(tout[..., 3] == 0)
    assert np.abs(tout[..., :3].cpu().numpy() - ref).max() <= 2e-6 * np.abs(ref).max()
    step = torch.empty_like(field)
    _launch("b200drr_svf_square", field, step, s=s, D=D)
    assert torch.equal(out, step)
    again, _ = _jvp(field, tan, s, D, primal=False)
    assert torch.equal(again, tout)   # one write per node, with or without out: bit for bit
    assert not torch.any(_jvp(field, torch.zeros_like(tan), s, D)[0])


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_is_the_transpose_of_the_adjoint_kernel(name, s):
    D, u, w = _case(name)
    field, tan, gout = _pad(u), _pad(_tangent(name)), _pad(w)
    jt, _ = _jvp(field, tan, s, D, primal=False)
    gin = torch.empty_like(field)
    _launch("b200drr_svf_square_bwd", field, gout, gin, s=s, D=D)
    lhs = float((gout.double() * jt.double()).sum())
    rhs = float((gin.double() * tan.double()).sum())
    assert lhs != 0 and abs(lhs - rhs) <= 1e-5 * abs(rhs), (lhs, rhs)


@pytest.mark.parametrize("per_pose", [False, True])
def test_exp_velocity_jvp_matches_fp64_forward_mode(per_pose):
    _, drr = _scene()
    B = 2 if per_pose else None
    v, t = _velocity(B, seed=1), _velocity(B, seed=2, amp=1.0)
    u, du = exp_velocity_jvp(drr, v, t, steps=8)
    assert u.shape == du.shape == v.shape and not u.requires_grad
    assert torch.equal(u, exp_velocity(drr, v, steps=8))
    A = drr._affine.reshape(4, 4)[:3, :3].double().cpu()
    Ainv = torch.linalg.inv(A)

    def f(w):
        wb = w if w.dim() == 5 else w[None]
        out = torch.einsum("ij,bxyzj->bixyz", A, so.exp(torch.einsum("ij,bjxyz->bxyzi", Ainv, wb), 8, DIMS))
        return out if w.dim() == 5 else out[0]

    ref_u, ref_du = torch.func.jvp(f, (v.double().cpu(),), (t.double().cpu(),))
    assert relerr(u.cpu().numpy(), ref_u.numpy()) <= 1e-5
    assert np.abs(ref_du.numpy()).max() > 0
    assert relerr(du.cpu().numpy(), ref_du.numpy()) <= 2e-5


# ---- DiffeomorphicLevenbergMarquardt ---------------------------------------------------------------------------------------------
def _lm_scene(per_pose, seed=20):
    _, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=seed))
    U_true = _field(2 if per_pose else None, seed=seed + 1, amp=6.0)
    with torch.no_grad():
        target = drr.render_deformed(rot, xyz, field=U_true, n_points=150, **KW)
    V = _field(2 if per_pose else None, seed=seed + 2, amp=2.0)
    return drr, rot, xyz, V, target


@pytest.mark.parametrize("per_pose", [False, True])
def test_model_gradient_equals_autograd_through_the_exponential(per_pose):
    """g = d/dV of (1/2N) |z(img) - z(t)|^2 (mean over views for a shared velocity, summed over the per-pose objectives)
    + smoothness R(V), img = render_deformed(field=exp_velocity(V)), by autograd."""
    drr, rot, xyz, V, target = _lm_scene(per_pose)
    lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, V.clone(), target, steps=8, smoothness=1e-2, n_points=150, **KW)
    g = lm.gradient()
    Vr = V.clone().requires_grad_(True)
    img = drr.render_deformed(rot, xyz, field=exp_velocity(drr, Vr, steps=8), n_points=150, **KW)
    N = img[0].numel()
    z, zt = ncc_z(img.reshape(2, N), lm.eps)[0], ncc_z(target.reshape(2, N), lm.eps)[0]
    per_view = ((z - zt) ** 2).sum(-1) / (2 * N)
    Vs = Vr if per_pose else Vr[None]
    E = (per_view.sum() if per_pose else per_view.mean()) + 1e-2 * field_smoothness(Vs).sum()
    E.backward()
    assert g.shape == V.shape and float(Vr.grad.abs().max()) > 0
    assert relerr(g.cpu().numpy(), Vr.grad.cpu().numpy()) <= 1e-4


@pytest.mark.parametrize("per_pose", [False, True])
def test_product_is_symmetric_and_positive(per_pose):
    drr, rot, xyz, V, target = _lm_scene(per_pose, seed=30)
    lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, V.clone(), target, n_points=150, **KW)
    v, w = _field(2 if per_pose else None, seed=31, amp=1.0), _field(2 if per_pose else None, seed=32, amp=1.0)
    Hv, Hw = lm.product(v), lm.product(w)
    a, b = float((w.double() * Hv.double()).sum()), float((Hw.double() * v.double()).sum())
    scale = float((w.double() * Hw.double()).sum() * (v.double() * Hv.double()).sum()) ** 0.5
    assert abs(a - b) <= 1e-4 * scale, (a, b, scale)   # Cauchy-Schwarz scale; both transposes sum with fp32 reductions
    for x, Hx in ((v, Hv), (w, Hw)):
        if per_pose:
            assert bool(((x * Hx).flatten(1).sum(1) >= 0).all())
        else:
            assert float((x * Hx).sum()) >= 0


@pytest.mark.parametrize("per_pose", [False, True])
def test_steps_never_increase_the_objective_and_make_no_host_sync(per_pose):
    drr, rot, xyz, V, target = _lm_scene(per_pose, seed=40)
    velocity = V.clone()
    lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, velocity, target, cg_iters=5, n_points=150, **KW)
    with torch.no_grad():
        img0 = drr.render_deformed(rot, xyz, field=exp_velocity(drr, velocity), n_points=150, **KW)
        E0 = lm._objective(img0, lm._systems(velocity))
    losses = [lm.step()]   # the first step renders the first image and sets the damping
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(9):
            losses.append(lm.step())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert losses[0].shape == (() if not per_pose else (2,))
    E = torch.stack([E0.reshape(losses[0].shape)] + losses).cpu()
    assert torch.isfinite(E).all() and bool((E[1:] <= E[:-1]).all()), E
    assert bool((E[-1] < E[0]).all())
    assert not torch.equal(velocity, V)   # updated in place
    # the kept levels are the current velocity's: its image and the returned objective are what a fresh render gives
    with torch.no_grad():
        img = drr.render_deformed(rot, xyz, field=exp_velocity(drr, velocity), n_points=150, **KW)
        assert relerr(lm._img.cpu().numpy(), img.cpu().numpy()) <= 1e-5
        levels, phi = square_chain(voxel_field(drr, velocity), lm.steps, DIMS)
        assert torch.equal(lm._exp[1], phi) and all(torch.equal(a, b) for a, b in zip(lm._exp[0], levels))


def test_refusals_raise_before_any_launch():
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=13))
    V = _field()
    target = torch.zeros(2, 1, 40, 40, device=DEV)
    siddon = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40)).to(DEV)
    torch.cuda.synchronize()
    with pytest.raises(TypeError, match="global NCC only"):
        DiffeomorphicLevenbergMarquardt(drr, rot, xyz, V.clone(), target, loss=NormalizedCrossCorrelation2d(patch_size=5), **KW)
    for kw in (dict(patch_size=10), dict(p_subsample=0.3)):
        with pytest.raises(NotImplementedError, match="full detector only"):
            DiffeomorphicLevenbergMarquardt(_scene(**kw)[1], rot, xyz, V.clone(), target, **KW)
    with pytest.raises(NotImplementedError, match="Trilinear renderer"):
        DiffeomorphicLevenbergMarquardt(siddon, rot, xyz, V.clone(), target, **KW)
    for bad in (0, 17, 2.5, True):
        with pytest.raises(ValueError, match="steps must be"):
            DiffeomorphicLevenbergMarquardt(drr, rot, xyz, V.clone(), target, steps=bad, **KW)
    for bad in (V.double(), V[0], torch.zeros(2, 6, 6, 6, device=DEV)):
        with pytest.raises(ValueError, match="velocity must be"):
            DiffeomorphicLevenbergMarquardt(drr, rot, xyz, bad, target, **KW)
    with pytest.raises(ValueError, match="displacement lattice"):   # per-pose velocities must match the poses
        DiffeomorphicLevenbergMarquardt(drr, rot, xyz, torch.zeros(3, 3, 6, 6, 6, device=DEV), target, **KW)
    with pytest.raises(_lib.B200DRRError, match="no CPU"):
        DiffeomorphicLevenbergMarquardt(drr, rot, xyz, V.cpu(), target, **KW)
    with pytest.raises(ValueError, match="tangent must be"):
        exp_velocity_jvp(drr, V, V.double())
    with pytest.raises(ValueError, match="steps must be"):
        exp_velocity_jvp(drr, V, V, steps=0)
    torch.cuda.synchronize()


def test_registration_meets_the_adam_bounds():
    """test_gpu_svf.test_diffeomorphic_registration_lowers_ncc_and_stays_invertible's scene (128^3 phantom, four views at 96^2, an
    8^3 velocity from zero towards a target rendered from a smooth 6 mm field, smoothness 1e-3, n_points = 250): the velocity LM
    must meet that test's bounds, mean 1 - NCC lowered 2x and det grad phi > 0 at every interior node, within 20 steps."""
    import deform_cases as dc

    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(96), renderer="trilinear").to(DEV)
    rot = torch.tensor([[0.0, 0.0, 0.0], [torch.pi / 2, 0.0, 0.0], [0.0, torch.pi / 2, 0.0], [torch.pi / 4, torch.pi / 4, 0.0]],
                       device=DEV)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(4, 3).contiguous()
    grid = (8, 8, 8)
    U_true = torch.as_tensor(dc.smooth_field(np.random.default_rng(21), 1, grid, 6.0)[0], device=DEV)
    kw = dict(n_points=250, **KW)
    with torch.no_grad():
        target = drr.render_deformed(rot, xyz, field=U_true, **kw)
    ncc = NormalizedCrossCorrelation2d()
    lin = drr._affine_inverse.reshape(4, 4)[:3, :3].double()

    def measure(V):
        with torch.no_grad():
            u = exp_velocity(drr, V)
            loss = float((1 - ncc(drr.render_deformed(rot, xyz, field=u, **kw), target)).mean())
            det = so.jacobian_det(torch.einsum("ij,jxyz->xyzi", lin, u.double())[None].cpu(), (n, n, n))
        return loss, float(det.min())

    V = torch.zeros_like(U_true)
    lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, V, target, steps=10, smoothness=1e-3, cg_iters=10, **kw)
    loss0 = measure(V)[0]
    reached, hist = None, []
    for k in range(1, 21):
        lm.step()
        hist.append(measure(V))
        if reached is None and loss0 / hist[-1][0] >= 2.0 and hist[-1][1] > 0:
            reached = k
    print(f"diffeomorphic LM: mean 1 - NCC {loss0:.3e}; per step (1 - NCC, min det) "
          f"{[(f'{a:.3e}', f'{b:.3f}') for a, b in hist]}; bounds met at step {reached}")
    assert reached is not None, (loss0, hist)
    assert all(d > 0 for _, d in hist[reached - 1:]), hist
