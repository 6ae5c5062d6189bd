"""GPU tests of the NCC normal equations (csrc/ncc_normal.cu) and of LevenbergMarquardt on the patch, multiscale and gradient NCC:
the kernels against the host emulation and the explicit fp64 reference, both J layouts, run-to-run identical bits and the
workspace bound, the default loss against the torch formula it replaced, g against autograd's pose gradient of the Gauss-Newton
objective, the LM invariants, and registration from the starts of the Adam tests."""
import numpy as np
import pytest
import torch

from gpu_common import DEV
from test_ncc_normal_cpu import CASES, _p, _windows, make_case, reference, relerr, sobel_strides

pytestmark = pytest.mark.gpu


def _kernel(x, t, J, strides, P, p, eps=1e-5, weight=1.0):
    from diffdrr_b200.registration import ncc_normal_equations
    B = x.shape[0]
    A = torch.zeros(B, P, P, dtype=torch.float64, device=DEV)
    g = torch.zeros(B, P, dtype=torch.float64, device=DEV)
    ncc_normal_equations(x.to(DEV).contiguous(), t.to(DEV).contiguous(), J.to(DEV).contiguous(), strides, p, eps, weight, A, g)
    return A.cpu().numpy(), g.cpu().numpy()


@pytest.mark.parametrize("shape,p,C,P", CASES)
def test_kernels_match_emulation_and_reference(shape, p, C, P):
    from hostemu import emu_ncc_normal
    H, W = shape
    p = _p(shape, p)
    B = 2
    x, t, J = make_case(B, C, H, W, P, offset=500.0 if P in (6, 16) else 0.0, constant=P != 1, seed=P + 7 * C)
    st = sobel_strides(B, C, H, W, P)
    A, g = _kernel(x, t, J, st, P, p)
    Ae, ge = emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), J.numpy(), st, P, 0 if p is None else p)
    if p == 1:
        assert not A.any() and not g.any()
        return
    Ar, gr = reference(x, t, J.permute(0, 2, 3, 4, 1), p)
    # the same math in another summation order, with fused multiply-adds on the device: 2.1e-11 at most on the H100
    assert relerr(A, Ae) < 1e-10 and relerr(g, ge) < 1e-10, (relerr(A, Ae), relerr(g, ge))
    assert relerr(A, Ar.numpy()) < 1e-9 and relerr(g, gr.numpy()) < 1e-9
    assert np.array_equal(A, A.transpose(0, 2, 1))


@pytest.mark.parametrize("P", [6, 7])
@pytest.mark.parametrize("p", [None, 13])
def test_256_both_layouts(P, p):
    """256^2, B = 4, C = 2: the Sobel-plane layout (B, P, 2, H, W) and DRR.jacobian's strided (B, H W, P) shared by both channels,
    against the explicit fp64 reference (one pose and channel at a time: 0.5 GB of Jz each at p = 13)."""
    B, C, H, W = 4, 2, 256, 256
    x, t, J = make_case(B, C, H, W, P, offset=40.0, seed=P)
    Jd = torch.randn(B, H * W, P, generator=torch.Generator().manual_seed(1))
    for Jin, strides, Jref in ((J, sobel_strides(B, C, H, W, P), J.permute(0, 2, 3, 4, 1)),
                               (Jd, (H * W * P, 0, 1, P), Jd.view(B, 1, H, W, P).expand(B, C, H, W, P))):
        A, g = _kernel(x, t, Jin, strides, P, p)
        Ar, gr = torch.zeros(B, P, P, dtype=torch.float64), torch.zeros(B, P, dtype=torch.float64)
        for b in range(B):
            for c in range(C):
                a_, g_ = reference(x[b:b + 1, c:c + 1].to(DEV), t[b:b + 1, c:c + 1].to(DEV), Jref[b:b + 1, c:c + 1].to(DEV), p)
                Ar[b] += a_[0].cpu()
                gr[b] += g_[0].cpu()
        assert relerr(A, Ar.numpy()) < 1e-9 and relerr(g, gr.numpy()) < 1e-9, (relerr(A, Ar.numpy()), relerr(g, gr.numpy()))


@pytest.mark.parametrize("p", [None, 13])
def test_repeated_runs_are_bitwise_identical_and_workspace_is_bounded(p):
    from diffdrr_b200 import _lib
    B, C, H, W, P = 16, 2, 256, 256, 6
    x, t, J = make_case(B, C, H, W, P, seed=3)
    st = sobel_strides(B, C, H, W, P)
    A0, g0 = _kernel(x, t, J, st, P, p)
    for _ in range(3):
        A, g = _kernel(x, t, J, st, P, p)
        assert np.array_equal(A, A0) and np.array_equal(g, g0)
    lib = _lib.load()
    for b in (1, 4, 16):
        for q in (6, 16):
            per_pose = lib.b200drr_ncc_normal_workspace_bytes(b, 2, 256, 256, 13 if p else 0, q) / b
            assert 0 < per_pose < 64 * 2**20, (b, q, per_pose)


def _problem():
    from test_gpu_registration import _problem as problem
    return problem()


def _torch_global_system(img, J, target, eps):
    """The float64 torch statement LevenbergMarquardt.step used before the kernel (global NCC, unweighted sums)."""
    B = img.shape[0]
    znorm = lambda v: (v - v.mean(1, keepdim=True)) / ((v - v.mean(1, keepdim=True)).square().mean(1, keepdim=True) + eps).sqrt()  # noqa: E731
    x = img.reshape(B, -1).double()
    Jx = J.reshape(B, x.shape[1], -1).double()
    xc = x - x.mean(dim=1, keepdim=True)
    s = (xc.square().mean(dim=1, keepdim=True) + eps).sqrt()
    z = xc / s
    Jz = (Jx - Jx.mean(dim=1, keepdim=True) - z.unsqueeze(-1) * (z.unsqueeze(-1) * Jx).mean(dim=1, keepdim=True)) / s.unsqueeze(-1)
    r = (z - znorm(target.reshape(target.shape[0], -1).double())).unsqueeze(-1)
    return Jz.mT @ Jz, (Jz.mT @ r).squeeze(-1)


def test_default_loss_reproduces_the_torch_formula():
    from diffdrr_b200 import LevenbergMarquardt, NormalizedCrossCorrelation2d
    from diffdrr_b200.jacobian import drr_jacobian
    drr, reg, _, target, _, _ = _problem()
    img, J = drr_jacobian(drr, reg.rotation.detach(), reg.translation.detach(), parameterization="euler_angles", convention="ZXY",
                          stop_grad=False)
    Ar, gr = _torch_global_system(img, J, target, 1e-5)
    N = img[0].numel()
    for lm in (LevenbergMarquardt(reg, target), LevenbergMarquardt(reg, target, loss=NormalizedCrossCorrelation2d())):
        A, g = lm.normal_equations(img, J)
        assert relerr((A * N).cpu().numpy(), Ar.cpu().numpy()) < 1e-12
        assert relerr((g * N).cpu().numpy(), gr.cpu().numpy()) < 1e-12


def _losses():
    from diffdrr_b200 import (GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d,
                              NormalizedCrossCorrelation2d)
    return {"global": lambda: NormalizedCrossCorrelation2d(),
            "patch13": lambda: NormalizedCrossCorrelation2d(patch_size=13),
            "multiscale": lambda: MultiscaleNormalizedCrossCorrelation2d([None, 13], [0.5, 0.5]),
            "gradient": lambda: GradientNormalizedCrossCorrelation2d(),
            "gradient_patch9": lambda: GradientNormalizedCrossCorrelation2d(patch_size=9, sigma=1.0)}


def _phi(loss, x, t):
    """Sum_s w_s / (2 N_s) sum_w |z(x_w) - z(t_w)|^2 per pose with the loss's torch formulas (fp64 in, fp64 out)."""
    from diffdrr_b200 import GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d
    if isinstance(loss, GradientNormalizedCrossCorrelation2d):
        x, t = loss.sobel(x), loss.sobel(t)
    scales = ([(n.patch_size, w, n.eps) for n, w in zip(loss.nccs, loss.patch_weights)]
              if isinstance(loss, MultiscaleNormalizedCrossCorrelation2d) else [(loss.patch_size, 1.0, loss.eps)])
    _, C, H, W = x.shape
    out = 0.0
    for p, w, eps in scales:
        N = C * H * W if p is None else C * (H - p + 1) * (W - p + 1) * p * p
        z = lambda a: (a - a.mean(-1, keepdim=True)) / (a.var(-1, keepdim=True, correction=0) + eps).sqrt()  # noqa: E731
        out = out + w / (2 * N) * ((z(_windows(x, p)) - z(_windows(t, p))) ** 2).sum(dim=(1, 2, 3))
    return out


@pytest.mark.parametrize("loss_name", list(_losses()))
def test_g_matches_autograd_pose_gradient(loss_name):
    """Adjoint identity: LM's g is autograd's pose gradient of the Gauss-Newton objective, chained through the render's pose
    backward (a DRR that keeps the ray-length term, as LM's J does)."""
    from diffdrr_b200 import DRR, LevenbergMarquardt, Registration, synthetic
    from diffdrr_b200.jacobian import drr_jacobian
    drr = DRR(synthetic.make_subject(synthetic.make_volume(128, "smooth", seed=1)), **synthetic.detector_kwargs(96),
              renderer="siddon").to(DEV)
    kw = dict(parameterization="euler_angles", convention="ZXY")
    true_rot, true_xyz = torch.tensor([[0.0, 0.0, 0.0]], device=DEV), torch.tensor([[0.0, 850.0, 0.0]], device=DEV)
    with torch.no_grad():
        target = drr(true_rot, true_xyz, **kw)
    rot = (true_rot + torch.tensor([[0.05, -0.04, 0.03]], device=DEV)).repeat(2, 1)
    xyz = (true_xyz + torch.tensor([[5.0, -10.0, 4.0]], device=DEV)).repeat(2, 1)
    rot[1] += 0.02
    reg = Registration(drr, rot.clone(), xyz.clone(), **kw)
    loss = _losses()[loss_name]()
    lm = LevenbergMarquardt(reg, target, loss=loss)
    img, J = drr_jacobian(drr, rot, xyz, stop_grad=False, **kw)
    _, g = lm.normal_equations(img, J)
    r, x = rot.clone().requires_grad_(True), xyz.clone().requires_grad_(True)
    phi = _phi(loss, drr(r, x, **kw).double(), target.double().expand(2, -1, -1, -1))
    gr, gx = torch.autograd.grad(phi.sum(), (r, x))
    ref = torch.cat([gr, gx], dim=1).double()
    err = relerr(g.cpu().numpy(), ref.cpu().numpy())
    print(f"{loss_name}: adjoint identity {err:.2e}")
    assert err < 1e-5, err


def _start(f):
    drr, _, _, target, true_rot, true_xyz = _problem()
    rot = true_rot + f * torch.tensor([[0.12, -0.08, 0.06]], device=DEV)
    xyz = true_xyz + f * torch.tensor([[10.0, -20.0, 8.0]], device=DEV)
    return drr, target, true_rot, true_xyz, rot, xyz


@pytest.mark.parametrize("loss_name", ["patch13", "multiscale", "gradient", "gradient_patch9"])
def test_lm_invariants(loss_name):
    """The per-pose loss never increases; no host synchronisation; each pose of a batch gets its single-pose system."""
    from diffdrr_b200 import LevenbergMarquardt, Registration
    drr, target, _, _, rot, xyz = _start(0.7)
    rot2, xyz2 = torch.cat([rot, rot * 0.5]), torch.cat([xyz, xyz + torch.tensor([[3.0, 2.0, -1.0]], device=DEV)])
    reg = Registration(drr, rot2.clone(), xyz2.clone(), "euler_angles", "ZXY")
    lm = LevenbergMarquardt(reg, target, loss=_losses()[loss_name]())
    hist = [lm.step()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(5):
            hist.append(lm.step())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    h = torch.stack(hist).cpu()
    assert (h[1:] <= h[:-1]).all(), h
    # the poses are independent: the batched system of each pose is its single-pose system (the render routes for one and two
    # poses differ by fp32 round-off); whole trajectories are not compared, a trial within round-off of the current loss may be
    # accepted in one run and rejected in the other
    from diffdrr_b200.jacobian import drr_jacobian
    kw = dict(parameterization="euler_angles", convention="ZXY")
    A2, g2 = lm.normal_equations(*drr_jacobian(drr, rot2, xyz2, stop_grad=False, **kw))
    for i in range(2):
        single = Registration(drr, rot2[i:i + 1].clone(), xyz2[i:i + 1].clone(), "euler_angles", "ZXY")
        lm1 = LevenbergMarquardt(single, target, loss=_losses()[loss_name]())
        A1, g1 = lm1.normal_equations(*drr_jacobian(drr, rot2[i:i + 1], xyz2[i:i + 1], stop_grad=False, **kw))
        assert relerr(A2[i:i + 1].cpu().numpy(), A1.cpu().numpy()) < 1e-4
        assert relerr(g2[i:i + 1].cpu().numpy(), g1.cpu().numpy()) < 1e-4


def _lm_registration(loss_name, f, steps=30):
    from diffdrr_b200 import LevenbergMarquardt, Registration
    drr, target, true_rot, true_xyz, rot, xyz = _start(f)
    reg = Registration(drr, rot.clone(), xyz.clone(), "euler_angles", "ZXY")
    loss = _losses()[loss_name]()
    lm = LevenbergMarquardt(reg, target, loss=loss)
    for it in range(steps):
        final = float(lm.step())
        rot_err = float((reg.rotation.detach() - true_rot).abs().max())
        xyz_err = float((reg.translation.detach() - true_xyz).abs().max())
        if final < 1e-3 and rot_err < 0.02 and xyz_err < 2.0:
            break
    with torch.no_grad():
        assert np.isclose(float(1.0 - loss(target, reg()).mean()), final, rtol=1e-3, atol=1e-6)
    print(f"LM {loss_name} from {f}x: {it + 1} steps, 1 - score {final:.2e}, rotation {rot_err:.2e} rad, translation "
          f"{xyz_err:.3f} mm")
    return final, rot_err, xyz_err, it + 1


@pytest.mark.xfail(strict=True, reason="on the H100, 30 LM steps end in the neighbouring optimum the Adam tests describe: gradient "
                                       "NCC from 0.7x reaches 1 - score 7.8e-5 and 0.17 mm but stops 0.028 rad off in rotation; "
                                       "multiscale NCC from 0.9x reaches 4.1e-4 but stops 0.057 rad and 18 mm off (README)")
@pytest.mark.parametrize("loss_name,f", [("gradient", 0.7), ("multiscale", 0.9)])
def test_lm_registration_reaches_the_bounds(loss_name, f):
    final, rot_err, xyz_err, steps = _lm_registration(loss_name, f)
    assert final < 1e-3 and rot_err < 0.02 and xyz_err < 2.0, \
        f"after {steps} LM steps: 1 - score {final:.2e}, rotation error {rot_err:.3e} rad, translation error {xyz_err:.2f} mm"
