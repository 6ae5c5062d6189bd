"""The blended-rigid render's per-pixel motion Jacobian and its Levenberg-Marquardt on the GPU (DRR.polyrigid_jacobian,
PolyrigidLevenbergMarquardt; DESIGN.md 6j): b200drr_polyrigid_jac on the seeded cases of polyrigid_cases.py against the per-ray fp64
reference of test_polyrigid_lm_cpu.py, plain / packed / 16-bit routes and reproducible bits, the module against render_polyrigid
(bit for bit), its backward (the adjoint identity) and an fp64 central difference, the block-sparse normal equations against a
dense statement, and the registration: monotone, free of host syncs, and its convergence on the two-structure scene."""
import math

import numpy as np
import pytest
import torch

import polyrigid_cases as pc
import trilinear_cases as tc
import polyrigid_oracle as po
from conftest import relerr
from diffdrr_b200 import DRR, PolyrigidLevenbergMarquardt, Trilinear, polyrigid_weights, synthetic
from diffdrr_b200 import polyrigid as pr
from diffdrr_b200.pose import convert
from diffdrr_b200.registration import ncc_normal_structures_equations
from diffdrr_b200.structures import apply_increments, se3_exp
from test_gpu_structures_lm import _about, _dense, _moved, registration_errors
from test_polyrigid_lm_cpu import case_tangents, grid_of, jac_reference, smooth_rays

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
FLOOR = 1e-4
DIMS = (48, 56, 40)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _kernel(c, packed=False, dtype=torch.float32, vol=None):
    """The case through b200drr_polyrigid_jac(_v16) -> numpy dict(img (B, N), J (B, K, N, 6), rects (B, K, 4))."""
    vol = _t(c["vol"] if vol is None else vol).to(dtype)
    pk = Trilinear()._packed_volume(vol) if packed else None
    assert (pk is not None) == packed
    src, tgt, raylen, M, T, w = (_t(a) for a in (c["src"], c["tgt"], c["raylen"], c["M"], c["T"], c["weights"]))
    K, g0, g1, g2 = w.shape
    B, N = tgt.shape[:2]
    H, W = grid_of(c)
    lib = pr._lib.load()
    wp = torch.empty(int(lib.b200drr_polyrigid_weight_floats(K, g0, g1, g2)), device=DEV)
    pr._lib.check(lib.b200drr_polyrigid_pack_weights(pr._ptr(w), K, g0, g1, g2, pr._ptr(wp), pr._stream()), "pack_weights")
    arange = torch.tensor([c["amin"], c["amax"]], device=DEV)
    img = torch.empty(B, N, device=DEV)
    J = torch.full((B, K, N, 6), float("nan"), device=DEV)
    rects = torch.empty(B, K, 4, dtype=torch.int32, device=DEV)
    fn, head, name = pr._vol_entry(lib, "b200drr_polyrigid_jac", vol)
    head = (pr._ptr(vol) if pk is None else None, pr._ptr(pk), *head[1:])
    pr._lib.check(fn(*head, *vol.shape, pr._ptr(src), pr._ptr(tgt), pr._ptr(raylen), pr._ptr(M), M.shape[0], K, pr._ptr(wp), g0, g1, g2,
                     pr._ptr(T), pr._ptr(img), pr._ptr(J), pr._ptr(rects), B, H, W, 0.5, 1e-8, c["n_points"], pr._ptr(arange),
                     pr._stream()), name)
    return dict(img=img.cpu().numpy(), J=J.cpu().numpy(), rects=rects.cpu().numpy())


@pytest.fixture(scope="module", params=sorted(pc.CASES))
def case(request):
    c = pc.CASES[request.param]()
    c["T"] = case_tangents(c)
    a = pc.args(c)
    c["jref"] = jac_reference(*a[:6], c["T"], *a[6:])
    c["j32"] = jac_reference(*a[:6], c["T"], *a[6:], dtype=np.float32)
    return c


@pytest.mark.parametrize("packed", [False, True])
def test_kernel_matches_fp64_reference(case, packed):
    c = case
    got = _kernel(c, packed)
    sm = smooth_rays(c)
    ref, r32 = c["jref"][:, :, sm], c["j32"][:, :, sm]
    assert np.isfinite(got["J"]).all()                        # every entry written
    assert relerr(got["J"][:, :, sm], ref) <= tc.tol(r32, ref, FLOOR)
    assert relerr(got["img"], po.fwd(*pc.args(c))) <= 1e-4
    H, W = grid_of(c)
    J = got["J"].reshape(*got["J"].shape[:2], H, W, 6)
    for b in range(J.shape[0]):
        for k in range(J.shape[1]):
            w0, w1, h0, h1 = got["rects"][b, k]
            outside = np.ones((H, W), bool)
            outside[max(h0, 0):h1 + 1, max(w0, 0):w1 + 1] = False
            assert not J[b, k][outside].any(), (b, k)


def test_image_is_the_forward_kernel_bitwise_and_repeats(case):
    c = case
    a, b = _kernel(c), _kernel(c)
    for key in a:
        assert np.array_equal(a[key], b[key]), key        # rects too: integer min / max do not depend on order
    fwd = pr._PolyrigidFunction.apply(_t(c["vol"]), None, _t(c["src"][:, None]), _t(c["tgt"]), _t(c["raylen"][:, None]), _t(c["M"]),
                                      torch.tensor([c["amin"], c["amax"]], device=DEV), *_packed(c), 0.5, 1e-8, c["n_points"],
                                      grid_of(c))
    assert np.array_equal(a["img"], fwd.cpu().numpy()[:, 0])
    p = _kernel(c, packed=True)
    for key in a:
        assert np.array_equal(a[key], p[key]), key


def _packed(c):
    w = _t(c["weights"])
    K, g0, g1, g2 = w.shape
    lib = pr._lib.load()
    wp = torch.empty(int(lib.b200drr_polyrigid_weight_floats(K, g0, g1, g2)), device=DEV)
    pr._lib.check(lib.b200drr_polyrigid_pack_weights(pr._ptr(w), K, g0, g1, g2, pr._ptr(wp), pr._stream()), "pack_weights")
    return wp, (g0, g1, g2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("packed", [False, True])
def test_16bit_density_equals_fp32_on_the_upcast_volume(dtype, packed):
    c = pc.CASES["k8_shared"]()
    c["T"] = case_tangents(c)
    up = _t(c["vol"]).to(dtype).float().cpu().numpy()
    a, b = _kernel(c, packed=packed, dtype=dtype), _kernel(c, vol=up)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


# ---- through DRR.polyrigid_jacobian -------------------------------------------------------------------------------------------
def _scene(H=40, **kw):
    vol = tc.volume(DIMS)
    lab = np.zeros(DIMS, np.float32)
    lab[8:20, 10:26, 6:18], lab[26:40, 30:48, 20:34], lab[10:22, 34:50, 22:36] = 3, 7, 12
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(H), renderer="trilinear",
              **kw).to(DEV)
    W = polyrigid_weights(drr.mask, (3, 7, 12), grid=(12, 14, 10), sigma=12.0, spacing=(4.0, 4.0, 4.0))
    return vol, drr, W


def _twists(K, B=None, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    shape = (K, 6) if B is None else (B, K, 6)
    xi = (torch.rand(*shape, generator=g) * 2 - 1) * torch.tensor([0.08, 0.08, 0.08, 10.0, 10.0, 10.0]) * scale
    return xi.to(DEV)


@pytest.mark.parametrize("per_pose", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_image_is_render_polyrigid_and_columns_are_its_backward(per_pose, dtype):
    """img equals render_polyrigid bit for bit; sum_n gout_n J[b, k, n] equals autograd's gradient of sum(gout * render_polyrigid)
    with respect to the increments xi at xi = 0, through apply_increments' map T(c) exp(xi^) T(-c) X with the exponential taken by
    torch.linalg.matrix_exp (se3_exp's closed form has no derivative at theta = 0: its norm is a square root)."""
    _, drr, W = _scene()
    if dtype != torch.float32:
        drr.density = drr.density.to(dtype)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=1))
    X = se3_exp(_twists(3, 2 if per_pose else None, seed=2)).float()
    img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=150, return_footprints=True, **KW)
    assert img.shape == (2, 1, 40, 40) and J.shape == (2, 3, 40, 40, 6) and rects.shape == (2, 3, 4)
    assert not img.requires_grad and not J.requires_grad
    with torch.no_grad():
        ref = drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=150, **KW)
    assert torch.equal(img, ref)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(3)).to(DEV)
    lhs = torch.einsum("bhw,bkhwi->bki", gout[:, 0].double(), J.double())
    if not per_pose:
        lhs = lhs.sum(0)
    xi = torch.zeros(*X.shape[:-2], 6, dtype=torch.float64, device=DEV, requires_grad=True)
    out = drr.render_polyrigid(rot, xyz, motions=_moved(X, xi, pr.polyrigid_pivots(drr, W)), weights=W, n_points=150, **KW)
    (gout * out).sum().backward()
    assert float(xi.grad.abs().max()) > 0
    assert relerr(lhs.cpu().numpy(), xi.grad.cpu().numpy()) <= 1e-5


def test_jacobian_column_matches_an_fp64_central_difference():
    """Independent of every fp32 kernel: polyrigid_oracle's fp64 forward on the module's rays, differenced along omega_y and v_z of
    structure 1 with the maps formed in float64."""
    vol, drr, W = _scene(H=24)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(1, seed=4))
    X = se3_exp(_twists(3, seed=5)).float()
    _, J = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=120, **KW)
    with torch.no_grad():
        source, target = drr.detector(convert(rot, xyz, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = drr.affine_inverse(source)[:, 0], drr.affine_inverse(target)
    src, tgt, raylen = (t.double().cpu().numpy() for t in (src, tgt, raylen))
    amin, amax = tc.range_of(DIMS, src.astype(np.float32), tgt.astype(np.float32))
    g = 1.0 + torch.rand(24, 24, generator=torch.Generator().manual_seed(6)).double()
    A = drr._affine.reshape(4, 4).double().cpu()
    pivots = pr.polyrigid_pivots(drr, W).cpu()
    Wn = W.cpu().numpy()
    h = 1e-6

    def f(k, col, s):
        xi = torch.zeros(3, 6, dtype=torch.float64)
        xi[k, col] = s
        Xk = apply_increments(X.cpu().double(), xi, pivots)
        M = (torch.linalg.inv(A) @ torch.linalg.inv(Xk) @ A)[None, :, :3, :].numpy()
        return float((g.numpy().reshape(1, -1) * po.fwd(vol, src, tgt, raylen, M, Wn, 120, float(amin), float(amax))).sum())

    for k, col in ((1, 1), (1, 5)):
        an = float((g.to(DEV) * J[0, k, ..., col].double()).sum())
        fd = (f(k, col, h) - f(k, col, -h)) / (2 * h)
        assert abs(fd) > 0 and abs(an - fd) < 1e-3 * abs(fd), (k, col, an, fd)


def test_normal_equations_on_the_jacobian_equal_the_dense_statement():
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=7))
    X = se3_exp(_twists(3, seed=8)).float()
    img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=150, return_footprints=True, **KW)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=se3_exp(_twists(3, seed=9, scale=0.5)).float(), weights=W, n_points=150, **KW)
    B, K = 2, 3
    x, t = img.reshape(B, 40, 40).contiguous(), target.reshape(B, 40, 40).contiguous()
    assert ((rects[..., 1] - rects[..., 0] + 1) * (rects[..., 3] - rects[..., 2] + 1) < 40 * 40).any()   # footprints do cull
    A = torch.zeros(B, 6 * K, 6 * K, dtype=torch.float64, device=DEV)
    g = torch.zeros(B, 6 * K, dtype=torch.float64, device=DEV)
    ncc_normal_structures_equations(x, t, J, rects, 1e-5, 1.0, A, g)
    Ar, gr = _dense(x, t, J.reshape(B, K, 40 * 40, 6), K)
    assert relerr(A.cpu().numpy(), Ar.cpu().numpy()) <= 1e-9 and relerr(g.cpu().numpy(), gr.cpu().numpy()) <= 1e-9


@pytest.mark.parametrize("per_pose", [False, True])
def test_lm_never_increases_the_loss_and_makes_no_host_sync(per_pose):
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(3, seed=10))
    X_true = se3_exp(_twists(3, 3 if per_pose else None, seed=11, scale=0.5)).float()
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=X_true, weights=W, n_points=150, **KW)
    X = torch.eye(4, device=DEV).expand(*X_true.shape).clone()
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=150, **KW)
    hist = [lm.step()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(5):
            hist.append(lm.step())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    h = torch.stack(hist).cpu()
    assert h.shape == ((6, 3) if per_pose else (6,))
    assert (h[1:] <= h[:-1]).all(), h
    assert (h[-1] < h[0]).all(), h


# ---- convergence on the two-structure scene -------------------------------------------------------------------------------------
def _two_structures():
    """The scene of test_gpu_polyrigid.test_registration_recovers_two_structures: 128^3, two blocks, three orthogonal views, 96^2,
    a 32^3 lattice, the target rendered blended with known motions -> (drr, rot, xyz, W, target, X_true, centroids)."""
    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    rng = np.random.default_rng(3)
    lab = np.zeros((n, n, n), np.float32)
    lab[30:58, 40:70, 36:60] = 1
    lab[70:100, 60:86, 66:96] = 2
    vol = (vol + (lab > 0) * (1.0 + 0.5 * rng.random((n, n, n)))).astype(np.float32)
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(96), renderer="trilinear").to(DEV)
    aff = torch.as_tensor(synthetic.make_affine(n), dtype=torch.float32)
    W = polyrigid_weights(drr.mask, (1, 2), grid=(32, 32, 32), sigma=6.0, spacing=tuple(float(aff[a, a]) for a in range(3)))
    centre = torch.stack([torch.as_tensor(np.argwhere(lab == k).mean(0), dtype=torch.float32) for k in (1, 2)])
    centre = (centre @ aff[:3, :3].T + aff[:3, 3]).to(DEV)
    rot = torch.tensor([[0.0, 0.0, 0.0], [math.pi / 2, 0.0, 0.0], [0.0, math.pi / 2, 0.0]], device=DEV)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(3, 3).contiguous()
    w_true = torch.tensor([[0.05, -0.03, 0.04], [-0.04, 0.05, 0.03]], device=DEV)
    t_true = torch.tensor([[8.0, -6.0, 5.0], [-7.0, 9.0, -4.0]], device=DEV)
    X_true = _about(w_true, t_true, centre)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=X_true, weights=W, n_points=250, **KW)
    return drr, rot, xyz, W, target, X_true, centre, w_true, t_true


def _run_lm(X, steps, rad, mm):
    drr, rot, xyz, W, target, X_true, centre, w_true, t_true = _two_structures()
    X = X(centre, w_true, t_true) if callable(X) else X
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=250, **KW)
    for k in range(1, steps + 1):
        loss = lm.step()
        err_r, err_t = registration_errors(X, X_true, centre)
        print(f"step {k}: rotation error {err_r:.3e} rad, centroid error {err_t:.3e} mm, loss {float(loss):.3e}")
        if err_r < rad and err_t < mm:
            return k, err_r, err_t, float(loss)
    raise AssertionError(f"after {steps} steps: rotation error {err_r:.4f} rad, centroid error {err_t:.3f} mm, loss {float(loss):.3g}")


def test_lm_recovers_two_structures():
    """The scene and start of test_gpu_polyrigid.test_registration_recovers_two_structures (three orthogonal views, shared motions,
    identity start; the Adam test there runs 500 steps): LM to 0.02 rad and 2 mm within 40 steps."""
    steps, err_r, err_t, loss = _run_lm(torch.eye(4, device=DEV).expand(2, 4, 4).clone(), 40, 0.02, 2.0)
    print(f"LM recovered both structures in {steps} steps: {err_r:.2e} rad, {err_t:.3f} mm, loss {loss:.3g}")


def test_lm_converges_quadratically_near_the_solution():
    """The same problem from 80 % of the way there (rotations at 0.8 x, translations at 0.98 x the truth): 1e-3 rad and 0.02 mm
    within 6 steps."""
    steps, err_r, err_t, loss = _run_lm(lambda c, w, t: _about(0.8 * w, 0.98 * t, c), 6, 1e-3, 0.02)
    print(f"LM from 80 % of the way: {steps} steps, {err_r:.2e} rad, {err_t:.3f} mm, loss {loss:.3g}")
    assert steps <= 6
