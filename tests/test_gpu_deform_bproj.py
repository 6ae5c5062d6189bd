"""The deformable render's transpose in the density on the GPU (b200drr_deform_bproj; DESIGN.md 6l): the kernel on the seeded cases
of deform_cases.py against the fp64 backprojection of deform_bproj_oracle.py, adjointness with b200drr_deform_fwd, the zero-field
identity with the Trilinear renderer's volume gradient, repeatability, `render_deformed(..., density=)` with and without a gradient
(shared and per-pose fields; full, sub-sampled and patched detectors; joint density + field + pose), no host sync, CUDA-graph
capture, the refusals, and a motion-compensated reconstruction."""
import math

import numpy as np
import pytest
import torch

import deform_bproj_oracle as bo
import deform_cases as dc
import trilinear_cases as tc
from conftest import relerr
from diffdrr_b200 import DRR, Trilinear, _lib, synthetic
from diffdrr_b200 import deform as dm
from diffdrr_b200.pose import convert
from diffdrr_b200.renderers import _ptr, _stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
FLOOR = 1e-4
DIMS = (48, 56, 40)
REORDER = 1e-5   # the volume gradient is summed with atomics: results agree to fp32 reordering


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bproj(c, gout=None, U=None):
    """The case through b200drr_deform_bproj -> g_V (D0, D1, D2) numpy."""
    src, tgt, raylen = _t(c["src"]), _t(c["tgt"]), _t(c["raylen"])
    field = _t(dc.pack(c["U"] if U is None else U))
    gout = _t(c["gout"] if gout is None else gout)
    arange = torch.tensor([c["amin"], c["amax"]], device=DEV)
    B, N = c["tgt"].shape[:2]
    g_vol = torch.full(c["vol"].shape, float("nan"), device=DEV)   # the entry overwrites it
    lib = _lib.load()
    _lib.check(lib.b200drr_deform_bproj(*c["vol"].shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(field), field.shape[0],
                                        *field.shape[1:4], _ptr(gout), _ptr(g_vol), B, N, c["H"], c["W"], 0.5, 1e-8, c["n_points"],
                                        _ptr(arange), _stream()), "b200drr_deform_bproj")
    return g_vol.cpu().numpy()


def _fwd(c, vol):
    """b200drr_deform_fwd of the case's rays and field on the volume `vol` -> (B, N) numpy."""
    grid = (c["H"], c["W"]) if c["H"] else None
    out = dm._DeformFunction.apply(_t(vol), None, _t(c["src"][:, None]), _t(c["tgt"]), _t(c["raylen"][:, None]), _t(dc.pack(c["U"])),
                                   torch.tensor([c["amin"], c["amax"]], device=DEV), 0.5, 1e-8, c["n_points"], grid)
    return out.cpu().numpy()[:, 0]


@pytest.fixture(scope="module", params=sorted(dc.CASES))
def case(request):
    c = dc.CASES[request.param]()
    a = (c["vol"], c["src"], c["tgt"], c["raylen"], c["U"], c["gout"], c["n_points"], c["amin"], c["amax"])
    c["ref"] = bo.bproj(*a)
    c["r32"] = bo.bproj(*a, dtype=np.float32)
    return c


def test_kernel_matches_fp64_oracle(case):
    c = case
    got = _bproj(c)
    assert np.abs(c["ref"]).max() > 0
    assert relerr(got, c["ref"]) <= tc.tol(c["r32"], c["ref"], FLOOR)


def test_kernel_is_the_transpose_of_the_forward(case):
    """sum_n w_n fwd(dV)_n = <bproj(w), dV>, b200drr_deform_fwd against b200drr_deform_bproj on the same rays and field."""
    c = case
    dV = np.random.default_rng(3).normal(size=c["vol"].shape).astype(np.float32)
    lhs = float((c["gout"].astype(np.float64) * _fwd(c, dV)).sum())
    rhs = float((_bproj(c).astype(np.float64) * dV).sum())
    scale = float((np.abs(c["gout"]).astype(np.float64) * _fwd(c, np.abs(dV))).sum())
    assert lhs != 0 and abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


def test_zero_field_is_the_trilinear_volume_gradient(case):
    """u = 0: the samples, cells and weights are the Trilinear renderer's, so the two scatters differ only in the atomics' order."""
    c = case
    V = _t(c["vol"]).requires_grad_(True)
    out = Trilinear()(V, _t(c["src"][:, None]), _t(c["tgt"]), _t(c["raylen"][:, None]), n_points=c["n_points"], alphamin=c["amin"],
                      alphamax=c["amax"])
    out.backward(_t(c["gout"])[:, None])
    got = _bproj(c, U=np.zeros_like(c["U"]))
    assert np.abs(got).max() > 0 and relerr(got, V.grad.cpu().numpy()) <= REORDER


def test_two_calls_agree(case):
    a, b = _bproj(case), _bproj(case)
    assert relerr(b, a) <= REORDER


# ---- through DRR.render_deformed(..., density=) ---------------------------------------------------------------------------------
def _scene(H=40, **kw):
    vol = tc.volume(DIMS)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear", **kw).to(DEV)
    return vol, drr


def _field(B=None, grid=(10, 12, 9), seed=0, amp=10.0):
    U = dc.smooth_field(np.random.default_rng(seed), 1 if B is None else B, grid, amp)
    return _t(U[0] if B is None else U)


def _rays(drr, rot, xyz):
    with torch.no_grad():
        source, target = drr.detector(convert(rot, xyz, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = drr.affine_inverse(source), drr.affine_inverse(target)
    src, tgt, raylen = (t.cpu().numpy() for t in (src[:, 0], tgt, raylen))
    return src, tgt, raylen, tc.range_of(DIMS, src, tgt)


def _voxel_np(drr, U):
    lin = drr._affine_inverse.reshape(4, 4)[:3, :3].double().cpu().numpy()
    U = U.double().cpu().numpy()
    U = U if U.ndim == 5 else U[None]
    return np.einsum("ij,bjxyz->bixyz", lin, U)


def test_density_without_grad_is_the_default_call_bitwise():
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=1))
    U = _field(2, seed=2)
    want = drr.render_deformed(rot, xyz, field=U, n_points=150, **KW)
    V = _t(vol)   # another tensor with the same values
    assert torch.equal(drr.render_deformed(rot, xyz, field=U, n_points=150, density=V, **KW), want)
    assert torch.equal(drr.render_deformed(rot, xyz, field=U, n_points=150, density=drr.density, **KW), want)


@pytest.mark.parametrize("per_pose", [False, True])
def test_autograd_to_density_matches_fp64_oracle(per_pose):
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=3))
    U = _field(2 if per_pose else None, seed=4)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(5)).to(DEV)
    V = _t(vol).requires_grad_(True)
    img = drr.render_deformed(rot, xyz, field=U, n_points=150, density=V, **KW)
    (img * gout).sum().backward()
    src, tgt, raylen, (amin, amax) = _rays(drr, rot, xyz)
    a = (vol, src, tgt, raylen, _voxel_np(drr, U), gout.cpu().numpy().reshape(2, -1), 150, amin, amax)
    ref, r32 = bo.bproj(*a), bo.bproj(*a, dtype=np.float32)
    assert np.abs(ref).max() > 0
    assert relerr(V.grad.cpu().numpy(), ref) <= tc.tol(r32, ref, FLOOR)


def test_subsampled_and_patched_detectors_backproject_their_pixels():
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=6))
    amin, amax = _rays(drr, rot, xyz)[3]       # one explicit range: Trilinear's own is that of the rays in the call
    kw = dict(n_points=120, alphamin=amin, alphamax=amax, **KW)
    U = _field(2, seed=7)
    w = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(8)).to(DEV)

    def grad(d, weights):
        V = _t(vol).requires_grad_(True)
        (d.render_deformed(rot, xyz, field=U, density=V, **kw) * weights).sum().backward()
        return V.grad.cpu().numpy()

    full = grad(drr, w)
    _, patched = _scene(patch_size=10)
    assert relerr(grad(patched, w), full) <= REORDER
    _, sub = _scene(p_subsample=0.3)
    keep = torch.zeros(2, 40 * 40, device=DEV)
    keep[:, sub.detector.pick_tensor()] = 1.0
    masked = w * keep.view(2, 1, 40, 40)
    assert relerr(grad(sub, w), grad(drr, masked)) <= REORDER


def test_joint_density_field_and_pose_gradients():
    """The camera and field gradients do not change when the density also wants one: per-ray outputs bit for bit, the field's
    atomics to fp32 reordering; the density gradient is the density-only one."""
    vol, drr = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=9))
    U0 = _field(2, seed=10)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(11)).to(DEV)

    def run(with_density, with_motion=True):
        rot, xyz, U = (t.clone().requires_grad_(with_motion) for t in (rot0, xyz0, U0))
        V = _t(vol).requires_grad_(with_density)
        img = drr.render_deformed(rot, xyz, field=U, n_points=150, density=V, **KW)
        (img * gout).sum().backward()
        return img.detach(), rot.grad, xyz.grad, U.grad, V.grad

    joint, motion, dens = run(True), run(False), run(True, with_motion=False)
    assert torch.equal(joint[0], motion[0]) and torch.equal(joint[0], dens[0])
    assert torch.equal(joint[1], motion[1]) and torch.equal(joint[2], motion[2])
    assert relerr(joint[3].cpu().numpy(), motion[3].cpu().numpy()) <= REORDER
    assert motion[4] is None and dens[1] is None
    assert relerr(joint[4].cpu().numpy(), dens[4].cpu().numpy()) <= REORDER


def test_no_host_sync_and_cuda_graph_capture():
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=12))
    U = _field(2, seed=13)
    w = torch.rand(2, 1, 40, 40, device=DEV)
    V = _t(vol).requires_grad_(True)

    def step():
        img = drr.render_deformed(rot, xyz, field=U, n_points=100, density=V, **KW)
        (g,) = torch.autograd.grad(img, V, w)
        return img.detach(), g

    img_e, g_e = step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        img_g, g_g = step()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(img_g, img_e)
    assert relerr(g_g.cpu().numpy(), g_e.cpu().numpy()) <= REORDER


def test_density_refusals_raise_before_any_launch():
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=14))
    U = _field()
    call = lambda density, d=drr: d.render_deformed(rot, xyz, field=U, density=density, **KW)   # noqa: E731
    torch.cuda.synchronize()
    for bad in (_t(vol)[:-1], _t(vol)[None], torch.from_numpy(vol), vol):
        with pytest.raises(ValueError, match="drr.density's shape"):
            call(bad)
    for dtype in (torch.float16, torch.bfloat16):
        with pytest.raises(NotImplementedError, match="no volume gradient to a"):
            call(_t(vol).to(dtype).requires_grad_(True))
    with pytest.raises(NotImplementedError, match="fp32 / fp16 / bf16"):
        call(_t(vol).double())
    grad_vol = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(DEV)
    grad_vol.density.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="no volume gradient.*density="):
        grad_vol.render_deformed(rot, xyz, field=U, **KW)
    with pytest.raises(NotImplementedError, match="Trilinear renderer"):   # the other refusals still hold with a density
        call(_t(vol).requires_grad_(True), DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40)).to(DEV))
    with pytest.raises(ValueError, match="displacement lattice"):
        drr.render_deformed(rot, xyz, field=U.double(), density=_t(vol).requires_grad_(True), **KW)
    torch.cuda.synchronize()
    # a 16-bit density without a gradient is rendered, as drr.density would be
    V16 = _t(vol).to(torch.bfloat16)
    drr16 = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(DEV)
    drr16.density = V16
    assert torch.equal(call(V16), drr16.render_deformed(rot, xyz, field=U, **KW))


# ---- motion-compensated reconstruction ------------------------------------------------------------------------------------------
def test_motion_compensated_reconstruction_beats_the_static_one():
    """96^3 phantom, 32 views on a circle at 64^2, n_points = 200.  Each view sees the volume under its own respiratory phase:
    U_b = sin(2 pi phase_b) U_0, U_0 a smooth 8^3 world-mm field of about 5 mm.  Fifteen CGLS iterations from zero on the linear
    problem A V = y, with A^T from autograd through render_deformed(..., density=V): once through the known fields
    (motion-compensated) and once with field = 0 (the static Trilinear model).  One run on an NVIDIA H100 80GB HBM3 (700 W):
    relative projection residual 0.0035 compensated against 0.0178 static (5.1x), volume RMS error inside the body 0.0454 against
    0.0721 (1.59x); the bounds below keep a margin for the atomics' reordering."""
    n, B, H = 96, 32, 64
    vol = synthetic.make_volume(n, "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear").to(DEV)
    theta = torch.arange(B, device=DEV, dtype=torch.float32) * (2 * math.pi / B)
    rot = torch.stack([theta, torch.zeros_like(theta), torch.zeros_like(theta)], -1)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(B, 3).contiguous()
    U0 = _field(grid=(8, 8, 8), seed=21, amp=5.0)
    phase = torch.arange(B, device=DEV, dtype=torch.float32) * (3.3 / B)          # a little over three breaths over the scan
    U = torch.sin(2 * math.pi * phase)[:, None, None, None, None] * U0
    kw = dict(n_points=200, **KW)
    V_true = drr.density
    with torch.no_grad():
        y = drr.render_deformed(rot, xyz, field=U, **kw)
    body = V_true > 0.1 * V_true.max()

    def cgls(field, iters=15):
        A = lambda V: drr.render_deformed(rot, xyz, field=field, density=V, **kw)    # noqa: E731

        def AT(w):
            V = torch.zeros_like(V_true, requires_grad=True)
            return torch.autograd.grad(A(V), V, w)[0]

        x = torch.zeros_like(V_true)
        r = y.clone()
        s = AT(r)
        p, gamma = s.clone(), (s * s).sum()
        for _ in range(iters):
            with torch.no_grad():
                q = A(p)
            alpha = gamma / (q * q).sum()
            x, r = x + alpha * p, r - alpha * q
            s = AT(r)
            gamma, gamma_old = (s * s).sum(), gamma
            p = s + (gamma / gamma_old) * p
        return float(r.norm() / y.norm()), float(((x - V_true)[body] ** 2).mean().sqrt())

    res_c, rms_c = cgls(U)
    res_s, rms_s = cgls(torch.zeros_like(U))
    print(f"reconstruction: projection residual {res_c:.4f} compensated vs {res_s:.4f} static ({res_s / res_c:.2f}x); volume RMS "
          f"error inside the body {rms_c:.4f} vs {rms_s:.4f} ({rms_s / rms_c:.2f}x)")
    assert res_s / res_c >= 3.0 and rms_s / rms_c >= 1.3, (res_c, res_s, rms_c, rms_s)
