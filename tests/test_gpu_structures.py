"""Piecewise-rigid renders on the GPU (DRR.render_structures; DESIGN.md 6f): every channel against the existing fused pose-in path
on density * (mask == label) with pose X^-1 P, gradients against autograd through that composition and an fp64 central
difference, 16-bit densities, culling, determinism, CUDA-graph capture, and a two-structure registration."""
import math

import numpy as np
import pytest
import torch

from conftest import relerr
from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, synthetic
from diffdrr_b200.pose import RigidTransform, convert
from diffdrr_b200.structures import _rigid_inverse

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
D = 64
BLOCKS = {3: (slice(8, 22), slice(20, 40), slice(10, 26)), 7: (slice(30, 50), slice(6, 20), slice(30, 50)),
          12: (slice(40, 60), slice(40, 58), slice(4, 18)), 9: (slice(2, 8), slice(50, 60), slice(50, 60))}


def _scene(kind="phantom"):
    vol = synthetic.make_volume(D, kind, seed=4)
    lab = np.zeros((D, D, D), np.float32)
    for label, sl in BLOCKS.items():
        lab[sl] = label
    return vol, lab


def _drr(vol, lab=None, H=48, **kw):
    mask = None if lab is None else torch.from_numpy(lab)
    return DRR(synthetic.make_subject(vol, mask=mask), **synthetic.detector_kwargs(H), **kw).to(DEV)


def _motion_params(K, B=None, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    shape = (K,) if B is None else (B, K)
    rot = (torch.rand(*shape, 3, generator=g) * 2 - 1) * 0.1 * scale
    xyz = (torch.rand(*shape, 3, generator=g) * 2 - 1) * 15.0 * scale
    return rot.to(DEV), xyz.to(DEV)


def _motions(rot, xyz):
    flat = convert(rot.reshape(-1, 3), xyz.reshape(-1, 3), parameterization="euler_angles", convention="XYZ").matrix
    return flat.reshape(*rot.shape[:-1], 4, 4)


def _reference(vol, lab, labels, rot, xyz, X, calibration=None, background=True, H=48, **kw):
    """Channel k by the existing fused path: DRR on density * (mask == labels[k]) with pose X_k^-1 P (background: every other
    voxel, pose P).  X^-1 is the rigid closed form render_structures composes, so the matrix gradients are comparable."""
    P = convert(rot, xyz, **KW).matrix
    B = P.shape[0]
    X = X.expand(B, *X.shape[-3:])
    chans = []
    for k, label in enumerate(labels):
        ref = _drr(vol * (lab == label), H=H, **kw)
        chans.append(ref(RigidTransform(_rigid_inverse(X[:, k]) @ P), calibration=calibration))
    if background:
        ref = _drr(vol * ~np.isin(lab, labels), H=H, **kw)
        chans.append(ref(RigidTransform(P), calibration=calibration))
    return torch.cat(chans, dim=1)


def _calibration(drr, on, B):
    """None, one calibration shared by the poses ("shared"), or a distinct one per pose ("per_pose")."""
    if not on:
        return None, None
    n = B if on == "per_pose" else 1
    C = drr.detector._calibration.reshape(1, 4, 4).repeat(n, 1, 1)
    C[:, 0, 0] *= 1.03 + 0.02 * torch.arange(n, device=C.device)
    C[:, 1, 3] += 2.0 - 1.5 * torch.arange(n, device=C.device)
    return C.requires_grad_(True), C.detach().clone().requires_grad_(True)


@pytest.mark.parametrize("B,K,calib,per_pose,stop_grad", [(1, 1, None, False, False), (4, 3, "shared", True, False),
                                                          (4, 3, None, False, True), (1, 3, "shared", True, True),
                                                          (4, 1, None, True, False), (4, 3, "per_pose", False, False)])
def test_channels_and_gradients_match_the_fused_path_composition(B, K, calib, per_pose, stop_grad):
    vol, lab = _scene()
    labels = (3, 7, 12)[:K]
    kw = dict(stop_gradients_through_grid_sample=stop_grad)
    drr = _drr(vol, lab, **kw)
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(max(B, 2), seed=B, rot_range=0.4, xyz_range=20.0))
    rot0, xyz0 = rot0[:B].contiguous(), xyz0[:B].contiguous()
    mrot, mxyz = _motion_params(K, B if per_pose else None, seed=K)
    mxyz[..., 0] += 40.0   # pushes part of a structure beyond the volume's original box
    X0 = _motions(mrot, mxyz)
    C, C_ref = _calibration(drr, calib, B)
    rot, xyz, X = (t.clone().requires_grad_(True) for t in (rot0, xyz0, X0))
    img = drr.render_structures(rot, xyz, motions=X, labels=labels, calibration=None if C is None else RigidTransform(C), **KW)
    rot_r, xyz_r, X_r = (t.clone().requires_grad_(True) for t in (rot0, xyz0, X0))
    ref = _reference(vol, lab, labels, rot_r, xyz_r, X_r, None if C_ref is None else RigidTransform(C_ref), **kw)
    assert img.shape == (B, K + 1, 48, 48) and ref.shape == img.shape
    for k in range(K + 1):
        assert relerr(img[:, k].detach().cpu().numpy(), ref[:, k].detach().cpu().numpy()) < 1e-4, k
    w = torch.rand(img.shape, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    (img * w).sum().backward()
    (ref * w).sum().backward()
    pairs = [(rot, rot_r), (xyz, xyz_r), (X, X_r)] + ([] if C is None else [(C, C_ref)])
    for a, b in pairs:
        assert relerr(a.grad.cpu().numpy(), b.grad.cpu().numpy()) < 1e-4


@pytest.mark.parametrize("B", [1, 3])
def test_matrix_and_rigidtransform_poses_match_the_euler_render(B):
    """The camera pose as a 'matrix' parameterization or a RigidTransform, and (B, K, 4, 4) motions wrapped in a RigidTransform,
    render what the Euler-angle parameters of the same poses render, with one image per pose."""
    vol, lab = _scene()
    drr = _drr(vol, lab)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(max(B, 2), seed=12))
    rot, xyz = rot[:B].contiguous(), xyz[:B].contiguous()
    labels = (3, 7, 12)
    for X in (_motions(*_motion_params(3, seed=9)), _motions(*_motion_params(3, B, seed=9))):
        ref = drr.render_structures(rot, xyz, motions=X, labels=labels, **KW)
        P = convert(rot, xyz, **KW).matrix
        for pose, kw in ((P, dict(parameterization="matrix")), (P[0] if B == 1 else P, dict(parameterization="matrix")),
                         (RigidTransform(P), {})):
            got = drr.render_structures(pose, motions=RigidTransform(X), labels=labels, **kw)
            assert got.shape == ref.shape == (B, 4, 48, 48)
            assert relerr(got.cpu().numpy(), ref.cpu().numpy()) < 1e-5


def test_identity_motions_sum_to_the_render_and_match_mask_channels():
    vol, lab = _scene()
    drr = _drr(vol, lab)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(4, seed=2))
    labels = (3, 7, 12)
    img = drr.render_structures(rot, xyz, motions=torch.eye(4, device=DEV).expand(3, 4, 4), labels=labels, **KW)
    whole = drr(rot, xyz, **KW)
    assert relerr(img.sum(1, keepdim=True).cpu().numpy(), whole.cpu().numpy()) < 1e-5
    chans = drr(rot, xyz, mask_to_channels=True, **KW)
    for k, label in enumerate(labels):
        assert relerr(img[:, k].cpu().numpy(), chans[:, label].cpu().numpy()) < 1e-5
    no_bg = drr.render_structures(rot, xyz, motions=torch.eye(4, device=DEV).expand(3, 4, 4), labels=labels, background=False,
                                  **KW)
    assert no_bg.shape == (4, 3, 48, 48) and torch.equal(no_bg, img[:, :3])


def test_motion_gradient_matches_an_fp64_central_difference():
    """Independent of every fp32 kernel: the fp64 reference-literal renderer on density * (mask == 7), differenced along the
    x translation of that structure's motion."""
    vol, lab = _scene("smooth")
    drr = _drr(vol, lab)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=6))
    mrot, mxyz = _motion_params(2, seed=3)
    X = _motions(mrot, mxyz).requires_grad_(True)
    img = drr.render_structures(rot, xyz, motions=X, labels=(3, 7), **KW)
    g = 1.0 + torch.rand(img[:, 1].shape, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    (g * img[:, 1]).sum().backward()
    an = float(X.grad[1, 0, 3])
    ref = _drr(vol * (lab == 7)).to(torch.float64)
    P = convert(rot.double(), xyz.double(), **KW).matrix
    h = 1e-6

    def f(t):
        Xt = X.detach().double()[1].clone()
        Xt[0, 3] += t
        with torch.no_grad():
            return (g.double() * ref(RigidTransform(torch.linalg.inv(Xt) @ P))[:, 0]).sum()

    fd = float((f(h) - f(-h)) / (2 * h))
    assert abs(an - fd) < 1e-3 * abs(fd), (an, fd)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_16bit_densities_equal_the_fp32_kernel_on_the_upcast_volume(dtype):
    vol, lab = _scene()
    drr16 = _drr(vol, lab)
    drr16.density = drr16.density.to(dtype)
    drr32 = _drr(drr16.density.float().cpu().numpy(), lab)
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=7))
    X0 = _motions(*_motion_params(3, seed=8))
    out = []
    for drr in (drr16, drr32):
        rot, X = rot0.clone().requires_grad_(True), X0.clone().requires_grad_(True)
        img = drr.render_structures(rot, xyz0, motions=X, labels=(3, 7, 12), **KW)
        img.square().sum().backward()
        out.append((img.detach(), rot.grad, X.grad))
    # the walk reads the same widened voxels: equal images; the gradients go through the pose reduction (summation order)
    assert torch.equal(out[0][0], out[1][0])
    for a, b in zip(out[0][1:], out[1][1:]):
        assert relerr(a.cpu().numpy(), b.cpu().numpy()) < 1e-5


def _footprint_rects(drr, rot, xyz, X, labels):
    """(B, K, 4) pixel rectangles {w0, w1, h0, h1} covering the projection of each structure's label box (planes at lo - 1/2,
    hi - 1/2) widened by one pixel, restated in float64 torch from the pose-in inputs: the footprint structures.cu culls to."""
    from diffdrr_b200.structures import _mask_state
    P = convert(rot, xyz, **KW).matrix
    B, K = P.shape[0], len(labels)
    src, G, _, rows, cols = drr._pose_in_inputs(RigidTransform((_rigid_inverse(X) @ P[:, None]).reshape(B * K, 4, 4)), None)
    src, G, rows, cols = src.double(), G.double(), rows.double(), cols.double()
    boxes = _mask_state(drr)["boxes"][list(labels)].double().repeat(B, 1)                      # (B*K, 6)
    bits = torch.tensor([[(c >> i) & 1 for i in range(3)] for c in range(8)], device=DEV, dtype=torch.float64)
    corners = boxes[:, None, :3] - 0.5 + bits * (boxes[:, None, 3:] - boxes[:, None, :3])      # (B*K, 8, 3)
    M = torch.stack([G[:, :, 0], G[:, :, 1], G[:, :, 2] + G[:, :, 3] - src], dim=-1)
    y = torch.linalg.solve(M[:, None].expand(-1, 8, -1, -1), (corners - src[:, None])[..., None])[..., 0]
    assert (y[..., 2] > 0).all()   # every box in front of the source: no whole-detector fallback in this scene
    pw = (y[..., 0] / y[..., 2] - cols[0]) / (cols[-1] - cols[0]) * (cols.numel() - 1)
    ph = (y[..., 1] / y[..., 2] - rows[0]) / (rows[-1] - rows[0]) * (rows.numel() - 1)
    r = torch.stack([pw.amin(1).floor() - 1, pw.amax(1).ceil() + 1, ph.amin(1).floor() - 1, ph.amax(1).ceil() + 1], dim=-1)
    return r.long().view(B, K, 4)


def test_outside_the_footprint_is_zero_and_calls_are_deterministic():
    vol, lab = _scene()
    drr = _drr(vol, lab, H=64)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=9))
    X = _motions(*_motion_params(3, seed=4)).requires_grad_(True)
    a = drr.render_structures(rot, xyz, motions=X, labels=(3, 7, 12), **KW)
    b = drr.render_structures(rot, xyz, motions=X, labels=(3, 7, 12), **KW)
    assert torch.equal(a, b)
    # the sensitivities the backward reduces are bitwise repeatable too (the reduction itself sums in any order)
    a.sum().backward()
    g1 = X.grad.clone()
    X.grad = None
    b.sum().backward()
    assert relerr(g1.cpu().numpy(), X.grad.cpu().numpy()) < 1e-5
    # every pixel outside each (pose, structure) footprint rectangle is exactly 0, not merely small; the rectangles cull
    rect = _footprint_rects(drr, rot, xyz, X.detach(), (3, 7, 12))
    H = W = 64
    hh, ww = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
    img = a.detach()
    culled = 0
    for b in range(2):
        for k in range(3):
            w0, w1, h0, h1 = rect[b, k].tolist()
            outside = (ww < w0) | (ww > w1) | (hh < h0) | (hh > h1)
            assert (img[b, k][outside] == 0).all(), (b, k)
            assert (img[b, k][~outside] != 0).any(), (b, k)
            culled += int(outside.sum())
    assert culled > 0.5 * 2 * 3 * H * W


def test_cuda_graph_replays_one_registration_step():
    vol, lab = _scene()
    drr = _drr(vol, lab)
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=10))
    X0 = _motions(*_motion_params(3, seed=5))
    w = torch.rand(2, 4, 48, 48, device=DEV)

    def step(r, x, X):
        img = drr.render_structures(r, x, motions=X, labels=(3, 7, 12), **KW)
        (img * w).sum().backward()
        return img.detach()

    r_e, x_e, X_e = (t.clone().requires_grad_(True) for t in (rot0, xyz0, X0))
    img_e = step(r_e, x_e, X_e)
    r_d, x_d, X_d = (t.clone().requires_grad_(True) for t in (rot0, xyz0, X0))
    step(r_d, x_d, X_d)   # creates the .grad tensors and the cached label tables outside the capture

    def body():
        for t in (r_d, x_d, X_d):
            t.grad.zero_()
        return step(r_d, x_d, X_d)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        img_g = body()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(img_g, img_e)
    for a, b in ((r_d, r_e), (x_d, x_e), (X_d, X_e)):
        assert relerr(a.grad.cpu().numpy(), b.grad.cpu().numpy()) < 1e-5


def _axis_angle(w):
    """(K, 3) rotation vectors -> (K, 3, 3), Rodrigues."""
    th = w.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    k = w / th
    Kx = torch.zeros(*w.shape[:-1], 3, 3, device=w.device, dtype=w.dtype)
    Kx[..., 0, 1], Kx[..., 0, 2], Kx[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    Kx = Kx - Kx.mT
    s, c = th.sin()[..., None], th.cos()[..., None]
    return torch.eye(3, device=w.device, dtype=w.dtype) + s * Kx + (1 - c) * (Kx @ Kx)


def _about(w, t, centre):
    """Rigid motion rotating by w about `centre` (K, 3), then translating by t: x -> R (x - c) + c + t."""
    R = _axis_angle(w)
    top = torch.cat([R, (centre + t - (R @ centre[..., None])[..., 0])[..., None]], dim=-1)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], device=w.device).expand(*w.shape[:-1], 1, 4)
    return torch.cat([top, bottom], dim=-2)


def test_registration_recovers_two_structures():
    """128^3, two labelled blocks and a background, three orthogonal views (every rotation axis is in-plane in one of them); the
    target is rendered with known motions of a few degrees and ~10 mm, then Adam on each block's rotation (about its own centroid)
    and translation, on the composite's NCC."""
    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    rng = np.random.default_rng(3)
    lab = np.zeros((n, n, n), np.float32)
    lab[30:58, 40:70, 36:60] = 1
    lab[70:100, 60:86, 66:96] = 2
    vol = vol + (lab > 0) * (1.0 + 0.5 * rng.random((n, n, n))).astype(np.float32)
    drr = _drr(vol.astype(np.float32), lab, H=96)
    aff = torch.as_tensor(synthetic.make_affine(n), dtype=torch.float32)
    centre = torch.stack([torch.as_tensor(np.argwhere(lab == k).mean(0), dtype=torch.float32) for k in (1, 2)])
    centre = (centre @ aff[:3, :3].T + aff[:3, 3]).to(DEV)
    rot = torch.tensor([[0.0, 0.0, 0.0], [math.pi / 2, 0.0, 0.0], [0.0, math.pi / 2, 0.0]], device=DEV)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(3, 3).contiguous()
    w_true = torch.tensor([[0.05, -0.03, 0.04], [-0.04, 0.05, 0.03]], device=DEV)
    t_true = torch.tensor([[8.0, -6.0, 5.0], [-7.0, 9.0, -4.0]], device=DEV)
    with torch.no_grad():
        target = drr.render_structures(rot, xyz, motions=_about(w_true, t_true, centre), labels=(1, 2), **KW).sum(1, keepdim=True)
    w = torch.full((2, 3), 1e-4, device=DEV, requires_grad=True)
    t = torch.zeros(2, 3, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[w], lr=5e-3), dict(params=[t], lr=0.5)])
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.996)
    ncc = NormalizedCrossCorrelation2d()
    steps = 800
    for _ in range(steps):
        opt.zero_grad()
        img = drr.render_structures(rot, xyz, motions=_about(w, t, centre), labels=(1, 2), **KW).sum(1, keepdim=True)
        loss = -ncc(img, target).mean()
        loss.backward()
        opt.step()
        sched.step()
    err_w = float((w.detach() - w_true).abs().max())
    err_t = float((t.detach() - t_true).abs().max())
    assert err_w < 0.02 and err_t < 2.0, (f"after {steps} steps: rotation error {err_w:.4f} rad, translation error {err_t:.3f} mm, "
                                          f"loss {float(loss):.5f}")
