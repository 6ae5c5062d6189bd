"""The training step through the brick kernel's sensitivities mode (csrc/siddon_brick.cu, SENS; b200drr_siddon_fwd_sens_grid
variant 42, and variant 0 / b200drr_siddon_fwd_sens_pose where siddon_sens_brick_route sends them): the image and the per-ray
sensitivities against the fp64 oracle, against the slab-major kernel (variant 41) on the same inputs and against the pose-in
entry point, and the module's training step routed to it."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import relerr
from gpu_common import DEV

pytestmark = pytest.mark.gpu

BRICK, SLAB = 42, 41


def _p(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from diffdrr_b200 import _lib as L
    return L, L.load()


def _rays(vol_np, H, B, seed=0, cubic=True):
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import convert
    if cubic:
        subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
        subj.volume.affine = synthetic.make_affine(vol_np.shape[0])
    else:
        subj = synthetic.make_subject(vol_np)
    drr = DRR(subj, **synthetic.detector_kwargs(H)).to(DEV)
    rot, xyz = synthetic.make_poses(max(B, 2), seed=seed)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot[:B].to(DEV), xyz[:B].to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
        src = drr.affine_inverse(src).reshape(B, 3).contiguous()
        tgt = drr.affine_inverse(tgt).contiguous()
    return src, tgt, raylen


def _sens(variant, vol, src, tgt, raylen, H, W):
    L, lib = _lib()
    B = tgt.shape[0]
    out = torch.full((B, H * W), float("nan"), device=DEV)
    sens = torch.full((B, H * W, 8), float("nan"), device=DEV)
    L.check(lib.b200drr_siddon_fwd_sens_grid(_p(vol), *vol.shape, _p(src), _p(tgt), _p(raylen), _p(out), _p(sens), B, H, W, 0.5,
                                             1e-8, variant, _stream()), "fwd_sens_grid")
    return out, sens


def _grads(sens, gout):
    L, lib = _lib()
    B, N = gout.shape
    g_src, g_tgt, g_len = torch.empty(B, 3, device=DEV), torch.empty(B, N, 3, device=DEV), torch.empty(B, N, device=DEV)
    L.check(lib.b200drr_siddon_bwd_sens(_p(sens), _p(gout), _p(g_src), _p(g_tgt), _p(g_len), B, N, 0, _stream()), "bwd_sens")
    return g_src, g_tgt, g_len


def _same_as_slab(vol, src, tgt, raylen, H, W):
    """Brick and slab-major kernels on the same inputs: image to 5e-5, every sensitivity component to 1e-4 of its maximum."""
    out_b, sens_b = _sens(BRICK, vol, src, tgt, raylen, H, W)
    out_s, sens_s = _sens(SLAB, vol, src, tgt, raylen, H, W)
    assert torch.isfinite(out_b).all() and torch.isfinite(sens_b).all()
    assert relerr(out_b.cpu().numpy(), out_s.cpu().numpy()) < 5e-5
    sb, ss = sens_b.cpu().numpy(), sens_s.cpu().numpy()
    for k in range(7):
        assert relerr(sb[..., k], ss[..., k]) < 1e-4, k
    assert not sb[..., 7].any()
    return out_b, sens_b


@pytest.mark.parametrize("B", [2, 16])
def test_brick_sensitivities_equal_the_slab_kernel(B):
    from diffdrr_b200 import synthetic
    D, H = 512, 256
    vol_np = synthetic.make_volume(D, "smooth", seed=0)
    src, tgt, raylen = _rays(vol_np, H, B)
    _same_as_slab(torch.as_tensor(vol_np).to(DEV), src, tgt, raylen, H, H)


def test_brick_sensitivities_vs_oracle_16_poses():
    """The bench's shape (512^3 -> 256^2, 16 poses), smooth volume (SURVEY 8c: on noise the reference's own fp32 end-point
    gradients are 1e-2 off), against the fp64 closed form; variant 0 routes to the same kernel at this batch."""
    from diffdrr_b200 import synthetic
    from oracle import oracle
    D, H, B = 512, 256, 16
    N = H * H
    vol_np = synthetic.make_volume(D, "smooth", seed=0)
    vol = torch.as_tensor(vol_np).to(DEV)
    src, tgt, raylen = _rays(vol_np, H, B)
    gout = torch.rand(B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    npy = [x.cpu().numpy() for x in (src, tgt, raylen, gout)]
    ref = oracle.siddon_bwd(vol_np, *npy, dtype=np.float64, want_vol=False)
    ref_img = oracle.siddon_fwd(vol_np, *npy[:3], dtype=np.float64).reshape(B, N)
    for variant in (BRICK, 0):
        out, sens = _sens(variant, vol, src, tgt, raylen, H, H)
        g_src, g_tgt, g_len = _grads(sens, gout)
        assert relerr(out.cpu().numpy(), ref_img) < 1e-4, variant
        assert relerr(g_tgt.cpu().numpy(), ref["g_target"]) < 2e-3, variant
        assert relerr(g_src.cpu().numpy(), ref["g_source"].reshape(B, 3)) < 2e-3, variant
        assert relerr(g_len.cpu().numpy(), ref["g_raylen"].reshape(B, N)) < 1e-4, variant


def test_brick_sensitivities_partial_bricks_on_every_axis():
    """250 x 270 x 196 voxels: the last brick of every axis is partial (24 x 32 x 32 bricks; the TMA copy zero-fills the rest)."""
    from diffdrr_b200 import synthetic
    from oracle import oracle
    H, B = 128, 3
    vol_np = synthetic.make_volume((250, 270, 196), "smooth", seed=1)
    src, tgt, raylen = _rays(vol_np, H, B, seed=2, cubic=False)
    out, _ = _same_as_slab(torch.as_tensor(vol_np).to(DEV), src, tgt, raylen, H, H)
    ref = oracle.siddon_fwd(vol_np, *[x.cpu().numpy() for x in (src, tgt, raylen)], dtype=np.float64).reshape(B, -1)
    assert relerr(out.cpu().numpy(), ref) < 1e-4


def test_brick_sensitivities_source_inside_the_volume():
    """Every ray starts inside the volume (alpha of the entry face < 0, quirk Q1: the whole line is integrated)."""
    from diffdrr_b200 import synthetic
    from oracle import oracle
    D, H, B = 256, 128, 3
    vol_np = synthetic.make_volume(D, "smooth", seed=3)
    src, tgt, raylen = _rays(vol_np, H, B, seed=3)
    src = (torch.tensor([[128.3, 101.7, 140.2], [60.1, 200.6, 90.4], [128.0, 128.0, 128.0]], device=DEV)).contiguous()
    raylen = (tgt - src[:, None, :]).norm(dim=-1).contiguous()
    out, sens = _same_as_slab(torch.as_tensor(vol_np).to(DEV), src, tgt, raylen, H, H)
    gout = torch.rand(B, H * H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    npy = [x.cpu().numpy() for x in (src, tgt, raylen, gout)]
    ref = oracle.siddon_bwd(vol_np, *npy, dtype=np.float64, want_vol=False)
    ref_img = oracle.siddon_fwd(vol_np, *npy[:3], dtype=np.float64).reshape(B, -1)
    g_src, g_tgt, _ = _grads(sens, gout)
    assert relerr(out.cpu().numpy(), ref_img) < 1e-4
    assert relerr(g_tgt.cpu().numpy(), ref["g_target"]) < 2e-3
    assert relerr(g_src.cpu().numpy(), ref["g_source"].reshape(B, 3)) < 2e-3


def _module(D=512, H=256):
    from diffdrr_b200 import DRR, synthetic
    vol_np = synthetic.make_volume(D, "smooth", seed=0)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H), renderer="siddon").to(DEV)
    drr.density = torch.as_tensor(vol_np).to(DEV)
    return drr


def test_brick_sensitivities_pose_in_against_ray_tensor_inputs():
    """b200drr_siddon_fwd_sens_pose (rays made in-kernel from the pose matrices: the module's training step; routed to the brick
    kernel at 16 poses) against variant 42 on the ray tensors of the same poses.  The two ray constructions differ by ~1e-4 voxel, which moves the line
    integral (and its end-point derivative) of the few rays that run almost inside a voxel-boundary plane."""
    from diffdrr_b200 import geometry, synthetic
    from diffdrr_b200.pose import convert
    L, lib = _lib()
    D, H, B = 512, 256, 16
    N = H * H
    drr = _module(D, H)
    vol = drr.density
    rot, xyz = synthetic.make_poses(B, seed=0)
    with torch.no_grad():
        pose = convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
        Q, r, Ainv = drr._pose_constants()
        src_p, G, Wd = geometry.pose_rays(pose.matrix, Q, r, Ainv)
        rows, cols = drr._grid_axes(None)
        s, t = drr.detector(pose, None)
        raylen = (t - s).norm(dim=-1).reshape(B, -1).contiguous()
        src = drr.affine_inverse(s).reshape(B, 3).contiguous()
        tgt = drr.affine_inverse(t).contiguous()
    src_p, G, Wd = src_p.contiguous(), G.contiguous(), Wd.contiguous()
    out_p = torch.full((B, N), float("nan"), device=DEV)
    sens_p = torch.full((B, N, 8), float("nan"), device=DEV)
    L.check(lib.b200drr_siddon_fwd_sens_pose(_p(vol), D, D, D, _p(src_p), _p(G), _p(Wd), _p(rows), _p(cols), _p(out_p), _p(sens_p),
                                             B, H, H, 0.5, 1e-8, _stream()), "fwd_sens_pose")
    out_t, sens_t = _sens(BRICK, vol, src, tgt, raylen, H, H)
    assert torch.isfinite(out_p).all() and torch.isfinite(sens_p).all()
    a, b = out_p.cpu().numpy(), out_t.cpu().numpy()
    err = np.abs(a - b) / np.abs(b).max()
    assert (err > 1e-4).mean() < 1e-3 and float(np.sqrt((err ** 2).mean())) < 1e-5
    sp, st = sens_p.cpu().numpy(), sens_t.cpu().numpy()
    for k in range(7):
        e = np.abs(sp[..., k] - st[..., k]) / np.abs(st[..., k]).max()
        assert (e > 1e-3).mean() < 5e-3 and float(np.median(e)) < 1e-5, k


def test_module_training_step_routes_to_the_brick_kernel_eager_and_in_a_graph():
    """DRR(rot, xyz) + backward() at 16 poses (512^3 -> 256^2): the forward launches the brick kernel and not the slab-major
    sensitivities kernel, and one CUDA graph of the step, replayed, gives what the eager step gives."""
    from diffdrr_b200 import synthetic
    drr = _module()
    B = 16
    rot, xyz = synthetic.make_poses(B, seed=0)
    w = torch.rand(B, 1, 256, 256, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))

    def step(r, x):
        img = drr(r, x, parameterization="euler_angles", convention="ZXY")
        (img * w).sum().backward()
        return img.detach()

    r0, x0 = rot.to(DEV).requires_grad_(True), xyz.to(DEV).requires_grad_(True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        img_e = step(r0, x0)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("siddon_fwd_brick_kernel" in n for n in names), sorted(set(names))
    assert not any("siddon_sens_slab_kernel" in n for n in names)
    g_rot_e, g_xyz_e = r0.grad.clone(), x0.grad.clone()

    r_d = torch.zeros(B, 3, device=DEV, requires_grad=True)
    x_d = torch.zeros(B, 3, device=DEV, requires_grad=True)
    r_d.grad, x_d.grad = torch.zeros_like(r_d), torch.zeros_like(x_d)
    rot_dev, xyz_dev = rot.to(DEV), xyz.to(DEV)

    def body():
        with torch.no_grad():
            r_d.copy_(rot_dev)
            x_d.copy_(xyz_dev)
            r_d.grad.zero_()
            x_d.grad.zero_()
        return step(r_d, x_d)

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
    # red.global.add order differs between runs: equal up to fp32 summation order
    assert relerr(img_g.cpu().numpy(), img_e.cpu().numpy()) < 1e-6
    assert relerr(r_d.grad.cpu().numpy(), g_rot_e.cpu().numpy()) < 1e-4
    assert relerr(x_d.grad.cpu().numpy(), g_xyz_e.cpu().numpy()) < 1e-4
