#!/usr/bin/env python
"""Small invocations of the round-2 kernels for compute-sanitizer (memcheck / racecheck / synccheck): brick-major TMA forward
(several bricks per CTA, partial bricks, two pose chunks), the locality-ordered slab kernels, the brick scatter (volume gradient),
the mask grid kernels, the un-reduced segment kernels, fp64, the trilinear pose-in step and the image losses (global and
patch-wise NCC, blur + Sobel, mutual information, on sizes that are not a multiple of the tiles); PeerGather is multi-GPU
only."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from diffdrr_b200 import (DRR, GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d,  # noqa: E402
                          MutualInformation, Siddon, _lib, renderers, synthetic)
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
for dims, H, B in (((50, 72, 64), 40, 3), ((30, 40, 36), 24, 35)):
    vol = torch.rand(*dims, device=dev)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(dims)
    drr = DRR(subj, **synthetic.detector_kwargs(H)).to(dev)
    rot, xyz = synthetic.make_poses(B, seed=1)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot.to(dev), xyz.to(dev), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
        src, tgt = drr.affine_inverse(src).reshape(B, 3).contiguous(), drr.affine_inverse(tgt).contiguous()
    N = H * H
    ref = torch.empty(B, N, device=dev)
    _lib.check(lib.b200drr_siddon_fwd(_ptr(vol), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(ref), B, N, 0.5, 1e-8, 0, 0, _stream()), "fwd")
    ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(B, H, H), dtype=torch.uint8, device=dev)
    for v in (0,):
        out = torch.zeros(B, N, device=dev)
        _lib.check(lib.b200drr_siddon_fwd_brick(_ptr(vol), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), None, None, None, None, _ptr(out),
                                                _ptr(ws), ws.numel(), B, H, H, 0.5, 1e-8, v, _stream()), "brick")
        torch.cuda.synchronize()
        print(dims, "brick variant", v, "maxdiff", float((out - ref).abs().max() / ref.abs().max()))
    renderers._SORT_MIN_RAYS = 1
    s3, t3, l3 = src.reshape(B, 1, 3).clone().requires_grad_(True), tgt.clone().requires_grad_(True), raylen.reshape(B, 1, N)
    o = Siddon()(vol, s3, t3, l3)
    o.sum().backward()
    torch.cuda.synchronize()
    print(dims, "sorted sens maxdiff", float((o.detach().reshape(B, N) - ref).abs().max() / ref.abs().max()))
    # volume gradient: the brick kernel as a scatter (swizzled accumulator brick, TMA store) vs the slab-major walk with atomics
    gout = torch.rand(B, N, device=dev)
    g_b, g_s = torch.full_like(vol, float("nan")), torch.zeros_like(vol)
    _lib.check(lib.b200drr_siddon_bwd_vol_brick(_ptr(gout), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), None, None, None, None, _ptr(g_b),
                                                _ptr(ws), ws.numel(), B, H, H, 0.5, 1e-8, _stream()), "bwd_vol_brick")
    _lib.check(lib.b200drr_siddon_bwd_grid(_ptr(vol), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), None, None, None, _ptr(g_s),
                                           B, H, H, 0.5, 1e-8, 0, 0, _stream()), "bwd_grid")
    torch.cuda.synchronize()
    print(dims, "brick scatter g_vol maxdiff", float((g_b - g_s).abs().max() / g_s.abs().max()))
    # mask_to_channels grid kernels (slab-major forward, tile-ordered backward), un-reduced segments + their backward, fp64
    lab = (torch.arange(dims[0], device=dev)[:, None, None] // 17 + 2 * (torch.arange(dims[2], device=dev)[None, None, :] // 20)).float()
    lab = lab.expand(*dims).contiguous()
    sid = Siddon()
    sid.detector_shape = (H, H)
    t4 = tgt.clone().requires_grad_(True)
    m = sid(vol, src.reshape(B, 1, 3), t4, l3, mask=lab)
    m.sum().backward()
    seg_mod = Siddon(reducefn=lambda x: x.square().sum(-1))
    t5 = tgt[:, :256].clone().requires_grad_(True)
    seg_mod(vol, src.reshape(B, 1, 3), t5, l3[:, :, :256].contiguous()).sum().backward()
    t6 = tgt[:, :256].double().clone().requires_grad_(True)
    Siddon()(vol.double(), src.reshape(B, 1, 3).double(), t6, l3[:, :, :256].double().contiguous()).sum().backward()
    torch.cuda.synchronize()
    print(dims, "mask / segments / fp64 ok", float(m.detach().sum()), float(t5.grad.abs().max()), float(t6.grad.abs().max()))
# trilinear pose-in training step (alpha-range reduction kernel, in-kernel rays, matrix gradients)
vol = synthetic.make_volume((40, 48, 56), "phantom", seed=5)
drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(24), renderer="trilinear").to(dev)
rot, xyz = synthetic.make_poses(3, seed=2)
rot, xyz = rot.to(dev).requires_grad_(True), xyz.to(dev).requires_grad_(True)
img = drr(rot, xyz, parameterization="euler_angles", convention="ZXY", n_points=64)
img.sum().backward()
torch.cuda.synchronize()
print("trilinear pose-in ok", float(img.sum()), float(rot.grad.abs().max()))
# per-pixel pose Jacobians (jacobian.cu): a ragged last pixel block, 6 and 13 pose parameters, both renderers
for renderer in ("siddon", "trilinear"):
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer=renderer).to(dev)
    for par in ("euler_angles", "quaternion_adjugate"):
        r, x = convert(rot.detach(), xyz.detach(), parameterization="euler_angles", convention="ZXY").convert(par, convention="ZXY")
        img, J = drr.jacobian(r.contiguous(), x.contiguous(), parameterization=par, convention="ZXY", n_points=64)
        torch.cuda.synchronize()
        print(renderer, par, "jacobian ok", tuple(J.shape), float(J.abs().max()))
# image losses: patch-wise NCC (p = 1, a single window row), blur + Sobel with halos past both image edges and a wide blur
for shape, losses in (((2, 1, 37, 45), (MultiscaleNormalizedCrossCorrelation2d([None, 5, 1], [0.5, 0.3, 0.2]),
                                        GradientNormalizedCrossCorrelation2d(patch_size=9), GradientNormalizedCrossCorrelation2d(sigma=2.5))),
                      ((1, 1, 9, 70), (MultiscaleNormalizedCrossCorrelation2d([9], [1.0]), GradientNormalizedCrossCorrelation2d(sigma=0.0)))):
    for loss in losses:
        a = torch.rand(*shape, device=dev).requires_grad_(True)
        b = torch.rand(*shape, device=dev).requires_grad_(True)
        loss(a, b).sum().backward()
        torch.cuda.synchronize()
        print(shape, type(loss).__name__, "ok", float(a.grad.abs().max()), float(b.grad.abs().max()))
# mutual information: 64- and 128-bin tiles with partial tails, ragged pixel chunks, one and both gradients
for shape, nb in (((2, 1, 37, 45), 37), ((1, 1, 9, 70), 100), ((3, 1, 33, 17), 256)):
    mi = MutualInformation(num_bins=nb).to(dev)
    a = torch.rand(*shape, device=dev).requires_grad_(True)
    b = torch.rand(*shape, device=dev).requires_grad_(True)
    mi(a, b).sum().backward()
    mi(a.detach(), b).sum().backward()
    torch.cuda.synchronize()
    print(shape, nb, "MutualInformation ok", float(a.grad.abs().max()), float(b.grad.abs().max()))
# NCC normal equations (ncc_normal.cu): partial window tiles and pixel chunks, p = 1, p = min(H, W), global, P = 1 and 16
from diffdrr_b200.registration import ncc_normal_equations  # noqa: E402
for (B, C, H, W), P, ps in (((2, 2, 37, 45), 1, (None, 1, 5, 37)), ((1, 1, 9, 70), 16, (None, 3, 9)), ((3, 2, 67, 13), 6, (13, None))):
    x, t = torch.rand(B, C, H, W, device=dev), torch.rand(B, C, H, W, device=dev)
    J = torch.randn(B, P, C, H, W, device=dev)
    for p in ps:
        A = torch.zeros(B, P, P, dtype=torch.float64, device=dev)
        g = torch.zeros(B, P, dtype=torch.float64, device=dev)
        ncc_normal_equations(x, t, J, (P * C * H * W, H * W, C * H * W, 1), p, 1e-5, 1.0, A, g)
        torch.cuda.synchronize()
        print((B, C, H, W), P, p, "ncc_normal ok", float(A.abs().max()), float(g.abs().max()))
# blended-rigid render (polyrigid.cu): a detector that is not a multiple of the 16 x 8 tiles, K = 3 (one padded channel), a lattice
# that does not divide the volume, per-pose motions, plain and sub-sampled (ragged) ray sets, fp32 and bf16 densities
from diffdrr_b200.structures import se3_exp  # noqa: E402
for kw, dtype in ((dict(), torch.float32), (dict(p_subsample=0.37), torch.float32), (dict(), torch.bfloat16)):
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer="trilinear", **kw).to(dev)
    drr.density = drr.density.to(dtype)
    W = torch.rand(3, 7, 5, 9, device=dev) / 3
    xi = ((torch.rand(3, 3, 6, device=dev) - 0.5) * torch.tensor([0.1, 0.1, 0.1, 8.0, 8.0, 8.0], device=dev)).requires_grad_(True)
    r, x = rot.detach().clone().requires_grad_(True), xyz.detach().clone().requires_grad_(True)
    img = drr.render_polyrigid(r, x, motions=se3_exp(xi), weights=W, n_points=64, parameterization="euler_angles", convention="ZXY")
    img.sum().backward()
    torch.cuda.synchronize()
    print("polyrigid", kw, dtype, "ok", float(img.sum()), float(r.grad.abs().max()), float(xi.grad.abs().max()))
# deformable render (deform.cu): the same detectors and densities, a 7 x 5 x 9 field per pose that pulls samples out of the volume
# and back, and a shared one, with the field scatter
for kw, dtype in ((dict(), torch.float32), (dict(p_subsample=0.37), torch.float32), (dict(), torch.bfloat16)):
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer="trilinear", **kw).to(dev)
    drr.density = drr.density.to(dtype)
    for shape in ((rot.shape[0], 3, 7, 5, 9), (3, 7, 5, 9)):
        u = ((torch.rand(*shape, device=dev) - 0.5) * 80.0).requires_grad_(True)
        r, x = rot.detach().clone().requires_grad_(True), xyz.detach().clone().requires_grad_(True)
        img = drr.render_deformed(r, x, field=u, n_points=64, parameterization="euler_angles", convention="ZXY")
        img.sum().backward()
        torch.cuda.synchronize()
        print("deform", kw, dtype, shape, "ok", float(img.sum()), float(r.grad.abs().max()), float(u.grad.abs().max()))
# blended-rigid motion Jacobian (polyrigid.cu: polyrigid_jac_kernel): the 23 x 23 detector (partial 16 x 8 tiles and partial warp
# bundles), K = 3, per-pose and shared motions, fp32 and bf16 densities
for dtype in (torch.float32, torch.bfloat16):
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer="trilinear").to(dev)
    drr.density = drr.density.to(dtype)
    W = torch.rand(3, 7, 5, 9, device=dev) / 3
    for shape in ((rot.shape[0], 3, 6), (3, 6)):
        xi = (torch.rand(*shape, device=dev) - 0.5) * torch.tensor([0.1, 0.1, 0.1, 8.0, 8.0, 8.0], device=dev)
        img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=se3_exp(xi), weights=W, n_points=64, return_footprints=True,
                                               parameterization="euler_angles", convention="ZXY")
        torch.cuda.synchronize()
        print("polyrigid_jac", dtype, shape, "ok", float(img.sum()), float(J.abs().max()), rects.tolist())
# deformable tangent march (deform.cu: deform_jvp_kernel): the 23 x 23 detector (partial 16 x 8 tiles), p_subsample (128-ray
# chunks), per-pose and shared fields that pull samples out of the volume and back, fp32 and bf16 densities
for kw, dtype in ((dict(), torch.float32), (dict(p_subsample=0.37), torch.float32), (dict(), torch.bfloat16)):
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer="trilinear", **kw).to(dev)
    drr.density = drr.density.to(dtype)
    for shape in ((rot.shape[0], 3, 7, 5, 9), (3, 7, 5, 9)):
        u, v = (torch.rand(*shape, device=dev) - 0.5) * 80.0, torch.rand(*shape, device=dev) - 0.5
        img, dimg = drr.deformed_jvp(rot, xyz, field=u, tangent=v, n_points=64, parameterization="euler_angles", convention="ZXY")
        torch.cuda.synchronize()
        print("deform_jvp", kw, dtype, shape, "ok", float(img.sum()), float(dimg.abs().max()))
# deformable density backprojection (deform.cu: deform_bproj_kernel): the 23 x 23 detector (partial 16 x 8 tiles), p_subsample
# (128-ray chunks) and patches, per-pose and shared fields that pull samples out of the volume and back, the density alone and
# jointly with the field
for kw in (dict(), dict(p_subsample=0.37), dict(patch_size=8, height=24)):
    kw = dict(kw)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(kw.pop("height", 23)), renderer="trilinear", **kw).to(dev)
    for shape in ((rot.shape[0], 3, 7, 5, 9), (3, 7, 5, 9)):
        for joint in (False, True):
            u = ((torch.rand(*shape, device=dev) - 0.5) * 80.0).requires_grad_(joint)
            V = drr.density.detach().clone().requires_grad_(True)
            img = drr.render_deformed(rot, xyz, field=u, n_points=64, density=V, parameterization="euler_angles", convention="ZXY")
            img.sum().backward()
            torch.cuda.synchronize()
            print("deform_bproj", kw, shape, joint, "ok", float(img.sum()), float(V.grad.abs().max()))
# tangent of a squaring step (svf.cu: svf_square_jvp_kernel) and the velocity LM over it: a 7 x 5 x 9 lattice (partial CTA), shared
# and per-pose velocities large enough that many lookups clamp, with and without the primal output
from diffdrr_b200 import DiffeomorphicLevenbergMarquardt, exp_velocity_jvp  # noqa: E402

drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer="trilinear").to(dev)
for shape in ((rot.shape[0], 3, 7, 5, 9), (3, 7, 5, 9)):
    v, t = (torch.rand(*shape, device=dev) - 0.5) * 80.0, torch.rand(*shape, device=dev) - 0.5
    u, du = exp_velocity_jvp(drr, v, t, steps=4)
    with torch.no_grad():
        target = drr.render_deformed(rot, xyz, field=u, n_points=64, parameterization="euler_angles", convention="ZXY")
    lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, torch.zeros_like(v), target, steps=4, cg_iters=2, n_points=64,
                                         parameterization="euler_angles", convention="ZXY")
    E = lm.step()
    torch.cuda.synchronize()
    print("svf_jvp", shape, "ok", float(du.abs().max()), E.tolist())
# blended-rigid density backprojection (polyrigid.cu: polyrigid_bproj_kernel): the 23 x 23 detector (partial 16 x 8 tiles),
# p_subsample (128-ray chunks) and patches, K = 3 and 6 (both channel paddings), per-pose and shared motions, a structure pulled
# from outside the volume, the density alone and jointly with the motions
for kw in (dict(), dict(p_subsample=0.37), dict(patch_size=8, height=24)):
    kw = dict(kw)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(kw.pop("height", 23)), renderer="trilinear", **kw).to(dev)
    for K in (3, 6):
        W = torch.rand(K, 7, 5, 9, device=dev) / K
        for shape in ((rot.shape[0], K, 6), (K, 6)):
            for joint in (False, True):
                xi = (torch.rand(*shape, device=dev) - 0.5) * torch.tensor([0.1, 0.1, 0.1, 8.0, 8.0, 8.0], device=dev)
                xi[..., 0, 3] += 300.0
                xi.requires_grad_(joint)
                V = drr.density.detach().clone().requires_grad_(True)
                r, x = (t.detach().clone().requires_grad_(joint) for t in (rot, xyz))
                img = drr.render_polyrigid(r, x, motions=se3_exp(xi), weights=W, n_points=64, density=V,
                                           parameterization="euler_angles", convention="ZXY")
                img.sum().backward()
                torch.cuda.synchronize()
                print("polyrigid_bproj", kw, K, shape, joint, "ok", float(img.sum()), float(V.grad.abs().max()))
# log-Euclidean motion Jacobian (svf.cu: svf_square_tangents_kernel; deform.cu: deform_jac_kernel): the 23 x 23 detector (partial
# 16 x 8 tiles), a 7 x 5 x 9 lattice (partial CTA), K = 3 and 6 (both register paddings), per-pose and shared motions, a structure
# pulled from outside the volume, fp32 and bf16 densities
for dtype in (torch.float32, torch.bfloat16):
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(23), renderer="trilinear").to(dev)
    drr.density = drr.density.to(dtype)
    for K in (3, 6):
        W = torch.rand(K, 7, 5, 9, device=dev) / K
        for shape in ((rot.shape[0], K, 6), (K, 6)):
            xi = (torch.rand(*shape, device=dev) - 0.5) * torch.tensor([0.1, 0.1, 0.1, 8.0, 8.0, 8.0], device=dev)
            xi[..., 0, 3] += 300.0
            img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=se3_exp(xi), weights=W, n_points=64, return_footprints=True,
                                                   blend="log_euclidean", steps=4, parameterization="euler_angles", convention="ZXY")
            torch.cuda.synchronize()
            print("log_euclidean_jac", dtype, K, shape, "ok", float(img.sum()), float(J.abs().max()), rects.tolist())
print("done")
