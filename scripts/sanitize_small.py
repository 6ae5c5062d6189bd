#!/usr/bin/env python
"""Small invocations of the round-2 kernels for compute-sanitizer (memcheck / racecheck / synccheck): brick-major TMA forward
(several bricks per CTA, partial bricks, two pose chunks), the locality-ordered slab kernels, the brick scatter (volume gradient),
the mask grid kernels, the un-reduced segment kernels, fp64, the trilinear pose-in step and the image losses (global and
patch-wise NCC, blur + Sobel, on sizes that are not a multiple of the tiles); PeerGather is multi-GPU only."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from diffdrr_b200 import (DRR, GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d, Siddon,  # noqa: E402
                          _lib, renderers, synthetic)
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
    for v in (0, 7):
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
print("done")
