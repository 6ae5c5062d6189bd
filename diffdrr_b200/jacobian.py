"""Per-pixel pose Jacobians of the fused pose-in renderers (`DRR.jacobian`; DESIGN.md 6e).

Every pixel of a pose-in render depends on one ray, and the training walk already stores that ray's end-point partials (the
sensitivities, include/b200drr.h).  So the N x p Jacobian of pose b's image with respect to its p parameters is
  1. the sensitivities walk (the kernel the training step runs),
  2. the tangents of theta -> (src, G, Wd), the pose-in kernels' inputs, computed here in float64 by forward-mode AD of the
     torch statement of that map (pose.convert + drr.pose_in_matrices), and for Trilinear the tangent of the batch-global
     sampling range,
  3. one streaming kernel that contracts the two per pixel (b200drr_siddon_jac_sens_pose / b200drr_trilinear_jac_sens_pose).
"""
from __future__ import annotations

import torch

from . import _lib, geometry
from .pose import PARAMETERIZATIONS, RigidTransform, convert
from .renderers import (_VOL16, Siddon, Trilinear, _check_vol16, _dims_tensor, _get_alpha_minmax, _ptr, _siddon_sens_pose,
                        _stream, _trilinear_sens_pose, pose_alpha_range)


def pose_in_tangents(rot, xyz, parameterization, convention, degrees, reorient, calib, A_inv):
    """d(src, G, Wd)/d theta of every pose in float64, theta = (the rotation's components, then the translation's 3):
    -> dsrc (B, p, 3), dG (B, p, 3, 4), dWd (B, p, 3, 4).

    The poses are independent, so one forward-mode pass over p stacked copies of the batch -- copy k carries the unit tangent of
    parameter k for every pose -- yields all p columns at once, with no host synchronisation."""
    from .drr import pose_in_matrices

    rot, xyz = rot.detach().double(), xyz.detach().double()
    B, r = rot.shape
    p = r + 3
    eye = torch.eye(p, dtype=torch.float64, device=rot.device)
    # dual tensors need their own memory: no stride-0 (expanded) views as primals or tangents
    stack = lambda x, n: x.unsqueeze(0).expand(p, B, n).reshape(p * B, n).clone()  # noqa: E731
    consts = (reorient.detach().double(), calib.detach().double(), A_inv.detach().double())

    def f(a, t):
        P = convert(a, t, parameterization=parameterization, convention=convention, degrees=degrees).matrix
        return pose_in_matrices(P, *consts)

    _, (dsrc, dG, dWd) = torch.func.jvp(f, (stack(rot, r), stack(xyz, 3)),
                                        (eye[:, None, :r].expand(p, B, r).reshape(p * B, r).clone(),
                                         eye[:, None, r:].expand(p, B, 3).reshape(p * B, 3).clone()))
    return (dsrc.view(p, B, 3).transpose(0, 1), dG.view(p, B, 3, 4).transpose(0, 1), dWd.view(p, B, 3, 4).transpose(0, 1))


def range_tangents(shape, voxel_shift, eps, src, G, rows, cols, arg, dsrc, dG):
    """drange (B, 2, p) float64: the derivative of the batch-global {alphamin, alphamax} with respect to pose b's parameters.

    renderers.pose_alpha_range rebuilds the range from the two rays that attain it (indices `arg`, on the device); this
    differentiates that same rebuild along the tangents (dsrc, dG).  Only the rows of the (at most two) poses owning an extreme
    ray are nonzero."""
    H, W = rows.numel(), cols.numel()
    B, p = dsrc.shape[0], dsrc.shape[1]
    dev = src.device
    b, n = arg // (H * W), arg % (H * W)
    one = torch.ones(2, dtype=torch.float64, device=dev)
    pt = torch.stack([cols.double()[n % W], rows.double()[n // W], one, one], dim=-1)           # (2, 4)
    src2 = src[b].double().unsqueeze(1).expand(2, p, 3).clone()  # dual tensors: no stride-0 views
    tgt2 = torch.einsum("kij,kj->ki", G[b].double(), pt).unsqueeze(1).expand(2, p, 3).clone()
    dims = _dims_tensor(shape, dev, torch.float64)

    def f(s, t):
        amin, amax = _get_alpha_minmax(s, t, dims, voxel_shift, eps)
        return torch.stack([amin[0, :, 0], amax[1, :, 0]])                                      # (2, p)

    _, d = torch.func.jvp(f, (src2, tgt2), (dsrc[b].contiguous(), torch.einsum("kpij,kj->kpi", dG[b], pt).contiguous()))
    drange = torch.zeros(B, 2, p, dtype=torch.float64, device=dev)
    drange.index_put_((b, torch.arange(2, device=dev)), d)
    return drange


def _params(args):
    if len(args) != 2 or not all(torch.is_tensor(a) for a in args):
        raise ValueError("jacobian takes the pose as two tensors: rotation parameters (B, r) and translation (B, 3)")
    rot, xyz = args
    if rot.dim() != 2 or xyz.dim() != 2 or xyz.shape[-1] != 3 or rot.shape[0] != xyz.shape[0]:
        raise ValueError(f"jacobian needs rotation (B, r) and translation (B, 3) with one batch size, got {tuple(rot.shape)} "
                         f"and {tuple(xyz.shape)}: every pose owns its parameters")
    return rot, xyz


def check_supported(drr, parameterization, args):
    """Refuse, before any launch, what the fused pose-in paths do not cover."""
    if parameterization is None or parameterization == "matrix":
        raise ValueError("jacobian needs pose parameters (a parameterization other than 'matrix'): the columns of J are the "
                         "derivatives with respect to them")
    if parameterization not in PARAMETERIZATIONS:
        raise ValueError(f"Must be in {PARAMETERIZATIONS}, not {parameterization}")
    _params(args)
    if drr.detector.n_subsample is not None:
        raise NotImplementedError("jacobian renders the full detector grid: the pose-in kernels generate every pixel's ray, "
                                  "a sub-sampled detector (p_subsample) has no such grid")
    if drr.patch_size is not None:
        raise NotImplementedError("jacobian renders the full detector grid in one pass; patch_size is not supported")
    r = drr.renderer
    if isinstance(r, Siddon):
        if r.mode != "nearest" or not isinstance(r.reducefn, str) or r.reducefn != "sum" or r.filter_intersections_outside_volume:
            raise NotImplementedError("jacobian supports Siddon with its default options (mode='nearest', reducefn='sum'), with "
                                      "or without stop_gradients_through_grid_sample: the sensitivities walk implements those")
    elif isinstance(r, Trilinear):
        if r.mode != "bilinear" or not isinstance(r.reducefn, str) or r.reducefn != "sum":
            raise NotImplementedError("jacobian supports Trilinear with its default options (mode='bilinear', reducefn='sum'): "
                                      "the sensitivities march implements those")
    else:
        raise NotImplementedError(f"jacobian supports the Siddon and Trilinear renderers, not {type(r).__name__}")
    vol = drr.density
    if vol.dtype == torch.float64:
        raise NotImplementedError("jacobian runs the fp32 sensitivities kernels: an fp64 density has no such walk (render it "
                                  "in fp32, fp16 or bf16)")
    if vol.dtype not in (torch.float32, *_VOL16) or vol.dim() != 3 or vol.numel() >= 2**31 - 1:
        raise NotImplementedError(f"jacobian needs a 3-D fp32 / fp16 / bf16 density below 2^31 voxels, got {vol.dtype} "
                                  f"{tuple(vol.shape)}")
    if not vol.is_cuda:
        raise _lib.B200DRRError(f"diffdrr_b200 renderers run on CUDA devices only (density is on {vol.device}); there is no "
                                "CPU fallback")
    if isinstance(r, Trilinear) and (not r.pack_corners or vol.requires_grad):
        raise NotImplementedError("jacobian with Trilinear reads the packed-corner copy of a static volume: the density must "
                                  "not require grad and pack_corners must be on")


def drr_jacobian(drr, *args, parameterization, convention=None, degrees=False, calibration=None, n_points=500,
                 return_range_terms=False, stop_grad=None):
    """See DRR.jacobian.  stop_grad: drop Siddon's ray-length term (None = the renderer's
    stop_gradients_through_grid_sample); LevenbergMarquardt models the image itself, so it asks for the full derivative."""
    check_supported(drr, parameterization, args)
    rot, xyz = _params(args)
    r, vol = drr.renderer, drr.density
    trilinear = isinstance(r, Trilinear)
    with torch.no_grad():
        packed = r._packed_volume(vol) if trilinear else None
        if trilinear and packed is None:
            raise NotImplementedError("jacobian with Trilinear reads the packed-corner copy of the volume, and it could not be "
                                      "made (pack_corners_max_bytes or device memory)")
        # the pose exactly as DRR.forward builds it, so that `img` is the image drr(...) renders
        if (parameterization == "euler_angles" and calibration is None and geometry.euler_convention_ok(convention)
                and all(a.is_cuda and a.dtype == torch.float32 for a in (rot, xyz))):
            pose = RigidTransform(geometry.euler_pose(rot.detach(), xyz.detach(), convention, degrees))
        else:
            pose = convert(rot.detach(), xyz.detach(), parameterization=parameterization, convention=convention,
                           degrees=degrees)
        src, G, Wd, rows, cols = drr._pose_in_inputs(pose, calibration)
        det = drr.detector
        calib = det._calibration if calibration is None else calibration.matrix
        tangents = pose_in_tangents(rot, xyz, parameterization, convention, degrees, det._reorient, calib, drr._affine_inverse)
        dsrc, dG, dWd = (t.float().contiguous() for t in tangents)
        B, H, W, P = G.shape[0], rows.numel(), cols.numel(), dsrc.shape[1]
        src, G, Wd = src.contiguous().float(), G.contiguous().float(), Wd.contiguous().float()
        rows, cols = rows.contiguous().float(), cols.contiguous().float()
        dev = vol.device
        J = torch.empty(B, H * W, P, dtype=torch.float32, device=dev)
        lib = _lib.load()
        if vol.dtype in _VOL16:
            _check_vol16(vol, src, G)
        with torch.cuda.device(dev):
            if not trilinear:
                out, sens = _siddon_sens_pose(vol.contiguous(), src, G, Wd, rows, cols, float(r.voxel_shift), float(r.eps))
                stop_grad = int(bool(r.stop_gradients_through_grid_sample if stop_grad is None else stop_grad))
                _lib.check(lib.b200drr_siddon_jac_sens_pose(_ptr(sens), _ptr(dsrc), _ptr(dG), _ptr(dWd), _ptr(Wd), _ptr(rows),
                                                            _ptr(cols), _ptr(J), B, H, W, P, stop_grad, _stream()),
                           "b200drr_siddon_jac_sens_pose")
                range_terms = (None, None, None)
            else:
                alpha_range, arg = pose_alpha_range(r, vol, src, G, Wd, rows, cols)
                arange = alpha_range.float().contiguous()
                drange = range_tangents(vol.shape, float(r.voxel_shift), float(r.eps), src, G, rows, cols, arg, tangents[0],
                                        tangents[1])
                drange = drange.float().contiguous()
                out, sens = _trilinear_sens_pose(vol, packed, src, G, Wd, rows, cols, float(r.voxel_shift), float(r.eps),
                                                 int(n_points), arange)
                _lib.check(lib.b200drr_trilinear_jac_sens_pose(_ptr(sens), _ptr(dsrc), _ptr(dG), _ptr(dWd), _ptr(Wd), _ptr(rows),
                                                               _ptr(cols), _ptr(drange), _ptr(J), B, H, W, P, _stream()),
                           "b200drr_trilinear_jac_sens_pose")
                range_terms = (sens[..., 7], sens[..., 8], drange)
    img = drr.reshape_transform(out.view(B, 1, H * W), batch_size=B)
    J = J.view(*img.shape, P)
    if not return_range_terms:
        return img, J
    if range_terms[0] is not None:
        range_terms = (range_terms[0].reshape(img.shape), range_terms[1].reshape(img.shape), range_terms[2])
    return img, J, range_terms
