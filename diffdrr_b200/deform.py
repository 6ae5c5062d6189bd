"""Deformable DRRs (`DRR.render_deformed`; DESIGN.md 6i): the volume under a dense displacement field, marched with the Trilinear
renderer's rays and samples.

Every sample at world point p reads the CT density at p + u(p): u is a pull-back displacement in world millimetres given on a
lattice over the volume (polyrigid.py's convention: node i of axis a at voxel coordinate (i + 1/2) D_a / g_a - 1/2, trilinear,
zero outside the lattice).  The kernels take u in voxel-index units, channel-last and padded to 4 channels; that conversion is
torch ops here, so autograd carries the kernel's field gradient (include/b200drr.h: b200drr_deform_bwd) back to the world-mm field
and on to whatever produced it.  Nothing is cached and nothing is read on the host: the field changes every optimiser step.

A density passed as `density=` may require grad (fp32): its gradient is the forward's transpose in the density, a backprojection
along the warped samples (b200drr_deform_bproj; DESIGN.md 6l), for motion-compensated reconstruction.
"""
from __future__ import annotations

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .pose import RigidTransform
from .renderers import _VOL16, Trilinear, _check_vol16, _dims_tensor, _get_alpha_minmax, _ptr, _stream, _vol_entry
from .structures import _batch_size, _camera_pose


def _check_renderer(drr, name, warp, kwargs):
    """The warped renders' (render_polyrigid, render_deformed: `name`) refusals of the renderer and its options, before any launch.
    warp: what bends the rays, for the message."""
    r = drr.renderer
    if not isinstance(r, Trilinear):
        raise NotImplementedError(f"{name} supports the Trilinear renderer, not {type(r).__name__}: {warp} bends the rays inside "
                                  "the volume, and Siddon's voxel walk follows straight lines")
    if r.mode != "bilinear" or not isinstance(r.reducefn, str) or r.reducefn != "sum":
        raise NotImplementedError(f"{name} supports Trilinear with its default options (mode='bilinear', reducefn='sum')")
    if kwargs.get("align_corners", False) or kwargs.get("mask") is not None or kwargs.get("mask_to_channels", False) or \
            set(kwargs) - {"align_corners", "mask", "mask_to_channels"}:
        raise NotImplementedError(f"{name} takes no renderer options besides n_points, alphamin and alphamax, got {sorted(kwargs)}")


def _check_density(vol, name, no_grad):
    """The warped renders' refusals of the density `vol`, before any launch: no_grad is the message refusing a density that
    requires grad, or None where the render has a gradient for it."""
    if vol.dtype not in (torch.float32, *_VOL16) or vol.dim() != 3 or vol.numel() >= 2**31 - 1:
        raise NotImplementedError(f"{name} needs a 3-D fp32 / fp16 / bf16 density below 2^31 voxels, got {vol.dtype} "
                                  f"{tuple(vol.shape)}")
    if vol.requires_grad and no_grad is not None:
        raise NotImplementedError(no_grad)
    if not vol.is_cuda:
        raise _lib.B200DRRError(f"diffdrr_b200 renderers run on CUDA devices only (density is on {vol.device}); there is no CPU "
                                "fallback")


def _rendered_density(drr, density, name, no_grad):
    """The density a warped render `name` marches -> (vol, the refusal _check_density takes): drr.density with `no_grad`, the
    refusal of a drr.density that requires grad; or the volume passed as density=, which must have drr.density's shape and device,
    and may require grad when it is fp32."""
    vol = drr.density
    if density is None:
        return vol, no_grad
    # the module keeps the geometry (affine, dims); the volume fitted through it is passed in
    if not torch.is_tensor(density) or density.shape != vol.shape or density.device != vol.device:
        got = f"{tuple(density.shape)} on {density.device}" if torch.is_tensor(density) else type(density).__name__
        raise ValueError(f"density must be a tensor of drr.density's shape {tuple(vol.shape)} on its device {vol.device}, got {got}")
    if density.dtype != torch.float32:
        return density, (f"{name} produces no volume gradient to a {density.dtype} density: 16-bit volumes are static densities "
                         "(optimise an fp32 volume for volume gradients)")
    return density, None


def check_supported(drr, args, parameterization, field, kwargs, density=None):
    """Refuse, before any launch, what the deformable render does not cover: -> B.  density: the volume rendered in place of
    drr.density (render_deformed's density=), or None."""
    _check_renderer(drr, "render_deformed", "the displacement field", kwargs)
    B = _batch_size(args, parameterization)
    if not torch.is_tensor(field) or field.dtype != torch.float32 or field.dim() not in (4, 5) or field.shape[-4] != 3 or \
            (field.dim() == 5 and field.shape[0] != B) or min(field.shape[-3:]) < 1:
        got = f"{field.dtype} {tuple(field.shape)}" if torch.is_tensor(field) else type(field).__name__
        raise ValueError(f"field must be an fp32 displacement lattice (3, g0, g1, g2) or (B={B}, 3, g0, g1, g2), got {got}")
    g0, g1, g2 = field.shape[-3:]
    if 4 * g0 * g1 * g2 >= 2**31 - 1:
        raise NotImplementedError(f"render_deformed takes a lattice below 2^31 floats per pose (4 channels), got {(g0, g1, g2)}")
    vol, no_grad = _rendered_density(drr, density, "render_deformed",
                                     "render_deformed produces no volume gradient to drr.density: the density must not require grad "
                                     "(pass the volume to fit as density= instead)")
    _check_density(vol, "render_deformed", no_grad)
    if field.device != vol.device:
        raise ValueError(f"field must be on the density's device {vol.device}, not {field.device}")
    return B


def _launch_args(name, vol, packed, source, target, raylen, grid):
    """The leading arguments of a warped-render entry point `name` (b200drr_polyrigid_*, b200drr_deform_*) -> (entry point: `name`
    or its 16-bit twin, its (vol, packed[, vol_type]) with exactly one of the two arrays passed, its name, (src (B, 3), tgt
    (B, N, 3), raylen (B, N)) contiguous fp32, (H, W) of a full detector grid or (0, 0) for any other ray set)."""
    B, N = target.shape[0], target.shape[1]
    fn, head, name = _vol_entry(_lib.load(), name, vol)
    head = (_ptr(vol) if packed is None else None, _ptr(packed), *head[1:])
    rays = (source.reshape(B, 3).contiguous().float(), target.contiguous().float(), raylen.reshape(B, N).contiguous().float())
    return fn, head, name, rays, (grid if grid is not None and grid[0] * grid[1] == N else (0, 0))


class _DeformFunction(torch.autograd.Function):
    """out (B, 1, N) for rays in voxel-index space, the kernels' field (Bf, g0, g1, g2, 4) in voxel units and the range
    alpha_range = [alphamin, alphamax]; the density comes from its packed-corner copy when there is one, fp32 or 16-bit, through
    the entry point that takes it."""

    @staticmethod
    def forward(ctx, volume, packed, source, target, img, field, alpha_range, voxel_shift, eps, n_points, grid):
        vol = volume.contiguous()
        fn, head, name, (src, tgt, raylen), (H, W) = _launch_args("b200drr_deform_fwd", vol, packed, source, target, img, grid)
        B, N = tgt.shape[0], tgt.shape[1]
        field = field.contiguous()
        arange = alpha_range.detach().to(device=vol.device, dtype=torch.float32).contiguous()
        out = torch.empty(B, N, dtype=torch.float32, device=vol.device)
        geom = (*vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(field), field.shape[0], *field.shape[1:4])
        with torch.cuda.device(vol.device):
            _lib.check(fn(*head, *geom, _ptr(out), B, N, H, W, voxel_shift, eps, n_points, _ptr(arange), _stream()), name)
        ctx.save_for_backward(vol, packed, src, tgt, raylen, field, arange)
        ctx.consts = (voxel_shift, eps, n_points, H, W, source.shape, img.shape)
        return out.view(B, 1, N)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        vol, packed, src, tgt, raylen, field, arange = ctx.saved_tensors
        voxel_shift, eps, n_points, H, W, source_shape, img_shape = ctx.consts
        B, N = tgt.shape[0], tgt.shape[1]
        dev = vol.device
        gout = gout.reshape(B, N).contiguous().float()
        lib = _lib.load()
        g_vol = None
        if ctx.needs_input_grad[0]:   # the forward's transpose in the density: a backprojection, no density read
            g_vol = torch.empty(vol.shape, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.b200drr_deform_bproj(*vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(field), field.shape[0],
                                                    *field.shape[1:4], _ptr(gout), _ptr(g_vol), B, N, H, W, voxel_shift, eps,
                                                    n_points, _ptr(arange), _stream()), "b200drr_deform_bproj")
        if not any(ctx.needs_input_grad[2:7]):   # a reconstruction step: the density is the only input that wants a gradient
            return g_vol, None, None, None, None, None, None, None, None, None, None
        g_src = torch.empty(B, 3, dtype=torch.float32, device=dev)
        g_tgt = torch.empty(B, N, 3, dtype=torch.float32, device=dev)
        g_raylen = torch.empty(B, N, dtype=torch.float32, device=dev)
        g_field = torch.empty_like(field) if ctx.needs_input_grad[5] else None   # NULL: the kernel skips the scatter
        g_range = torch.empty(2, dtype=torch.float32, device=dev)
        scratch = torch.empty(int(lib.b200drr_deform_scratch_floats(B, N, H, W)), dtype=torch.float32, device=dev)
        fn, head, name, _, _ = _launch_args("b200drr_deform_bwd", vol, packed, src, tgt, raylen, (H, W))
        with torch.cuda.device(dev):
            _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(field), field.shape[0], *field.shape[1:4],
                          _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_raylen), _ptr(g_field), _ptr(g_range), _ptr(scratch),
                          B, N, H, W, voxel_shift, eps, n_points, _ptr(arange), _stream()), name)
        return g_vol, None, g_src.view(source_shape), g_tgt, g_raylen.view(img_shape), g_field, g_range, None, None, None, None


def voxel_field(drr, field):
    """World-mm pull-back displacements (3, g0, g1, g2) or (B, 3, g0, g1, g2) -> the kernels' field (Bf, g0, g1, g2, 4): voxel-index
    vectors (the 3 x 3 linear part of drr.affine_inverse), channel last, a zero fourth channel.  Torch ops, differentiable."""
    lin = drr._affine_inverse.reshape(4, 4)[:3, :3].to(field.dtype)
    f = field if field.dim() == 5 else field[None]
    u = torch.einsum("ij,bjxyz->bxyzi", lin, f)
    return torch.nn.functional.pad(u, (0, 1)).contiguous()


def _marches(drr, args, B, parameterization, convention, degrees, calibration, alphamin, alphamax, vol=None):
    """The rays of a warped render in voxel-index space -> (source (B, 1, 3), marches of (target, raylen, alpha_range, grid)): a
    list of one march for the full or sub-sampled detector, or for patch_size (as DRR.render) an iterator of one march per patch
    whose range is built when the iterator reaches it.  Each march has its own sampling range (the batch-global range of its rays,
    as Trilinear.forward, unless alphamin / alphamax fix it) and, for a full detector grid, its (H, W).  Torch ops, differentiable
    in the camera pose and the calibration; the order in which the ranges and the marches are built is the order in which
    autograd sums their fp32 contributions to the camera gradient.  vol: the density rendered (default drr.density)."""
    vol, r = drr.density if vol is None else vol, drr.renderer
    P = _camera_pose(args, B, parameterization, convention, degrees)
    source, target = drr.detector(RigidTransform(P), calibration)
    img = (target - source).norm(dim=-1).unsqueeze(1)
    source, target = drr.affine_inverse(source), drr.affine_inverse(target)
    if vol.dtype in _VOL16:
        _check_vol16(vol, source, target)
    det = drr.detector
    full_grid = det.n_subsample is None and drr.patch_size is None
    dims = _dims_tensor(vol.shape, source.device, source.dtype)

    def march(tgt, lens, grid):
        if alphamin is None or alphamax is None:   # the batch-global range of the rays in this call, as Trilinear.forward
            amin, amax = _get_alpha_minmax(source, tgt, dims, r.voxel_shift, r.eps)
            lo, hi = amin.min(), amax.max()
        else:
            lo, hi = alphamin, alphamax
        alpha_range = torch.stack([torch.as_tensor(lo, dtype=torch.float32, device=vol.device),
                                   torch.as_tensor(hi, dtype=torch.float32, device=vol.device)])
        return tgt, lens, alpha_range, grid

    if drr.patch_size is None:
        return source, [march(target, img, (det.height, det.width) if full_grid else None)]
    return source, (march(t, i, None) for t, i in zip(target.chunk(drr.n_patches, dim=1), img.chunk(drr.n_patches, dim=-1)))


def render_deformed(drr, *args, field, parameterization=None, convention=None, degrees=False, calibration=None, n_points=500,
                    alphamin=None, alphamax=None, density=None, **kwargs):
    """See DRR.render_deformed."""
    B = check_supported(drr, args, parameterization, field, kwargs, density=density)
    vol = drr.density if density is None else density
    return render_voxel_field(drr, args, B, voxel_field(drr, field), parameterization, convention, degrees, calibration, n_points,
                              alphamin, alphamax, vol)


def render_voxel_field(drr, args, B, U, parameterization, convention, degrees, calibration, n_points, alphamin, alphamax, vol):
    """render_deformed after its checks, for the kernels' field U (Bf, g0, g1, g2, 4) in voxel units (voxel_field's output)."""
    r = drr.renderer
    source, marches = _marches(drr, args, B, parameterization, convention, degrees, calibration, alphamin, alphamax, vol=vol)
    marches = list(marches)   # every patch's range before the first march (render_polyrigid builds each just before its march)
    packed = r._packed_volume(vol)
    outs = [_DeformFunction.apply(vol, packed, source, tgt, lens, U, alpha_range, float(r.voxel_shift), float(r.eps), int(n_points),
                                  grid) for tgt, lens, alpha_range, grid in marches]
    out = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)   # serial patches with a range each, as DRR.render
    return drr.reshape_transform(out, batch_size=B)


def _check_tangent(field, tangent):
    if not torch.is_tensor(tangent) or tangent.shape != field.shape or tangent.dtype != field.dtype or tangent.device != field.device:
        got = f"{tangent.dtype} {tuple(tangent.shape)} on {tangent.device}" if torch.is_tensor(tangent) else type(tangent).__name__
        raise ValueError(f"tangent must be a field of the same shape, dtype and device as `field` ({field.dtype} "
                         f"{tuple(field.shape)} on {field.device}), got {got}")


def field_jvp(drr, packed, source, target, raylen, U, T, alpha_range, n_points, grid, img=None):
    """The directional derivative of one march along the voxel-unit tangent T (b200drr_deform_jvp): rays in voxel-index space
    (source (B, 1, 3), target (B, N, 3), raylen (B, 1, N)), U and T the kernels' fields (Bf, g0, g1, g2, 4) -> jv (B, N); `img`
    (B, N) fp32, if given, receives the march's image.  No autograd."""
    vol, r = drr.density, drr.renderer
    fn, head, name, (src, tgt, lens), (H, W) = _launch_args("b200drr_deform_jvp", vol, packed, source, target, raylen, grid)
    B, N = tgt.shape[0], tgt.shape[1]
    jv = torch.empty(B, N, dtype=torch.float32, device=vol.device)
    with torch.cuda.device(vol.device):
        _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(lens), _ptr(U), U.shape[0], *U.shape[1:4], _ptr(T), _ptr(img),
                      _ptr(jv), B, N, H, W, float(r.voxel_shift), float(r.eps), int(n_points), _ptr(alpha_range), _stream()), name)
    return jv


def field_vjp(drr, packed, source, target, raylen, U, w, alpha_range, n_points, grid, scratch=None):
    """The transpose of field_jvp: sum_n w_n dI_n / dU as the kernels' field (Bf, g0, g1, g2, 4), voxel units (b200drr_deform_bwd
    with only g_field wanted).  w (B, N) fp32; scratch: b200drr_deform_scratch_floats floats, allocated here when None."""
    vol, r = drr.density, drr.renderer
    fn, head, name, (src, tgt, lens), (H, W) = _launch_args("b200drr_deform_bwd", vol, packed, source, target, raylen, grid)
    B, N = tgt.shape[0], tgt.shape[1]
    if scratch is None:
        scratch = torch.empty(int(_lib.load().b200drr_deform_scratch_floats(B, N, H, W)), dtype=torch.float32, device=vol.device)
    g_field = torch.empty_like(U)
    with torch.cuda.device(vol.device):
        _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(lens), _ptr(U), U.shape[0], *U.shape[1:4], _ptr(w.contiguous()),
                      None, None, None, _ptr(g_field), None, _ptr(scratch), B, N, H, W, float(r.voxel_shift), float(r.eps),
                      int(n_points), _ptr(alpha_range), _stream()), name)
    return g_field


def deformed_jvp(drr, *args, field, tangent, parameterization=None, convention=None, degrees=False, calibration=None, n_points=500,
                 alphamin=None, alphamax=None, **kwargs):
    """See DRR.deformed_jvp."""
    B = check_supported(drr, args, parameterization, field, kwargs)
    _check_tangent(field, tangent)
    vol, r = drr.density, drr.renderer
    with torch.no_grad():
        source, marches = _marches(drr, args, B, parameterization, convention, degrees, calibration, alphamin, alphamax)
        U, T = voxel_field(drr, field), voxel_field(drr, tangent)
        packed = r._packed_volume(vol)
        imgs, jvs = [], []
        for tgt, lens, alpha_range, grid in marches:
            imgs.append(torch.empty(B, tgt.shape[1], dtype=torch.float32, device=vol.device))
            jvs.append(field_jvp(drr, packed, source, tgt, lens, U, T, alpha_range, n_points, grid, img=imgs[-1]))
        img, jv = (x[0] if len(x) == 1 else torch.cat(x, dim=-1) for x in (imgs, jvs))
        return drr.reshape_transform(img.view(B, 1, -1), batch_size=B), drr.reshape_transform(jv.view(B, 1, -1), batch_size=B)
