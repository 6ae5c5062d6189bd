"""Piecewise-rigid DRRs (`DRR.render_structures`; DESIGN.md 6f): every labelled structure of the CT under its own rigid motion.

A structure moved by X (world coordinates, x -> X x) and seen by camera P is the static structure seen by camera X^-1 P.  So channel
k of pose b is an ordinary pose-in render of the voxels labelled labels[k] with pose X_k^-1 P_b, and the optional background channel
renders every other voxel with P_b.  All B * S (pose, slot) pairs go through one kernel (include/b200drr.h:
b200drr_siddon_fwd_sens_structures) that walks each slot's label box only and skips the pixels outside the box's footprint; its
sensitivities have the layout of the pose-in training walk, so the backward is b200drr_siddon_bwd_sens_pose with batch B * S, and
torch carries the matrix gradients on to the camera pose, the calibration and the motions.
"""
from __future__ import annotations

import numbers

import torch
from torch.autograd.function import once_differentiable

from . import _lib, geometry
from .pose import RigidTransform, convert
from .renderers import _VOL16, Siddon, _check_vol16, _ptr, _stream, _vol_entry


def _label_tuple(labels):
    labels = labels.tolist() if torch.is_tensor(labels) else labels
    try:
        labels = tuple(labels)
    except TypeError:
        raise ValueError(f"labels must be a sequence of integer labels of drr.mask, got {labels!r}") from None
    if not labels:
        raise ValueError("labels must name at least one label of drr.mask")
    for lab in labels:
        if isinstance(lab, bool) or not isinstance(lab, numbers.Integral):
            raise ValueError(f"labels must be integers, got {lab!r}")
        if not 0 <= int(lab) <= 255:
            raise ValueError(f"labels must lie in 0..255 (the label volume is stored in 8 bits), got {int(lab)}")
    labels = tuple(int(lab) for lab in labels)
    if len(set(labels)) != len(labels):
        raise ValueError(f"labels must be distinct, got {labels}")
    return labels


def _batch_size(args, parameterization):
    """The number of camera poses the arguments describe, from shapes only (no conversion, no launch): the leading dimension of the
    pose matrix convert() builds -- the matrix's own for 'matrix' (a single (4, 4) matrix is one pose), the rotation's otherwise."""
    if parameterization is None:
        if len(args) != 1 or not isinstance(args[0], RigidTransform):
            raise ValueError("without a parameterization the camera pose is one RigidTransform")
        return len(args[0])
    if not args or not all(torch.is_tensor(a) for a in args):
        raise ValueError("the camera pose parameters must be tensors")
    if parameterization == "matrix":
        if args[0].dim() not in (2, 3) or tuple(args[0].shape[-2:]) != (4, 4):
            raise ValueError(f"a 'matrix' camera pose is (4, 4) or (B, 4, 4), got {tuple(args[0].shape)}")
        return args[0].shape[0] if args[0].dim() == 3 else 1
    if args[0].dim() != 2:
        raise ValueError(f"camera pose parameters must be (B, r), got {tuple(args[0].shape)}")
    return args[0].shape[0]


def _motion_matrices(motions, K, B):
    X = motions.matrix if isinstance(motions, RigidTransform) else motions
    if isinstance(motions, RigidTransform) and X.dim() == 5 and X.shape[0] == 1:
        X = X[0]   # RigidTransform adds a leading dimension to every matrix stack that is not 3-D: (B, K, 4, 4) arrives as 5-D
    if not torch.is_tensor(X) or X.dim() not in (3, 4) or tuple(X.shape[-3:]) != (K, 4, 4) or (X.dim() == 4 and X.shape[0] != B):
        shape = tuple(X.shape) if torch.is_tensor(X) else type(X).__name__
        raise ValueError(f"motions must be ({K}, 4, 4) or ({B}, {K}, 4, 4) for {K} labels and {B} camera poses, got {shape}")
    if X.dtype != torch.float32:
        raise ValueError(f"motions must be fp32, got {X.dtype}")
    return X


def _mask_state(drr):
    """(uint8 label copy, label boxes (256, 6) int32 or None on the CPU, set of present labels), cached per mask buffer."""
    mask = drr.mask
    key = (mask.data_ptr(), mask._version, mask.device, tuple(mask.shape))
    cached = getattr(drr, "_structures_cache", None)
    if cached is not None and cached["key"] == key:
        return cached
    with torch.no_grad():
        if mask.dim() != 3:
            raise ValueError(f"render_structures needs a 3-D label volume, got mask {tuple(mask.shape)}")
        m = mask.float()
        if bool(((m != m.round()) | (m < 0) | (m > 255)).any()):
            raise ValueError("render_structures needs integer labels 0..255 in drr.mask")
        labels_u8 = mask.to(torch.uint8).contiguous()
        boxes = None
        if labels_u8.is_cuda:
            boxes = torch.empty(256, 6, dtype=torch.int32, device=mask.device)
            with torch.cuda.device(mask.device):
                _lib.check(_lib.load().b200drr_label_boxes(_ptr(labels_u8), *labels_u8.shape, _ptr(boxes), _stream()),
                           "b200drr_label_boxes")
            present = (boxes[:, :3] < boxes[:, 3:]).all(dim=1).cpu()
        else:
            present = torch.bincount(labels_u8.flatten().long(), minlength=256) > 0
    cached = dict(key=key, labels=labels_u8, boxes=boxes, present={int(i) for i in present.nonzero().flatten().tolist()},
                  slots={})
    object.__setattr__(drr, "_structures_cache", cached)
    return cached


def _slots(state, labels, background, shape):
    """(slot_of_label (256,) int32, box (S, 6) int32) on the device for this label tuple, cached with the mask state."""
    key = (labels, background)
    if key not in state["slots"]:
        dev = state["boxes"].device
        slot = torch.full((256,), len(labels) if background else -1, dtype=torch.int32)
        slot[list(labels)] = torch.arange(len(labels), dtype=torch.int32)
        box = state["boxes"][torch.tensor(labels, device=dev, dtype=torch.long)]
        if background:
            whole = torch.tensor([[0, 0, 0, *shape]], dtype=torch.int32, device=dev)
            box = torch.cat([box, whole])
        state["slots"][key] = (slot.to(dev), box.contiguous())
    return state["slots"][key]


def check_supported(drr, args, parameterization, motions, labels, kwargs):
    """Refuse, before any launch, what the piecewise-rigid render does not cover: -> (labels, motion matrices, B)."""
    r = drr.renderer
    if not isinstance(r, Siddon):
        raise NotImplementedError(f"render_structures supports the Siddon renderer, not {type(r).__name__}: a trilinear sample "
                                  "straddles neighbouring structures")
    if r.mode != "nearest" or not isinstance(r.reducefn, str) or r.reducefn != "sum" or r.filter_intersections_outside_volume:
        raise NotImplementedError("render_structures supports Siddon with its default options (mode='nearest', reducefn='sum'), "
                                  "with or without stop_gradients_through_grid_sample")
    if kwargs.get("align_corners", False) or kwargs.get("mask") is not None or set(kwargs) - {"align_corners", "mask"}:
        raise NotImplementedError(f"render_structures takes no renderer options, got {sorted(kwargs)}")
    if drr.detector.n_subsample is not None:
        raise NotImplementedError("render_structures renders the full detector grid: p_subsample is not supported")
    if drr.patch_size is not None:
        raise NotImplementedError("render_structures renders the full detector grid in one pass: patch_size is not supported")
    if getattr(drr, "mask", None) is None:
        raise ValueError("render_structures needs a label volume: the subject has no mask")
    labels = _label_tuple(labels)
    B = _batch_size(args, parameterization)
    X = _motion_matrices(motions, len(labels), B)
    vol = drr.density
    if vol.dtype not in (torch.float32, *_VOL16) or vol.dim() != 3 or vol.numel() >= 2**31 - 1:
        raise NotImplementedError(f"render_structures needs a 3-D fp32 / fp16 / bf16 density below 2^31 voxels, got {vol.dtype} "
                                  f"{tuple(vol.shape)}")
    if vol.requires_grad:
        raise NotImplementedError("render_structures produces no volume gradient: the density must not require grad")
    cpu = _lib.B200DRRError(f"diffdrr_b200 renderers run on CUDA devices only (density is on {vol.device}); there is no CPU "
                            "fallback")
    if not vol.is_cuda and drr.mask.is_cuda:
        raise cpu
    if vol.is_cuda and (X.device != vol.device or drr.mask.device != vol.device):
        raise ValueError(f"motions and mask must be on the density's device {vol.device}, not {X.device} and {drr.mask.device}")
    # the last check that can refuse: on a CUDA mask the first call builds the label boxes (one launch, cached)
    absent = [lab for lab in labels if lab not in _mask_state(drr)["present"]]
    if absent:
        raise ValueError(f"labels {absent} do not occur in drr.mask")
    if not vol.is_cuda:   # a CPU mask is checked without a launch, so every argument error above is reported first
        raise cpu
    return labels, X, B


def _structures_walk(vol, labels, src, G, Wd, rows, cols, slot_of_label, box, S, voxel_shift, eps, want_sens):
    """The one launch site of b200drr_siddon_fwd_sens_structures: -> (out (B, S, H*W), sens (B, S, H*W, 8) or None for the
    image-only walk).  vol contiguous; src, G, Wd, rows, cols contiguous fp32."""
    BS, H, W = G.shape[0], rows.numel(), cols.numel()
    B = BS // S
    out = torch.empty(B, S, H * W, dtype=torch.float32, device=vol.device)
    sens = torch.empty(B, S, H * W, 8, dtype=torch.float32, device=vol.device) if want_sens else None
    fn, head, name = _vol_entry(_lib.load(), "b200drr_siddon_fwd_sens_structures", vol)
    with torch.cuda.device(vol.device):
        _lib.check(fn(*head, _ptr(labels), *vol.shape, _ptr(src), _ptr(G), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(slot_of_label),
                      _ptr(box), _ptr(out), _ptr(sens), B, S, H, W, voxel_shift, eps, _stream()), name)
    return out, sens


class _StructuresFunction(torch.autograd.Function):
    """(src, G, Wd) of the B * S (pose, slot) pairs -> out (B, S, H*W); gradients come back as the pose-in matrices'."""

    @staticmethod
    def forward(ctx, volume, labels, src, G, Wd, rows, cols, slot_of_label, box, S, voxel_shift, eps, stop_grad):
        vol = volume.contiguous()
        src, G, Wd = src.contiguous().float(), G.contiguous().float(), Wd.contiguous().float()
        rows, cols = rows.contiguous().float(), cols.contiguous().float()
        ctx.want = any(ctx.needs_input_grad[2:5])
        out, sens = _structures_walk(vol, labels, src, G, Wd, rows, cols, slot_of_label, box, S, voxel_shift, eps, ctx.want)
        if ctx.want:
            ctx.save_for_backward(sens, Wd, rows, cols)
        ctx.stop_grad = stop_grad
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        sens, Wd, rows, cols = ctx.saved_tensors
        BS, H, W = Wd.shape[0], rows.numel(), cols.numel()
        dev = sens.device
        gout = gout.reshape(BS, H * W).contiguous().float()
        g_src = torch.empty(BS, 3, dtype=torch.float32, device=dev)
        g_G = torch.empty(BS, 3, 4, dtype=torch.float32, device=dev)
        g_Wd = torch.empty(BS, 3, 4, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().b200drr_siddon_bwd_sens_pose(_ptr(sens), _ptr(gout), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(g_src),
                                                                _ptr(g_G), _ptr(g_Wd), BS, H, W, int(ctx.stop_grad), _stream()),
                       "b200drr_siddon_bwd_sens_pose")
        return None, None, g_src, g_G, g_Wd, None, None, None, None, None, None, None, None


def _rigid_inverse(X):
    """[R t; 0 1]^-1 = [R^T -R^T t; 0 1], differentiable and without the host check of RigidTransform.inverse."""
    Rt = X[..., :3, :3].mT
    t = -(Rt @ X[..., :3, 3:])
    bottom = torch.zeros_like(X[..., 3:, :])
    bottom[..., 3] = 1.0
    return torch.cat([torch.cat([Rt, t], dim=-1), bottom], dim=-2)


def _camera_pose(args, B, parameterization, convention, degrees):
    """The camera pose matrices (B, 4, 4), built as DRR.forward builds them."""
    if (parameterization == "euler_angles" and len(args) == 2 and geometry.euler_convention_ok(convention)
            and all(a.is_cuda and a.dtype == torch.float32 and a.dim() == 2 and a.shape[-1] == 3 for a in args)
            and args[0].shape == args[1].shape):
        P = geometry.euler_pose(args[0], args[1], convention, degrees)   # as DRR.forward builds it
    elif parameterization is None:
        P = args[0].matrix
    else:
        P = convert(*args, parameterization=parameterization, convention=convention, degrees=degrees).matrix
    if P.shape[0] != B:
        raise ValueError(f"the camera pose arguments describe {P.shape[0]} poses where their leading dimension says {B}")
    return P


def _slot_inputs(drr, P, X, K, background, calibration):
    """The pose-in inputs (src, G, Wd, rows, cols) of the B * S (pose, slot) pairs: slot k < K sees its structure through
    X_k^-1 P, the background slot through P."""
    B = P.shape[0]
    S = K + int(background)
    Ps = _rigid_inverse(X) @ P[:, None]                       # (B, K, 4, 4): structure k seen through X_k^-1 P
    if background:
        Ps = torch.cat([Ps, P[:, None]], dim=1)
    Ps = Ps.reshape(B * S, 4, 4)
    if calibration is not None and len(calibration) == B and B > 1:
        calibration = RigidTransform(calibration.matrix.repeat_interleave(S, dim=0))
    return drr._pose_in_inputs(RigidTransform(Ps), calibration)


def render_structures(drr, *args, motions, labels, parameterization=None, convention=None, degrees=False, calibration=None,
                      background=True, **kwargs):
    """See DRR.render_structures."""
    labels, X, B = check_supported(drr, args, parameterization, motions, labels, kwargs)
    vol = drr.density
    P = _camera_pose(args, B, parameterization, convention, degrees)
    K = len(labels)
    S = K + int(background)
    src, G, Wd, rows, cols = _slot_inputs(drr, P, X, K, background, calibration)
    if vol.dtype in _VOL16:
        _check_vol16(vol, src, G)
    state = _mask_state(drr)
    slot_of_label, box = _slots(state, labels, bool(background), tuple(vol.shape))
    r = drr.renderer
    out = _StructuresFunction.apply(vol, state["labels"], src, G, Wd, rows, cols, slot_of_label, box, S, float(r.voxel_shift),
                                    float(r.eps), bool(r.stop_gradients_through_grid_sample))
    return drr.reshape_transform(out, batch_size=B)


def structure_pivots(drr, labels):
    """(K, 3) world positions of the centres of the labels' boxes, float64, from the cached label boxes (no host sync).  Voxel i
    spans index coordinates [i - 1/2, i + 1/2], so a box [lo, hi) is centred at (lo + hi - 1) / 2; the affine maps it to world."""
    state = _mask_state(drr)
    slot_of_label, box = _slots(state, _label_tuple(labels), False, tuple(drr.density.shape))
    centre = (box[:, :3] + box[:, 3:]).double() * 0.5 - 0.5
    A = drr._affine.reshape(4, 4).double()
    return centre @ A[:3, :3].mT + A[:3, 3]


def _translation(c):
    """(..., 3) -> (..., 4, 4) translations by c."""
    T = torch.eye(4, dtype=c.dtype, device=c.device).expand(*c.shape[:-1], 4, 4).clone()
    T[..., :3, 3] = c
    return T


def twist_matrix(xi):
    """(..., 6) twists (omega, v) -> (..., 4, 4) matrices [[omega^, v], [0, 0]] (se(3)); their matrix exponential is the rigid
    motion exp(xi^)."""
    w, v = xi[..., :3], xi[..., 3:]
    z = torch.zeros_like(w[..., 0])
    rows = [torch.stack([z, -w[..., 2], w[..., 1], v[..., 0]], -1), torch.stack([w[..., 2], z, -w[..., 0], v[..., 1]], -1),
            torch.stack([-w[..., 1], w[..., 0], z, v[..., 2]], -1), torch.stack([z, z, z, z], -1)]
    return torch.stack(rows, dim=-2)


def se3_exp(xi):
    """(..., 6) twists (omega, v) -> exp(xi^) (..., 4, 4), the matrix exponential of twist_matrix(xi) in closed form:
    [[R, V v], [0, 1]] with R = I + a W + b W^2, V = I + b W + c W^2, W = omega^, theta = |omega|, a = sin(theta) / theta,
    b = (1 - cos(theta)) / theta^2, c = (theta - sin(theta)) / theta^3 (their Taylor series near 0).  No host sync, unlike
    torch.linalg.matrix_exp on CUDA, which reads the norm on the host to choose its degree."""
    W = twist_matrix(torch.cat([xi[..., :3], torch.zeros_like(xi[..., 3:])], dim=-1))[..., :3, :3]
    th2 = (xi[..., :3] ** 2).sum(-1)
    th = th2.sqrt()
    small = th < 1e-4
    ths = torch.where(small, torch.ones_like(th), th)
    a = torch.where(small, 1 - th2 / 6, ths.sin() / ths)
    b = torch.where(small, 0.5 - th2 / 24, (1 - ths.cos()) / ths**2)
    c = torch.where(small, 1.0 / 6 - th2 / 120, (ths - ths.sin()) / ths**3)
    eye = torch.eye(3, dtype=xi.dtype, device=xi.device)
    W2 = W @ W
    R = eye + a[..., None, None] * W + b[..., None, None] * W2
    V = eye + b[..., None, None] * W + c[..., None, None] * W2
    top = torch.cat([R, V @ xi[..., 3:, None]], dim=-1)
    bottom = torch.zeros_like(top[..., :1, :])
    bottom[..., 0, 3] = 1.0
    return torch.cat([top, bottom], dim=-2)


def apply_increments(X, xi, pivots):
    """X_k <- T(c_k) exp(xi_k^) T(-c_k) X_k: the left increment of every motion about its structure's pivot, in world coordinates.
    X (..., K, 4, 4) fp32; xi (..., K, 6) float64 (omega, v); pivots (K, 3) float64.  exp is the rigid motion se3_exp (the
    exponential of the 4 x 4 twist matrix; pose.se3_exp_map uses the transposed, right-multiplying convention)."""
    return (_translation(pivots) @ se3_exp(xi) @ _translation(-pivots) @ X.double()).to(X.dtype)


def motion_tangents(drr, P, X, pivots, K, background, calibration):
    """d(src, G, Wd)/d xi of every (pose, slot) in float64, xi_k = (omega, v) the left increment of motion k about pivot c_k:
    -> dsrc (B*S, 6, 3), dG, dWd (B*S, 6, 3, 4); the background slot's are zero.

    Slot k sees X_k(xi)^-1 P with X_k(xi) = T(c) exp(xi^) T(-c) X_k, so X_k(xi)^-1 P = X_k^-1 T(c) exp(-xi^) T(-c) P.  Only the
    derivative at xi = 0 is wanted, and exp(-xi^) = I - xi^ to first order, so the map below is that first-order form; one
    forward-mode pass over 6 stacked copies (copy i carries the unit tangent of parameter i) gives all six columns."""
    from .drr import pose_in_matrices

    B = P.shape[0]
    dev = P.device
    det = drr.detector
    Xi = _rigid_inverse(X.detach().double()).expand(B, K, 4, 4)
    left = Xi @ _translation(pivots)                                    # (B, K, 4, 4)
    right = _translation(-pivots) @ P.detach().double()[:, None]        # (B, K, 4, 4)
    calib = (det._calibration if calibration is None else calibration.matrix).detach().double().reshape(-1, 4, 4)
    calib = calib.reshape(1, -1, 1, 4, 4).expand(6, B, K, 4, 4).reshape(6 * B * K, 4, 4)
    consts = (det._reorient.detach().double(), drr._affine_inverse.detach().double())
    eye = torch.eye(6, dtype=torch.float64, device=dev)

    def f(xi):
        Ps = left @ (torch.eye(4, dtype=torch.float64, device=dev) - twist_matrix(xi)) @ right     # (6, B, K, 4, 4)
        return pose_in_matrices(Ps.reshape(6 * B * K, 4, 4), consts[0], calib, consts[1])

    zero = torch.zeros(6, B, K, 6, dtype=torch.float64, device=dev)
    _, (dsrc, dG, dWd) = torch.func.jvp(f, (zero,), (eye[:, None, None, :].expand(6, B, K, 6).clone(),))
    S = K + int(background)

    def slots(d):   # (6, B, K, ...) -> (B*S, 6, ...), zeros for the background slot
        d = d.reshape(6, B, K, *d.shape[1:]).movedim(0, 2)
        if background:
            d = torch.cat([d, torch.zeros_like(d[:, :1])], dim=1)
        return d.reshape(B * S, 6, *d.shape[3:])

    return slots(dsrc), slots(dG), slots(dWd)


def structures_jacobian(drr, *args, motions, labels, parameterization=None, convention=None, degrees=False, calibration=None,
                        background=True, stop_grad=None, return_footprints=False, **kwargs):
    """See DRR.structures_jacobian.  stop_grad: drop Siddon's ray-length term (None = the renderer's
    stop_gradients_through_grid_sample).  return_footprints adds the (B, S, 4) int32 pixel rectangles {w0, w1, h0, h1} the render
    culls each (pose, slot) to (b200drr_structure_footprints): J[:, k] is zero outside rectangle k."""
    labels, X, B = check_supported(drr, args, parameterization, motions, labels, kwargs)
    vol = drr.density
    r = drr.renderer
    K = len(labels)
    S = K + int(background)
    with torch.no_grad():
        P = _camera_pose(args, B, parameterization, convention, degrees)
        src, G, Wd, rows, cols = _slot_inputs(drr, P, X, K, background, calibration)
        if vol.dtype in _VOL16:
            _check_vol16(vol, src, G)
        state = _mask_state(drr)
        slot_of_label, box = _slots(state, labels, bool(background), tuple(vol.shape))
        src, G, Wd = src.contiguous().float(), G.contiguous().float(), Wd.contiguous().float()
        rows, cols = rows.contiguous().float(), cols.contiguous().float()
        shift = float(r.voxel_shift)
        out, sens = _structures_walk(vol.contiguous(), state["labels"], src, G, Wd, rows, cols, slot_of_label, box, S, shift,
                                     float(r.eps), True)
        dsrc, dG, dWd = (t.float().contiguous() for t in
                         motion_tangents(drr, P, X, structure_pivots(drr, labels), K, background, calibration))
        H, W = rows.numel(), cols.numel()
        J = torch.empty(B * S, H * W, 6, dtype=torch.float32, device=vol.device)
        stop_grad = int(bool(r.stop_gradients_through_grid_sample if stop_grad is None else stop_grad))
        lib = _lib.load()
        with torch.cuda.device(vol.device):
            _lib.check(lib.b200drr_siddon_jac_sens_pose(_ptr(sens), _ptr(dsrc), _ptr(dG), _ptr(dWd), _ptr(Wd), _ptr(rows), _ptr(cols),
                                                        _ptr(J), B * S, H, W, 6, stop_grad, _stream()),
                       "b200drr_siddon_jac_sens_pose")
            if return_footprints:
                rects = torch.empty(B, S, 4, dtype=torch.int32, device=vol.device)
                _lib.check(lib.b200drr_structure_footprints(_ptr(src), _ptr(G), _ptr(rows), _ptr(cols), _ptr(box), _ptr(rects), B,
                                                            S, H, W, shift, _stream()), "b200drr_structure_footprints")
    img = drr.reshape_transform(out, batch_size=B)
    J = J.view(B, S, *img.shape[2:], 6)[:, :K]
    return (img, J, rects) if return_footprints else (img, J)
