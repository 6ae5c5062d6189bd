"""`Registration`: pose parameters as nn.Parameters on top of a DRR module (reference diffdrr/registration.py:14-50).

`PoseRegressor` (a timm CNN) is not part of the projector path and is not provided.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .pose import convert


class Registration(nn.Module):
    """Automatic 2D-to-3D registration by differentiable rendering: holds the pose being optimised."""

    def __init__(self, drr, rotation: torch.Tensor, translation: torch.Tensor, parameterization: str,
                 convention: str | None = None):
        super().__init__()
        self.drr = drr
        self._rotation = nn.Parameter(rotation)
        self._translation = nn.Parameter(translation)
        self.parameterization = parameterization
        self.convention = convention

    def forward(self, **kwargs):
        # same pose as `self.drr(self.pose)` (registration.py:34-35); handing DRR.forward the parameters lets it run the
        # parameter -> pose-matrix algebra as one kernel on its fused path
        return self.drr(self._rotation, self._translation, parameterization=self.parameterization,
                        convention=self.convention, **kwargs)

    @property
    def pose(self):
        return convert(self._rotation, self._translation, parameterization=self.parameterization,
                       convention=self.convention)

    @property
    def rotation(self):
        return self._rotation

    @property
    def translation(self):
        return self._translation


def _damped_solve(A, g, damping):
    """The Levenberg-Marquardt step delta of (A + lambda diag A) delta = -g, solved per system in float64: A (S, P, P), g (S, P)
    and lambda = damping (S,) -> delta (S, P).  No host sync."""
    D = torch.diag_embed(torch.diagonal(A, dim1=-2, dim2=-1).clamp_min(1e-12))
    return torch.linalg.solve_ex(A + damping[:, None, None] * D, -g.unsqueeze(-1))[0].squeeze(-1)


def _next_damping(accept, damping):
    """The damping after a step: / 10 where the trial was accepted, x 10 where it was rejected, within [1e-12, 1e12]."""
    return torch.where(accept, damping / 10.0, damping * 10.0).clamp(1e-12, 1e12)


def _global_ncc(name, loss, eps):
    """The loss of the Levenberg-Marquardt solvers that model the global NCC only: None -> NormalizedCrossCorrelation2d(eps=eps);
    anything but a NormalizedCrossCorrelation2d without patch_size raises TypeError."""
    from .metrics import NormalizedCrossCorrelation2d

    if loss is None:
        return NormalizedCrossCorrelation2d(eps=eps)
    if type(loss) is not NormalizedCrossCorrelation2d or loss.patch_size is not None:
        raise TypeError(f"{name} models the global NCC only: NormalizedCrossCorrelation2d without patch_size (or loss=None), not "
                        f"{type(loss).__name__}{'' if getattr(loss, 'patch_size', None) is None else f'(patch_size={loss.patch_size})'}"
                        f"; patch-wise, multiscale and gradient NCC have no Gauss-Newton model here (use a first-order optimizer)")
    return loss


def _check_target(name, drr, target, args, parameterization, check_supported, full_detector=True):
    """The refusals of a warped-render Levenberg-Marquardt solver `name` for its target, in order: a one-channel (B, 1, H, W)
    image, a full detector (where `full_detector`), the detector's H x W, a batch of 1 or the poses' B, then the render's own
    refusals (`check_supported()`), then a CUDA fp32 tensor -> B."""
    from .structures import _batch_size

    if not torch.is_tensor(target) or target.dim() != 4 or target.shape[1] != 1:
        raise ValueError(f"{name} takes a one-channel target image (B, 1, H, W), got "
                         f"{tuple(target.shape) if torch.is_tensor(target) else type(target).__name__}")
    det = drr.detector
    if full_detector and (det.n_subsample is not None or drr.patch_size is not None):
        raise NotImplementedError(f"{name} covers the full detector only, not p_subsample or patch_size")
    if tuple(target.shape[-2:]) != (det.height, det.width):
        raise ValueError(f"the target {tuple(target.shape)} does not match the {det.height} x {det.width} detector")
    B = _batch_size(args, parameterization)
    if target.shape[0] not in (1, B):
        raise ValueError(f"the target's batch ({target.shape[0]}) must be 1 or the number of poses ({B})")
    check_supported()
    if not (target.is_cuda and target.dtype == torch.float32):
        raise ValueError(f"{name} runs on the GPU: the target must be a CUDA fp32 tensor")
    return B


def ncc_normal_equations(x, t, J, strides, patch_size, eps, weight, A, g):
    """A += weight * sum Jz^T Jz, g += weight * sum Jz^T r over every window of every channel of the global (patch_size None) or
    patch-wise NCC between x and t ((B, C, H, W) fp32 CUDA, contiguous), through b200drr_ncc_normal (csrc/ncc_normal.cu).
    J: fp32 CUDA tensor whose element (pose b, channel c, parameter k, pixel n) sits at the element strides `strides`
    (b, c, k, n) from its data pointer; A (B, P, P) and g (B, P) float64.  r = z(x) - z(t) per window, Jz its Jacobian
    (DESIGN.md 6e)."""
    from . import _lib
    B, C, H, W = x.shape
    P = g.shape[1]
    p = 0 if patch_size is None else int(patch_size)
    lib = _lib.load()
    ws = torch.empty(max(int(lib.b200drr_ncc_normal_workspace_bytes(B, C, H, W, p, P)) // 8, 1), dtype=torch.float64,
                     device=x.device)
    _lib.check(lib.b200drr_ncc_normal(x.data_ptr(), t.data_ptr(), J.data_ptr(), *(int(s) for s in strides), B, C, H, W, p, P,
                                      float(eps), float(weight), ws.data_ptr(), A.data_ptr(), g.data_ptr(),
                                      torch.cuda.current_stream(x.device).cuda_stream), "b200drr_ncc_normal")


class LevenbergMarquardt:
    """Levenberg-Marquardt steps of a `Registration` towards `target` on an NCC loss, built on DRR.jacobian (DESIGN.md 6e).

    `loss` is a NormalizedCrossCorrelation2d (global or any patch_size), a MultiscaleNormalizedCrossCorrelation2d or a
    GradientNormalizedCrossCorrelation2d (global or patch-wise, any sigma); None is the global NCC with `eps`.  Mutual
    information is not a sum of squares and other losses have no such model: they raise here.  The Gauss-Newton model of scale s
    is the z-normalised residual r_w = z(img_w) - z(target_w) of every window w of every channel, z(x) = (x - mean x) /
    sqrt(var x + eps) (population variance, as in metrics.py), for which w_s (1 - score_s) ~= w_s / (2 N_s) sum_w |r_w|^2 with
    N_s = C H' W' p^2 (C H W for the global NCC); the gradient NCC models the blurred Sobel gradients, which are linear in the
    image, so its J is the loss's own Sobel of the Jacobian planes.  Each step takes one Jacobian, accumulates the normal
    equations of every scale on the GPU (b200drr_ncc_normal), solves (A + lambda diag A) delta = -g per pose in float64, renders
    one trial image, and keeps the trial per pose only if its true loss (the module's own forward) is lower (lambda / 10 on
    accept, x 10 on reject).  The pose Parameters are updated in place and keep their identity, so an optimizer can take over.
    The poses are solved independently (for Trilinear with B > 1 the coupling through the batch-global sampling range is left
    out of the model; the true loss still decides).  No host sync."""

    def __init__(self, reg: Registration, target: torch.Tensor, loss=None, damping: float = 1e-3, eps: float = 1e-5):
        from .metrics import (GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d,
                              NormalizedCrossCorrelation2d)

        self.sobel = None
        if loss is None:
            loss = NormalizedCrossCorrelation2d(eps=eps)
            scales = [(None, 1.0, eps)]
        elif type(loss) is NormalizedCrossCorrelation2d:
            scales = [(loss.patch_size, 1.0, loss.eps)]
        elif type(loss) is GradientNormalizedCrossCorrelation2d:
            scales = [(loss.patch_size, 1.0, loss.eps)]
            self.sobel = loss.sobel
        elif type(loss) is MultiscaleNormalizedCrossCorrelation2d:
            scales = [(ncc.patch_size, float(w), ncc.eps) for ncc, w in zip(loss.nccs, loss.patch_weights)]
        else:
            raise TypeError(f"LevenbergMarquardt needs a loss that is a sum of squares: NormalizedCrossCorrelation2d, "
                            f"MultiscaleNormalizedCrossCorrelation2d or GradientNormalizedCrossCorrelation2d, not "
                            f"{type(loss).__name__} (mutual information has no Gauss-Newton model: use a first-order optimizer)")
        if not torch.is_tensor(target) or target.dim() != 4 or target.shape[1] != 1:
            raise ValueError(f"LevenbergMarquardt takes a one-channel target image (B, 1, H, W) like the DRR's, got "
                             f"{tuple(target.shape) if torch.is_tensor(target) else type(target).__name__}")
        B = reg._rotation.shape[0]
        Bt, _, H, W = target.shape
        if Bt not in (1, B):
            raise ValueError(f"the target's batch ({Bt}) must be 1 or the number of poses ({B})")
        for p, _, _ in scales:
            if p is not None and not (isinstance(p, int) and 1 <= p <= min(H, W)):
                raise ValueError(f"patch_size {p} outside 1 .. min(H, W) = {min(H, W)} of the {H} x {W} images")
        if self.sobel is not None and self.sobel.kernel_size // 2 >= min(H, W):
            raise ValueError(f"Sobel(sigma={self.sobel.sigma}): the blur's reflect padding of {self.sobel.kernel_size // 2} "
                             f"pixels needs images larger than that, got {H} x {W}")
        if not (target.is_cuda and target.dtype == torch.float32):
            raise ValueError("LevenbergMarquardt's normal equations run on the GPU: the target must be a CUDA fp32 tensor")
        self.reg, self.eps, self.loss, self.scales = reg, eps, loss, scales
        # the losses compare images of one shape: the target repeated for every pose
        self.target = target.detach().expand(B, *target.shape[1:]).contiguous()
        self.damping = torch.full((B,), float(damping), dtype=torch.float64, device=reg._rotation.device)
        with torch.no_grad():
            self._t = self.target if self.sobel is None else self.sobel(self.target)

    def _loss(self, img):
        return 1.0 - self.loss(self.target, img)

    def normal_equations(self, img, J):
        """(A (B, P, P), g (B, P)) float64 of the Gauss-Newton model at the image `img` (B, 1, H, W) with Jacobian J
        (B, 1, H, W, P): sum over the scales of w_s / N_s times the scale's sum_w Jz^T Jz and sum_w Jz^T r."""
        B, H, W, P = img.shape[0], img.shape[-2], img.shape[-1], J.shape[-1]
        if tuple(img.shape[1:]) != (1, H, W) or (H, W) != tuple(self._t.shape[-2:]):
            raise ValueError(f"the rendered image {tuple(img.shape)} does not match the target {tuple(self.target.shape)}")
        if self.sobel is None:
            x, Jv, strides = img.contiguous(), J.contiguous(), (H * W * P, 0, 1, P)
        else:
            # blur and Sobel are linear: the Jacobian of the gradient images is the Sobel of the Jacobian planes
            x = self.sobel(img)
            Jv = self.sobel(J.reshape(B, H * W, P).transpose(1, 2).reshape(B * P, 1, H, W))
            strides = (2 * P * H * W, H * W, 2 * H * W, 1)
        C = x.shape[1]
        A = torch.zeros(B, P, P, dtype=torch.float64, device=img.device)
        g = torch.zeros(B, P, dtype=torch.float64, device=img.device)
        for p, w, eps in self.scales:
            N = C * H * W if p is None else C * (H - p + 1) * (W - p + 1) * p * p
            ncc_normal_equations(x, self._t, Jv, strides, p, eps, w / N, A, g)
        return A, g

    def step(self) -> torch.Tensor:
        """One damped Gauss-Newton step; -> the per-pose 1 - loss(target, image) after it."""
        reg = self.reg
        rot, xyz = reg._rotation, reg._translation
        kw = dict(parameterization=reg.parameterization, convention=reg.convention)
        from .jacobian import drr_jacobian

        with torch.no_grad():
            # the model is of the image itself: the full derivative even if the renderer stops gradients for training
            img, J = drr_jacobian(reg.drr, rot, xyz, stop_grad=False, **kw)
            nr = rot.shape[1]
            A, g = self.normal_equations(img, J)
            delta = _damped_solve(A, g, self.damping).to(rot.dtype)
            rot_t, xyz_t = rot + delta[:, :nr], xyz + delta[:, nr:]
            loss, trial = self._loss(img), self._loss(reg.drr(rot_t, xyz_t, **kw))
            accept = trial < loss  # a NaN trial is rejected
            rot.copy_(torch.where(accept[:, None], rot_t, rot))
            xyz.copy_(torch.where(accept[:, None], xyz_t, xyz))
            self.damping = _next_damping(accept, self.damping)
            return torch.where(accept, trial, loss)


def ncc_normal_structures_equations(x, t, J, rects, eps, weight, A, g):
    """A += weight * sum_q Jz_q Jz_q^T, g += weight * sum_q Jz_q r_q of the global NCC between the composite x (B, H, W) and the
    target t (1 or B, H, W) (fp32 CUDA, contiguous), for the motions of K structures, through b200drr_ncc_normal_structures
    (csrc/ncc_normal_structures.cu).  J: DRR.structures_jacobian's (B, K, H, W, 6) (or (B, K, H*W, 6)) view; rects (B, S, 4)
    int32 its footprints; A (B, 6K, 6K) and g (B, 6K) float64 (DESIGN.md 6g)."""
    from . import _lib
    B, H, W = x.shape
    K, S = J.shape[1], rects.shape[1]
    sn = J.stride(-2)
    if (J.shape[0] != B or J.shape[-1] != 6 or J[0, 0, ..., 0].numel() != H * W or (J.dim() == 5 and J.stride(2) != W * sn)
            or tuple(rects.shape) != (B, S, 4) or S < K or tuple(A.shape) != (B, 6 * K, 6 * K) or tuple(g.shape) != (B, 6 * K)):
        raise ValueError(f"ncc_normal_structures_equations: J {tuple(J.shape)} must be (B, K, H, W, 6) or (B, K, H*W, 6) with "
                         f"evenly strided pixels, rects (B, S >= K, 4), A (B, 6K, 6K) and g (B, 6K) for x {tuple(x.shape)}; got "
                         f"rects {tuple(rects.shape)}, A {tuple(A.shape)}, g {tuple(g.shape)}")
    lib = _lib.load()
    ws = torch.empty(max(int(lib.b200drr_ncc_normal_structures_workspace_bytes(B, K, H, W)) // 8, 1), dtype=torch.float64,
                     device=x.device)
    _lib.check(lib.b200drr_ncc_normal_structures(x.data_ptr(), t.data_ptr(), t.shape[0], J.data_ptr(), J.stride(0), J.stride(1), sn,
                                                 J.stride(-1), rects.data_ptr(), B, K, S, H, W, float(eps), float(weight),
                                                 ws.data_ptr(), A.data_ptr(), g.data_ptr(),
                                                 torch.cuda.current_stream(x.device).cuda_stream), "b200drr_ncc_normal_structures")


class _MotionLevenbergMarquardt:
    """The Levenberg-Marquardt step of the rigid-motion solvers (StructuresLevenbergMarquardt, PolyrigidLevenbergMarquardt) on the
    global NCC of the composite image, with the camera pose fixed.

    The unknowns are the motions: `motions` (K, 4, 4), shared by the B views, or (B, K, 4, 4), one set per pose; a tensor or a
    Parameter, fp32 on the density's device, updated in place by step().  Each step takes one Jacobian of the image (_jacobian: the
    image, the per-pixel columns of every motion and their footprints), forms the Gauss-Newton system of the z-normalised residual
    block by block over the footprints (b200drr_ncc_normal_structures), solves (A + lambda diag A) delta = -g in float64, and
    renders one trial image (_render).  delta_k = (omega, v) moves structure k as
        X_k <- T(c_k) exp(delta_k^) T(-c_k) X_k,
    a left increment about the pivot c_k (exp is the matrix exponential of the twist, not pose.se3_exp_map's transposed
    convention).  The trial is kept if its true loss is lower (lambda / 10 on accept, x 10 on reject).  Shared motions: one
    system, the mean over the views of the per-view systems, modelling the mean of 1 - NCC, and one decision per step on that
    mean.  Per-pose motions: B independent systems and decisions.  No host sync.

    Only the global NCC is modelled: `loss` None (NormalizedCrossCorrelation2d(eps=eps)) or a NormalizedCrossCorrelation2d
    without patch_size; anything else raises TypeError here."""

    def __init__(self, drr, rot, xyz, motions, target, parameterization, loss, damping, eps, check_supported, full_detector):
        name = type(self).__name__
        loss = _global_ncc(name, loss, eps)
        if not torch.is_tensor(motions) or motions.dim() not in (3, 4):
            raise ValueError(f"motions must be a (K, 4, 4) or (B, K, 4, 4) tensor updated in place, got "
                             f"{tuple(motions.shape) if torch.is_tensor(motions) else type(motions).__name__}")
        B = _check_target(name, drr, target, (rot, xyz), parameterization, check_supported, full_detector)
        det = drr.detector
        self.drr, self.rot, self.xyz, self.motions = drr, rot.detach(), xyz.detach(), motions
        self.loss, self.eps = loss, float(loss.eps)
        self.shared = motions.dim() == 3
        self.target = target.detach().expand(B, 1, det.height, det.width).contiguous()
        self._t = self.target[:, 0]
        self.damping = torch.full((1 if self.shared else B,), float(damping), dtype=torch.float64, device=motions.device)

    def _composite(self, img):
        """The image the loss compares with the target, (B, 1, H, W)."""
        return img

    def _loss(self, img):
        """(B,) 1 - NCC of the composite of each view."""
        return 1.0 - self.loss(self.target, self._composite(img))

    def normal_equations(self, img, J, rects):
        """(A (B, 6K, 6K), g (B, 6K)) float64 of each view's Gauss-Newton model of 1 - NCC (weight 1 / (H W)) at the image `img`
        with Jacobian J (B, K, H, W, 6) and footprints rects."""
        B, K, H, W = img.shape[0], J.shape[1], self._t.shape[-2], self._t.shape[-1]
        x = self._composite(img).reshape(B, H, W).contiguous()
        A = torch.zeros(B, 6 * K, 6 * K, dtype=torch.float64, device=img.device)
        g = torch.zeros(B, 6 * K, dtype=torch.float64, device=img.device)
        ncc_normal_structures_equations(x, self._t, J, rects, self.eps, 1.0 / (H * W), A, g)
        return A, g

    def step(self) -> torch.Tensor:
        """One damped Gauss-Newton step; -> the loss after it: the mean over the views of 1 - NCC (a 0-d tensor) for shared
        motions, the per-pose (B,) losses otherwise."""
        from .structures import apply_increments

        X = self.motions
        with torch.no_grad():
            img, J, rects = self._jacobian(X)
            A, g = self.normal_equations(img, J, rects)
            loss = self._loss(img)
            if self.shared:
                A, g = A.mean(0, keepdim=True), g.mean(0, keepdim=True)
            delta = _damped_solve(A, g, self.damping)
            X_t = apply_increments(X.detach(), delta.reshape(*X.shape[:-2], 6), self.pivots)   # (..., K, 6): (omega, v) per k
            trial = self._loss(self._render(X_t))
            if self.shared:
                loss, trial = loss.mean(), trial.mean()
            accept = trial < loss  # a NaN trial is rejected
            X.copy_(torch.where(accept.reshape(-1, *[1] * (X.dim() - 1)), X_t, X))
            self.damping = _next_damping(accept, self.damping)
            return torch.where(accept, trial, loss)


class StructuresLevenbergMarquardt(_MotionLevenbergMarquardt):
    """Levenberg-Marquardt registration of the K structures of a piecewise-rigid DRR (DRR.render_structures) towards `target`
    on the global NCC of the composite image (the sum of the channels), with the camera pose fixed (DESIGN.md 6g).

    The step is _MotionLevenbergMarquardt's.  The Jacobian is DRR.structures_jacobian's (the full derivative of the image,
    whatever the renderer's stop_gradients_through_grid_sample), the trial render DRR.render_structures', and the pivot c_k of
    structure k the world centre of label k's box (structures.structure_pivots)."""

    def __init__(self, drr, rot: torch.Tensor, xyz: torch.Tensor, motions: torch.Tensor, labels, target: torch.Tensor,
                 parameterization: str = "euler_angles", convention: str | None = None, degrees: bool = False, calibration=None,
                 background: bool = True, loss=None, damping: float = 1e-3, eps: float = 1e-5):
        from .structures import _label_tuple, check_supported, structure_pivots

        def check():
            self.labels = check_supported(drr, (rot, xyz), parameterization, motions, _label_tuple(labels), {})[0]

        super().__init__(drr, rot, xyz, motions, target, parameterization, loss, damping, eps, check, full_detector=False)
        self.kw = dict(parameterization=parameterization, convention=convention, degrees=degrees, calibration=calibration,
                       background=background)
        self.pivots = structure_pivots(drr, self.labels)

    def _composite(self, img):
        return img.sum(1, keepdim=True)

    def _jacobian(self, X):
        from .structures import structures_jacobian
        return structures_jacobian(self.drr, self.rot, self.xyz, motions=X, labels=self.labels, stop_grad=False,
                                   return_footprints=True, **self.kw)

    def _render(self, X):
        from .structures import render_structures
        return render_structures(self.drr, self.rot, self.xyz, motions=X, labels=self.labels, **self.kw)


class PolyrigidLevenbergMarquardt(_MotionLevenbergMarquardt):
    """Levenberg-Marquardt registration of the K motions of a blended-rigid DRR (DRR.render_polyrigid) towards `target` on the
    global NCC of the image, with the camera pose fixed (DESIGN.md 6j).

    The step is _MotionLevenbergMarquardt's.  `weights` is render_polyrigid's lattice.  The Jacobian is DRR.polyrigid_jacobian's
    (one march: the image, the per-pixel columns of every motion and their footprints), the trial render render_polyrigid's, and
    the pivot c_k the weight-weighted centroid of channel k's lattice (polyrigid.polyrigid_pivots).  The sampling range is
    Trilinear's batch-global one unless alphamin / alphamax fix it; its dependence on the motions is nil (the rays do not move),
    so the model is the image's full derivative.  Full detectors only.  No host sync once the lattice has been seen.

    blend / steps are render_polyrigid's: with blend="log_euclidean" the Jacobian is that of the exponential's render (DESIGN.md
    6p: the 6K motion tangents through the `steps` squarings and one march) and the trial render render_polyrigid(blend=
    "log_euclidean", steps=steps).  A blend other than the two or a bad steps raises ValueError here."""

    def __init__(self, drr, rot: torch.Tensor, xyz: torch.Tensor, motions: torch.Tensor, weights: torch.Tensor, target: torch.Tensor,
                 parameterization: str = "euler_angles", convention: str | None = None, degrees: bool = False, calibration=None,
                 n_points: int = 500, alphamin=None, alphamax=None, loss=None, damping: float = 1e-3, eps: float = 1e-5,
                 blend: str = "linear", steps: int = 10):
        from .polyrigid import check_supported, polyrigid_pivots

        if blend not in ("linear", "log_euclidean"):
            raise ValueError(f"blend must be 'linear' or 'log_euclidean', got {blend!r}")
        if blend == "log_euclidean":
            from .svf import check_steps

            check_steps(steps)
        super().__init__(drr, rot, xyz, motions, target, parameterization, loss, damping, eps,
                         lambda: check_supported(drr, (rot, xyz), parameterization, motions, weights, {}), full_detector=True)
        self.weights = weights
        self.kw = dict(parameterization=parameterization, convention=convention, degrees=degrees, calibration=calibration,
                       n_points=n_points, alphamin=alphamin, alphamax=alphamax, blend=blend, steps=steps)
        self.pivots = polyrigid_pivots(drr, weights)

    def _jacobian(self, X):
        from .polyrigid import polyrigid_jacobian
        return polyrigid_jacobian(self.drr, self.rot, self.xyz, motions=X, weights=self.weights, return_footprints=True, **self.kw)

    def _render(self, X):
        from .polyrigid import render_polyrigid
        return render_polyrigid(self.drr, self.rot, self.xyz, motions=X, weights=self.weights, **self.kw)


def ncc_z(x, eps):
    """(z, sigma) of the global NCC per row of x (B, N): z = (x - mean x) / sigma, sigma = sqrt(var x + eps) (population variance,
    as metrics.NormalizedCrossCorrelation2d.norm); sigma (B, 1)."""
    mu = x.mean(-1, keepdim=True)
    sigma = (x.var(-1, keepdim=True, correction=0) + eps).sqrt()
    return (x - mu) / sigma, sigma


def ncc_z_jvp(y, z, sigma):
    """The Jacobian of z(x) (ncc_z) at the x with (z, sigma), applied to y (B, N): (y - mean y - z <z, y> / N) / sigma.  The
    matrix is symmetric, so this is also its transpose (DESIGN.md 6k)."""
    N = y.shape[-1]
    return (y - y.mean(-1, keepdim=True) - z * (z * y).sum(-1, keepdim=True) / N) / sigma


def field_smoothness(U):
    """R(U) = sum_a mean((U[.., i + 1, ..] - U[.., i, ..])^2) over the three lattice axes, the squared differences of neighbouring
    nodes; U (S, 3, g0, g1, g2) -> (S,).  Axes of one node contribute nothing."""
    R = U.new_zeros(U.shape[0])
    for ax in (2, 3, 4):
        if U.shape[ax] > 1:
            R = R + (U.diff(dim=ax) ** 2).flatten(1).mean(1)
    return R


def field_smoothness_grad(U):
    """dR/dU of field_smoothness, in closed form; U (S, 3, g0, g1, g2).  R is quadratic, so this is also its Hessian applied to U."""
    G = torch.zeros_like(U)
    for ax in (2, 3, 4):
        g = U.shape[ax]
        if g > 1:
            d = U.diff(dim=ax)
            c = d * (2.0 / d[0].numel())
            G.narrow(ax, 1, g - 1).add_(c)
            G.narrow(ax, 0, g - 1).sub_(c)
    return G


def batched_cg(H, b, mu, iters):
    """`iters` conjugate-gradient iterations on the S systems (H + mu_s I) x_s = b_s from x = 0; b (S, ...), mu (S,) and H a
    symmetric positive semi-definite product (S, ...) -> (S, ...).  A system whose residual vanishes or whose curvature
    p^T (H + mu I) p is not positive stops where it is: fixed work, no host sync and no NaN."""
    S = b.shape[0]

    def dot(a, c):
        return (a * c).reshape(S, -1).sum(1)

    def each(s):
        return s.reshape(S, *[1] * (b.dim() - 1))

    x, r = torch.zeros_like(b), b.clone()
    p, rr = r.clone(), dot(r, r)
    active = rr > 0
    for _ in range(iters):
        Ap = H(p) + each(mu.to(b.dtype)) * p
        pAp = dot(p, Ap)
        active = active & (pAp > 0) & torch.isfinite(pAp)
        a = torch.where(active, rr / torch.where(active, pAp, torch.ones_like(pAp)), torch.zeros_like(pAp))
        on = each(active)
        x = torch.where(on, x + each(a) * p, x)
        r = torch.where(on, r - each(a) * Ap, r)
        rr_new = dot(r, r)
        beta = torch.where(active, rr_new / torch.where(rr > 0, rr, torch.ones_like(rr)), torch.zeros_like(rr))
        p = torch.where(on, r + each(beta) * p, p)
        rr = torch.where(active, rr_new, rr)
        active = active & (rr > 0)
    return x


class DeformableLevenbergMarquardt:
    """Levenberg-Marquardt registration of the displacement field of a deformable DRR (DRR.render_deformed) towards `target`, with
    the camera pose fixed (DESIGN.md 6k).

    The objective is E(U) = mean over the views of (1 - NCC(target, img)) + smoothness R(U), R the squared differences of
    neighbouring nodes (field_smoothness).  `field` (3, g0, g1, g2) in world mm is shared by the B views (one objective);
    (B, 3, g0, g1, g2) gives B independent objectives, each with its own view.  It is a fp32 tensor on the density's device,
    updated in place by step().

    A field has 3 g0 g1 g2 unknowns, far too many for a dense Jacobian, so the Gauss-Newton system is used matrix-free: per view
    the residual is r = z(img) - z(target) with the global NCC's z, M its Jacobian (ncc_z_jvp), and
        g = (1/B) sum_b (1/N) J_b^T M_b r_b + smoothness grad R(U),
        H v = (1/B) sum_b (1/N) J_b^T M_b^2 J_b v + smoothness grad R(v),
    (1/B dropped for per-pose fields), J v from the tangent march (b200drr_deform_jvp) and J^T w from the field scatter of
    b200drr_deform_bwd.  Each step runs `cg_iters` conjugate-gradient iterations on (H + mu I) delta = -g from delta = 0
    (batched_cg: one system for a shared field, B for per-pose ones), renders one trial image at U + delta with render_deformed
    and keeps it where the true E is lower (mu / 10 on accept, x 10 on reject).  mu is identity damping; the first step sets
    mu = damping g^T H g / g^T g, so `damping` is dimensionless.  The accepted trial image is the next step's image, so a step
    costs 2 cg_iters + 1 marches and one forward.  The rays and the sampling range do not depend on the field: the model is the
    image's full derivative.  No host sync once warm.

    Only the global NCC is modelled: `loss` None (NormalizedCrossCorrelation2d(eps=eps)) or a NormalizedCrossCorrelation2d
    without patch_size; anything else raises TypeError here.  Full detectors only."""

    def __init__(self, drr, rot: torch.Tensor, xyz: torch.Tensor, field: torch.Tensor, target: torch.Tensor,
                 smoothness: float = 1e-3, cg_iters: int = 10, parameterization: str = "euler_angles", convention: str | None = None,
                 degrees: bool = False, calibration=None, n_points: int = 500, alphamin=None, alphamax=None, loss=None,
                 damping: float = 1e-3, eps: float = 1e-5):
        from . import _lib
        from .deform import _marches, check_supported

        name = type(self).__name__
        loss = _global_ncc(name, loss, eps)
        B = _check_target(name, drr, target, (rot, xyz), parameterization,
                          lambda: check_supported(drr, (rot, xyz), parameterization, field, {}))
        if not (isinstance(cg_iters, int) and cg_iters >= 1):
            raise ValueError(f"cg_iters must be a positive int, got {cg_iters!r}")
        det = drr.detector
        self.drr, self.rot, self.xyz, self.field = drr, rot.detach(), xyz.detach(), field
        self.kw = dict(parameterization=parameterization, convention=convention, degrees=degrees, calibration=calibration,
                       n_points=n_points, alphamin=alphamin, alphamax=alphamax)
        self.loss, self.eps = loss, float(loss.eps)
        self.smoothness, self.cg_iters, self.damping = float(smoothness), cg_iters, float(damping)
        self.shared = field.dim() == 4
        self.B, self.N = B, det.height * det.width
        self.target = target.detach().expand(B, 1, det.height, det.width).contiguous()
        # the views' residual weights 1 / N, and 1 / B for the mean over the views of a shared field's one objective
        self._wt = 1.0 / (self.N * (B if self.shared else 1))
        with torch.no_grad():
            self._zt = ncc_z(self.target.reshape(B, self.N), self.eps)[0]
            source, marches = _marches(drr, (self.rot, self.xyz), B, parameterization, convention, degrees, calibration, alphamin,
                                       alphamax)
        self._rays = (source, *marches[0])
        lib = _lib.load()
        self._scratch = torch.empty(int(lib.b200drr_deform_scratch_floats(B, self.N, det.height, det.width)), dtype=torch.float32,
                                    device=field.device)
        self._lin = drr._affine_inverse.reshape(4, 4)[:3, :3].to(field.dtype)
        self.mu = None     # (S,) identity damping, set on the first step
        self._img = None   # the image at the current field (B, 1, H, W)

    def _systems(self, U):
        """U's shape -> (S, 3, g0, g1, g2): one system for a shared field, B for per-pose ones."""
        return U[None] if self.shared else U

    def _render(self, U):
        from .deform import render_deformed
        return render_deformed(self.drr, self.rot, self.xyz, field=U, **self.kw)

    def _objective(self, img, Us):
        """E of each system (S,) at the image `img` and the system-batched field Us."""
        ncc = 1.0 - self.loss(self.target, img)
        return (ncc.mean(0, keepdim=True) if self.shared else ncc) + self.smoothness * field_smoothness(Us)

    def _chain(self, Us):
        """The field map of the model at the system-batched unknowns Us -> (the kernels' field the march is linearised at, the
        map from a tangent of the unknowns (S, 3, g0, g1, g2) to a tangent of that field, the adjoint of that map): here the field
        is Us itself in voxel units (voxel_field), and the map is voxel_field, whose adjoint in voxel units is the identity."""
        from .deform import voxel_field

        return voxel_field(self.drr, Us), lambda v: voxel_field(self.drr, v), lambda g: g

    def _model(self, Us, img):
        """(grad, H) of the Gauss-Newton model at the system-batched unknowns Us and their image: grad() -> g (S, 3, g0, g1, g2)
        (one scatter march) and the product H(v) on the same shape (two marches), each through the field map of _chain."""
        from .deform import field_jvp, field_vjp

        drr, packed = self.drr, self.drr.renderer._packed_volume(self.drr.density)
        source, tgt, lens, arange, grid = self._rays
        n_points = int(self.kw["n_points"])
        U, tangent, adjoint = self._chain(Us)
        z, sigma = ncc_z(img.reshape(self.B, self.N), self.eps)

        def JT(w):
            gv = adjoint(field_vjp(drr, packed, source, tgt, lens, U, w, arange, n_points, grid, scratch=self._scratch))
            return torch.einsum("ij,bxyzi->bjxyz", self._lin, gv[..., :3])

        def H(v):
            jv = field_jvp(drr, packed, source, tgt, lens, U, tangent(v), arange, n_points, grid)
            return JT(self._wt * ncc_z_jvp(ncc_z_jvp(jv, z, sigma), z, sigma)) + self.smoothness * field_smoothness_grad(v)

        def grad():
            return JT(self._wt * ncc_z_jvp(z - self._zt, z, sigma)) + self.smoothness * field_smoothness_grad(Us)

        return grad, H

    def _current_image(self):
        if self._img is None:
            self._img = self._render(self.field.detach())
        return self._img

    def _keep(self, accept, img_t, img):
        """The next step's image: the trial's for the accepted systems (accept (S,)), the current one's for the others."""
        return torch.where(accept.reshape(-1, 1, 1, 1), img_t, img)

    def gradient(self) -> torch.Tensor:
        """The model's gradient g at the current field, in the field's shape (world mm)."""
        with torch.no_grad():
            grad, _ = self._model(self._systems(self.field.detach()), self._current_image())
            return grad().reshape(self.field.shape)

    def product(self, v: torch.Tensor) -> torch.Tensor:
        """The model's Gauss-Newton product H v at the current field, v and H v in the field's shape (world mm)."""
        with torch.no_grad():
            _, H = self._model(self._systems(self.field.detach()), self._current_image())
            return H(self._systems(v)).reshape(self.field.shape)

    def step(self) -> torch.Tensor:
        """One damped Gauss-Newton step; -> E after it: a 0-d tensor for a shared field, the per-pose (B,) objectives
        otherwise."""
        U = self.field
        with torch.no_grad():
            img = self._current_image()
            Us = self._systems(U.detach())
            grad, H = self._model(Us, img)
            g, S = grad(), Us.shape[0]
            if self.mu is None:
                gg, gHg = (g * g).reshape(S, -1).sum(1), (g * H(g)).reshape(S, -1).sum(1)
                self.mu = torch.where(gg > 0, self.damping * gHg / torch.where(gg > 0, gg, torch.ones_like(gg)),
                                      torch.full_like(gg, self.damping)).clamp(1e-12, 1e12)
            delta = batched_cg(H, -g, self.mu, self.cg_iters)
            Us_t = Us + delta
            U_t = Us_t.reshape(U.shape)
            img_t = self._render(U_t)
            E, E_t = self._objective(img, Us), self._objective(img_t, Us_t)
            accept = E_t < E  # a NaN trial is rejected
            U.copy_(torch.where(accept.reshape(-1, *[1] * 4), Us_t, Us).reshape(U.shape))
            self._img = self._keep(accept, img_t, img)
            self.mu = _next_damping(accept, self.mu)
            out = torch.where(accept, E_t, E)
            return out[0] if self.shared else out


class DiffeomorphicLevenbergMarquardt(DeformableLevenbergMarquardt):
    """Levenberg-Marquardt registration of a stationary velocity field V towards `target`, rendered through its exponential:
    render_deformed(field=exp_velocity(drr, V, steps)), with the camera pose fixed (DESIGN.md 6n).  The map exp(V) stays
    invertible however large the step, where DeformableLevenbergMarquardt's displacement can fold.

    The objective is E(V) = mean over the views of (1 - NCC(target, img)) + smoothness R(V), R = field_smoothness of the velocity.
    `velocity` (3, g0, g1, g2) in world mm is shared by the B views (one objective); (B, 3, g0, g1, g2) gives B independent
    objectives.  It is a fp32 tensor on the density's device, updated in place by step().

    The Gauss-Newton model is DeformableLevenbergMarquardt's with the Jacobian of the march chained to that of the exponential:
    J v = J_render J_exp v, J_exp v from the tangent squarings (b200drr_svf_square_jvp) over the levels of the current V, and
    J^T w through the field scatter, then the squarings' adjoints (b200drr_svf_square_bwd) over the same levels, whose exact
    transpose the tangent is.  Everything between the kernels stays in voxel units.  step(), the batched conjugate gradients, the
    damping and the accept / reject rule are DeformableLevenbergMarquardt's; the levels of the current V (steps fields of
    Bf g0 g1 g2 16 bytes) are computed once with its image and kept with the accepted trial's, so a step costs 2 cg_iters + 1
    marches, 2 cg_iters steps small lattice launches and one forward.  No autograd and no host sync once warm.

    The refusals are DeformableLevenbergMarquardt's, plus exp_velocity's for the velocity and for `steps` (1..16)."""

    def __init__(self, drr, rot: torch.Tensor, xyz: torch.Tensor, velocity: torch.Tensor, target: torch.Tensor, steps: int = 10,
                 smoothness: float = 1e-3, cg_iters: int = 10, parameterization: str = "euler_angles", convention: str | None = None,
                 degrees: bool = False, calibration=None, n_points: int = 500, alphamin=None, alphamax=None, loss=None,
                 damping: float = 1e-3, eps: float = 1e-5):
        from .svf import check_velocity

        check_velocity(drr, velocity, steps)
        super().__init__(drr, rot, xyz, velocity, target, smoothness=smoothness, cg_iters=cg_iters,
                         parameterization=parameterization, convention=convention, degrees=degrees, calibration=calibration,
                         n_points=n_points, alphamin=alphamin, alphamax=alphamax, loss=loss, damping=damping, eps=eps)
        self.steps, self._dims = steps, tuple(drr.density.shape)
        self._exp = None     # (levels, exp) of the current velocity, the kernels' fields in voxel units
        self._trial = None   # (levels, exp) of the last render

    def _render(self, V):
        from .deform import render_voxel_field, voxel_field
        from .svf import square_chain

        self._trial = square_chain(voxel_field(self.drr, V), self.steps, self._dims)
        if self._img is None:   # the current velocity's image (_current_image), not a trial's
            self._exp = self._trial
        kw = self.kw
        return render_voxel_field(self.drr, (self.rot, self.xyz), self.B, self._trial[1], kw["parameterization"], kw["convention"],
                                  kw["degrees"], kw["calibration"], kw["n_points"], kw["alphamin"], kw["alphamax"],
                                  self.drr.density)

    def _keep(self, accept, img_t, img):
        on = accept.reshape(-1, 1, 1, 1, 1)
        (levels_t, phi_t), (levels, phi) = self._trial, self._exp
        self._exp = ([torch.where(on, a, b) for a, b in zip(levels_t, levels)], torch.where(on, phi_t, phi))
        return super()._keep(accept, img_t, img)

    def _chain(self, Vs):
        """The exponential at the current velocity: the march is linearised at exp(V), a velocity tangent goes through the tangent
        squarings (square_chain_jvp) and a field gradient back through their adjoints (square_chain_bwd), over the levels of the
        current V."""
        from .deform import voxel_field
        from .svf import square_chain_bwd, square_chain_jvp

        levels, phi = self._exp
        return (phi, lambda v: square_chain_jvp(levels, voxel_field(self.drr, v), self._dims)[1],
                lambda g: square_chain_bwd(levels, g, self._dims))
