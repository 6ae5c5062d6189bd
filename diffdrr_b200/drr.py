"""`DRR`: the reference's nn.Module surface (reference diffdrr/drr.py:23-312) hosted on the sm_90a renderers.

Same constructor arguments, buffers (`_affine`, `_affine_inverse`, `density`, `mask`), properties and methods
(`forward`, `render`, `set_intrinsics_`, `rescale_detector_`, `perspective_projection`, `inverse_projection`),
so registration / reconstruction code written against DiffDRR runs unchanged:

    drr = DRR(subject, sdd=1020.0, height=200, delx=2.0).to("cuda")
    img = drr(rotations, translations, parameterization="euler_angles", convention="ZXY")   # (B, 1, H, W)

`subject` is duck-typed: anything with `.volume.affine`, `.density.data`, `.mask`, `.reorient`
(a torchio.Subject from diffdrr.data.read, or diffdrr_b200.synthetic.Subject).
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn
from torch.utils.checkpoint import checkpoint

from . import geometry
from .detector import Detector
from .pose import RigidTransform, convert
from .renderers import Siddon, Trilinear, siddon_pose_render, trilinear_pose_render

# B200DRR_TRILINEAR_POSE_IN=0 sends Trilinear training steps through detector.forward + the ray-tensor kernels (A/B runs)
_TRILINEAR_POSE_IN = os.environ.get("B200DRR_TRILINEAR_POSE_IN", "1") != "0"


class DRR(nn.Module):
    """PyTorch module that computes differentiable digitally reconstructed radiographs on an H100."""

    def __init__(
        self,
        subject,  # torchio.Subject-like wrapper of the CT volume
        sdd: float,  # source-to-detector distance
        height: int,  # image height in pixels
        delx: float,  # pixel size along x
        width: int | None = None,
        dely: float | None = None,
        x0: float = 0.0,
        y0: float = 0.0,
        p_subsample: float | None = None,
        reshape: bool = True,
        reverse_x_axis: bool = True,
        patch_size: int | None = None,
        renderer: str = "siddon",
        voxel_shift: float = 0.5,
        persistent: bool = True,
        compile_renderer: bool = False,
        checkpoint_gradients: bool = False,
        **renderer_kwargs,
    ):
        super().__init__()
        width = height if width is None else width
        dely = delx if dely is None else dely
        n_subsample = None if p_subsample is None else int(height * width * p_subsample)
        self.detector = Detector(sdd, height, width, delx, dely, x0, y0, subject.reorient,
                                 reverse_x_axis=reverse_x_axis, n_subsample=n_subsample)

        self.subject = subject
        affine = torch.as_tensor(subject.volume.affine, dtype=torch.float32).unsqueeze(0)
        self.register_buffer("_affine", affine, persistent=persistent)
        self.register_buffer("_affine_inverse", affine.inverse(), persistent=persistent)
        self.register_buffer("density", subject.density.data.squeeze(), persistent=persistent)
        if subject.mask is not None:
            self.register_buffer("mask", subject.mask.data.to(torch.float32).squeeze(), persistent=persistent)

        if renderer == "siddon":
            self.renderer = Siddon(voxel_shift, **renderer_kwargs)
        elif renderer == "trilinear":
            self.renderer = Trilinear(voxel_shift, **renderer_kwargs)
        else:
            raise ValueError(f"renderer must be 'siddon' or 'trilinear', not {renderer}")
        # compile_renderer (reference drr.py:102-103 wraps the renderer in torch.compile): here the renderer already IS one
        # fused CUDA kernel per direction behind a C ABI, so there is nothing for a tracing compiler to fuse.  The flag is
        # honoured explicitly instead of being ignored: the renderer is marked opaque to dynamo (an enclosing torch.compile
        # of the user's model then graph-breaks around it instead of failing on the ctypes calls) and the user is told once.
        self.compile_renderer = compile_renderer
        if compile_renderer:
            import warnings

            self.renderer.forward = torch.compiler.disable(self.renderer.forward)
            warnings.warn("diffdrr_b200: compile_renderer=True has nothing to compile -- the renderer is already a fused sm_90a "
                          "kernel; it is kept as an opaque call (torch.compiler.disable) so an outer torch.compile can wrap it",
                          stacklevel=2)
        self.reshape = reshape
        self.patch_size = patch_size
        self.checkpoint_gradients = checkpoint_gradients

    # ---- geometry helpers -------------------------------------------------------------------------------
    @property
    def affine(self):
        return RigidTransform(self._affine)

    @property
    def affine_inverse(self):
        return RigidTransform(self._affine_inverse)

    @property
    def n_patches(self):
        return (self.detector.height * self.detector.width) // (self.patch_size**2)

    @property
    def device(self):
        return self.density.device

    @property
    def dtype(self):
        return self.density.dtype

    def reshape_transform(self, img, batch_size):
        if not self.reshape:
            return img
        if self.detector.n_subsample is None:
            return img.view(batch_size, -1, self.detector.height, self.detector.width)
        return reshape_subsampled_drr(img, self.detector, batch_size)

    # ---- rendering --------------------------------------------------------------------------------------
    def forward(self, *args, parameterization: str = None, convention: str = None, calibration: RigidTransform = None,
                mask_to_channels: bool = False, degrees: bool = False, **kwargs):
        """SE(3) pose (a RigidTransform, or rotation/translation parameters) -> DRR of shape (B, C, H, W)."""
        fused = self._pose_in_ok(mask_to_channels, kwargs) or self._pose_in_trilinear_ok(mask_to_channels, kwargs, args)
        if (fused and parameterization == "euler_angles" and calibration is None and len(args) == 2
                and geometry.euler_convention_ok(convention) and all(
                    torch.is_tensor(a) and a.is_cuda and a.dtype == torch.float32 and a.dim() == 2 and a.shape[-1] == 3
                    for a in args)
                and args[0].shape == args[1].shape):  # the kernel takes ONE batch size; broadcasting goes through convert()
            # pose parameters -> pose matrix in one kernel (same algebra as pose.convert)
            pose = RigidTransform(geometry.euler_pose(args[0], args[1], convention, degrees))
        elif parameterization is None:
            pose = args[0]
        else:
            pose = convert(*args, parameterization=parameterization, convention=convention, degrees=degrees)
        if fused:
            return self.reshape_transform(self._render_pose_in(pose, calibration, n_points=kwargs.get("n_points", 500)),
                                          batch_size=len(pose))
        source, target = self.detector(pose, calibration)
        if self.detector.n_subsample is not None and hasattr(self.renderer, "ray_subset"):
            # sub-sampled detector: tell the renderer which pixels the rays are and where the full grid's corners project, so
            # that inference batches can take the brick-major kernel (its cost per ray does not depend on the ray spacing)
            det = self.detector
            cached = getattr(self, "_pix_index", None)
            if cached is None or cached[0] is not det or cached[1] != len(det.subsamples) or cached[2].device != source.device:
                cached = (det, len(det.subsamples), det.pixel_index())
                object.__setattr__(self, "_pix_index", cached)
            corners = self.affine_inverse(det.corner_targets(pose, calibration))
            self.renderer.ray_subset = (cached[2], corners, det.height, det.width, len(det.subsamples[-1]))
        if self.checkpoint_gradients:
            # kept for API parity; the fused autograd.Function saves inputs only, so this changes nothing memory-wise
            img = checkpoint(self.render, self.density, source, target, mask_to_channels, **kwargs, use_reentrant=False)
        else:
            img = self.render(self.density, source, target, mask_to_channels, **kwargs)
        return self.reshape_transform(img, batch_size=len(pose))

    # ---- fused pose-in path (SURVEY.md 8f-2) ------------------------------------------------------------------
    def _pose_in_ok(self, mask_to_channels, kwargs) -> bool:
        """True when the whole pose -> rays -> Siddon chain can run as ONE kernel with in-kernel ray generation."""
        r = self.renderer
        return (isinstance(r, Siddon) and r.mode == "nearest" and r.reducefn == "sum"
                and not r.filter_intersections_outside_volume and not mask_to_channels
                and not kwargs.get("align_corners", False) and kwargs.get("mask") is None
                and self.detector.n_subsample is None and self.patch_size is None
                and self.density.is_cuda and self.density.dtype == torch.float32 and self.density.dim() == 3
                and self.density.numel() < 2**31 - 1)

    def _pose_in_trilinear_ok(self, mask_to_channels, kwargs, args) -> bool:
        """True when pose -> rays -> trilinear march can run with in-kernel ray generation: the TRAINING step (pose gradients
        wanted) of a static volume whose packed-corner copy exists; everything else takes the general path."""
        r = self.renderer
        if not (isinstance(r, Trilinear) and r.mode == "bilinear" and r.reducefn == "sum" and _TRILINEAR_POSE_IN
                and not mask_to_channels and set(kwargs) <= {"n_points"}
                and self.detector.n_subsample is None and self.patch_size is None and torch.is_grad_enabled()
                and self.density.is_cuda and self.density.dtype == torch.float32 and self.density.dim() == 3
                and not self.density.requires_grad):
            return False
        wants_grad = any((a.matrix if isinstance(a, RigidTransform) else a).requires_grad
                         for a in args if isinstance(a, RigidTransform) or torch.is_tensor(a))
        return wants_grad and r._packed_volume(self.density) is not None

    def _render_pose_in(self, pose: RigidTransform, calibration: RigidTransform | None, rows: tuple | None = None,
                        n_points: int = 500):
        """detector.forward (detector.py:144-154) + ray lengths / affine_inverse (drr.py:201-205) collapsed into two
        3x4 matrices per pose; the rays themselves are generated inside the CUDA kernel.  `rows=(h0, h1)` renders only
        that block of detector rows (ray sharding across GPUs, parallel.py) -> (B, 1, (h1-h0)*W)."""
        det = self.detector
        if calibration is None and pose.matrix.dtype == torch.float32:
            # the whole composition below as one kernel per direction (include/b200drr.h: b200drr_pose_rays_fwd/_bwd)
            Q, r, Ainv = self._pose_constants()
            src, G, Wd = geometry.pose_rays(pose.matrix, Q, r, Ainv)
            return self._pose_render(src, G, Wd, *self._grid_axes(rows), n_points)
        grid = det.target.view(det.height, det.width, 3)
        if rows is not None:
            grid = grid[rows[0]:rows[1]]
        calib = det._calibration if calibration is None else calibration.matrix
        M = pose.matrix @ det._reorient            # canonical C-arm frame -> world   (reorient.compose(extrinsic))
        T = M @ calib                              # ... including the intrinsic scaling of the detector plane
        A_inv = self._affine_inverse               # world -> voxel index
        G = (A_inv @ T)[:, :3, :]
        src = (A_inv @ M)[:, :3, 3]                # the canonical source is the origin
        Wd = torch.cat([T[:, :3, :3], (T[:, :3, 3] - M[:, :3, 3]).unsqueeze(-1)], dim=-1)  # target - source, world
        return self._pose_render(src, G, Wd, grid[:, 0, 1], grid[0, :, 0], n_points)

    def _pose_render(self, src, G, Wd, rows, cols, n_points):
        if isinstance(self.renderer, Trilinear):
            return trilinear_pose_render(self.renderer, self.density, self.renderer._packed_volume(self.density), src, G, Wd,
                                         rows, cols, n_points)
        return siddon_pose_render(self.renderer, self.density, src, G, Wd, rows, cols)

    def _grid_axes(self, rows: tuple | None):
        """Detector-plane coordinates of the pixel rows / columns (grid[:, 0, 1], grid[0, :, 0]) as contiguous fp32 tensors, cached:
        the strided slices cost two copy kernels per call, and one-pose registration steps are launch-bound."""
        det = self.detector
        key = (id(det), det.target.data_ptr(), det.target._version, det.height, det.width, rows)
        cached = getattr(self, "_grid_axes_cache", None)
        if cached is None or cached[0] != key:
            with torch.no_grad():
                grid = det.target.view(det.height, det.width, 3)
                if rows is not None:
                    grid = grid[rows[0]:rows[1]]
                cached = (key, (grid[:, 0, 1].float().contiguous().clone(), grid[0, :, 0].float().contiguous().clone()))
            object.__setattr__(self, "_grid_axes_cache", cached)
        return cached[1]

    def _pose_constants(self):
        """Q = reorient . calibration, r = reorient[:, 3], Ainv = affine_inverse as contiguous device tensors, rebuilt only
        when the detector / affine buffers change (set_intrinsics_, .to(device))."""
        det = self.detector
        key = (id(det), det._calibration.data_ptr(), det._calibration._version, det._reorient.data_ptr(), det._reorient._version,
               self._affine_inverse.data_ptr(), self._affine_inverse._version)
        cached = getattr(self, "_pose_consts", None)
        if cached is None or cached[0] != key:
            with torch.no_grad():
                reorient = det._reorient.reshape(4, 4).float()
                Q = (reorient @ det._calibration.reshape(4, 4).float()).contiguous()
                r = reorient[:, 3].contiguous()
                Ainv = self._affine_inverse.reshape(4, 4).float().contiguous()
            cached = (key, (Q, r, Ainv))
            object.__setattr__(self, "_pose_consts", cached)
        return cached[1]

    def render(self, density: torch.Tensor, source: torch.Tensor, target: torch.Tensor, mask_to_channels: bool = False,
               grid_shape: tuple | None = None, **kwargs):
        """World-space rays -> line integrals (B, C, N); public because reconstruction code calls it directly.
        `grid_shape=(h, W)` (not in the reference) declares that `target` is a row-major block of h full detector rows, so
        the tiled kernels can be used for it (ray sharding, parallel.py)."""
        img = (target - source).norm(dim=-1).unsqueeze(1)  # ray lengths in world units
        source = self.affine_inverse(source)  # world -> voxel-index coordinates
        target = self.affine_inverse(target)
        kwargs["mask"] = self.mask if mask_to_channels else None
        det = self.detector
        full_grid = det.n_subsample is None and self.patch_size is None and target.shape[1] == det.height * det.width
        if grid_shape is not None and (det.n_subsample is not None or self.patch_size is not None
                                       or grid_shape[1] != det.width or grid_shape[0] * grid_shape[1] != target.shape[1]):
            raise ValueError("grid_shape must describe whole detector rows of an un-sub-sampled, un-patched detector")
        if hasattr(self.renderer, "detector_shape"):  # hint for the tiled kernels; never changes results
            self.renderer.detector_shape = (tuple(grid_shape) if grid_shape is not None
                                            else (det.height, det.width) if full_grid else None)
        if self.patch_size is None:
            try:
                return self.renderer(density, source, target, img, **kwargs)
            finally:
                if hasattr(self.renderer, "ray_subset"):
                    self.renderer.ray_subset = None   # one-shot hint (set by forward() for sub-sampled detectors)
        # serial patches, as the reference does (drr.py:217-225); note Trilinear is not patch-invariant (quirk Q3)
        parts = [
            self.renderer(density, source, t, i, **kwargs)
            for t, i in zip(target.chunk(self.n_patches, dim=1), img.chunk(self.n_patches, dim=-1))
        ]
        return torch.cat(parts, dim=-1)

    # ---- intrinsics editing (drr.py:230-266) ---------------------------------------------------------------
    def set_intrinsics_(self, sdd: float = None, height: int = None, width: int = None, delx: float = None,
                        dely: float = None, x0: float = None, y0: float = None, n_subsample: int = None,
                        reverse_x_axis: bool = None):
        """Replace the detector in place; unspecified parameters keep their current values."""
        d = self.detector
        pick = lambda new, old: old if new is None else new  # noqa: E731
        self.detector = Detector(
            pick(sdd, d.sdd), pick(height, d.height), pick(width, d.width), pick(delx, d.delx), pick(dely, d.dely),
            pick(x0, -d.x0), pick(y0, -d.y0),  # the x0/y0 properties are negated (quirk Q9): undo it
            self.subject.reorient, pick(n_subsample, d.n_subsample), pick(reverse_x_axis, d.reverse_x_axis),
        ).to(self.density)
        # the fused path caches Q = reorient . calibration per detector: a NEW detector must never find the old constants
        # (its buffers can land on the freed addresses of a previous one; ADVICE r1)
        object.__setattr__(self, "_pose_consts", None)
        object.__setattr__(self, "_grid_axes_cache", None)

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)  # .to(device) / .float() / ... replace the buffers
        object.__setattr__(self, "_pose_consts", None)
        object.__setattr__(self, "_grid_axes_cache", None)
        return out

    def rescale_detector_(self, scale: float):
        """Rescale the detector plane in place (multiscale registration)."""
        d = self.detector
        self.set_intrinsics_(height=int(d.height * scale), width=int(d.width * scale), delx=float(d.delx / scale),
                             dely=float(d.dely / scale))

    # ---- 3D <-> 2D helpers (drr.py:269-312) ----------------------------------------------------------------
    def perspective_projection(self, pose: RigidTransform, pts: torch.Tensor):
        """World points (B,N,3) -> pixel coordinates (B,N,2)."""
        camera = self.detector.reorient.compose(pose).inverse()
        x = camera(pts) @ self.detector.intrinsic.mT
        x = x / x[..., 2:3].clone()
        u = self.detector.width - x[..., 0] if self.detector.reverse_x_axis else x[..., 0]
        v = self.detector.height - x[..., 1]
        return torch.stack([u, v], dim=-1)

    def inverse_projection(self, pose: RigidTransform, pts: torch.Tensor):
        """Pixel coordinates (B,N,2) -> world points on the detector plane (B,N,3).  Mutates `pts` like the reference."""
        pts[..., 1] = self.detector.height - pts[..., 1]
        if self.detector.reverse_x_axis:
            pts[..., 0] = self.detector.width - pts[..., 0]
        homog = torch.nn.functional.pad(pts, (0, 1), value=1)
        x = self.detector.sdd * (homog @ self.detector.intrinsic.inverse().mT)
        return self.detector.reorient.compose(pose)(x)


def reshape_subsampled_drr(img: torch.Tensor, detector: Detector, batch_size: int):
    """Scatter sub-sampled rays back onto the (H, W) grid, zeros elsewhere (drr.py:142-147).  The reference's own version only
    broadcasts for batch_size == 1 (it assigns a (B, 1, n) image into a (B, n) slice); here any batch / channel count works."""
    img = img.reshape(batch_size, -1, img.shape[-1])
    drr = torch.zeros(batch_size, img.shape[1], detector.height * detector.width, dtype=img.dtype, device=img.device)
    drr[:, :, detector.pick_tensor().to(img.device)] = img
    return drr.view(batch_size, img.shape[1], detector.height, detector.width)
