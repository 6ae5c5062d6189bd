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
        """The dtype poses and rays are built in: the density's, or fp32 for a density stored in 16 bits (DESIGN.md 4.5)."""
        return torch.float32 if self.density.dtype in (torch.float16, torch.bfloat16) else self.density.dtype

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

    def jacobian(self, *args, parameterization: str, convention: str = None, degrees: bool = False,
                 calibration: RigidTransform = None, n_points: int = 500, return_range_terms: bool = False):
        """(img, J): the image `self(*args, parameterization=...)` renders and its per-pixel Jacobian with respect to each pose's
        own parameters, J of shape img.shape + (p,) -- the rotation's components first, then the translation's 3 (DESIGN.md 6e).

        Trilinear's sampling range is global over the batch, so with B > 1 pose b's image also depends on the (at most two)
        poses owning the extreme rays; `return_range_terms=True` adds (dI/dalphamin, dI/dalphamax, drange (B, 2, p)) to build
        those cross-pose columns: dI_b/dtheta_c = [b == c] J[b] + dI/dalphamin[b] drange[c, 0] + dI/dalphamax[b] drange[c, 1]
        for c != b.  (None, None, None) for Siddon.  Supported: the fused pose-in paths (Siddon with default options, with or
        without stop_gradients_through_grid_sample; Trilinear with default options and a packed static volume), fp32 / fp16 /
        bf16 densities, the full detector; anything else raises before any launch.  Detached results, no host sync of its own."""
        from .jacobian import drr_jacobian

        return drr_jacobian(self, *args, parameterization=parameterization, convention=convention, degrees=degrees,
                            calibration=calibration, n_points=n_points, return_range_terms=return_range_terms)

    def render_structures(self, *args, motions, labels, parameterization: str = None, convention: str = None,
                          degrees: bool = False, calibration: RigidTransform = None, background: bool = True, **kwargs):
        """Piecewise-rigid DRR (DESIGN.md 6f) -> (B, K + 1, H, W), or (B, K, H, W) with background=False.

        Channel k renders the voxels of `self.mask` labelled labels[k], moved by the rigid world motion motions[..., k, :, :]
        (x -> X x), with the camera pose `*args` (meaning as in forward); the last channel renders every other voxel, label 0
        included, with the camera pose alone.  motions: (K, 4, 4) shared by every pose, or (B, K, 4, 4), fp32 on the density's
        device (a tensor or a RigidTransform; it may require grad).  labels: K distinct integers 0..255 present in the mask.
        With identity motions the channels sum to forward(*args).  Gradients reach the camera pose, the calibration and the
        motions; the density must not require grad.  Supported: Siddon with default options (stop_gradients_through_grid_sample
        honoured), fp32 / fp16 / bf16 densities, the full detector; anything else raises before any launch."""
        from .structures import render_structures

        return render_structures(self, *args, motions=motions, labels=labels, parameterization=parameterization,
                                 convention=convention, degrees=degrees, calibration=calibration, background=background,
                                 **kwargs)

    def structures_jacobian(self, *args, motions, labels, parameterization: str = None, convention: str = None,
                            degrees: bool = False, calibration: RigidTransform = None, background: bool = True, stop_grad=None,
                            **kwargs):
        """(img, J): the render_structures image (B, S, H, W) and the per-pixel Jacobian J (B, K, H, W, 6) of channel k with
        respect to the increment xi_k = (omega, v) of structure k's motion (DESIGN.md 6g).  Only channel k depends on motion k,
        so J[:, k] is also the derivative of the composite img.sum(1).  xi_k is a left increment about the structure's pivot c_k,
        in world coordinates: X_k(xi) = T(c_k) exp(xi^) T(-c_k) X_k; c_k is the world position of the centre of label k's box
        (structures.structure_pivots).  Columns: the rotation's three, then the translation's three.  Arguments as in
        render_structures; stop_grad drops Siddon's ray-length term (None = the renderer's
        stop_gradients_through_grid_sample).  The same set as render_structures is supported, anything else raises before any
        launch.  Detached results; no host sync once the label tables are cached."""
        from .structures import structures_jacobian

        return structures_jacobian(self, *args, motions=motions, labels=labels, parameterization=parameterization,
                                   convention=convention, degrees=degrees, calibration=calibration, background=background,
                                   stop_grad=stop_grad, **kwargs)

    def render_polyrigid(self, *args, motions, weights, parameterization: str = None, convention: str = None,
                         degrees: bool = False, calibration: RigidTransform = None, n_points: int = 500, alphamin=None,
                         alphamax=None, blend: str = "linear", steps: int = 10, density=None, **kwargs):
        """Blended-rigid (skinned) DRR (DESIGN.md 6h, 6m) -> (B, 1, H, W): the volume deformed by K rigid motions that smooth weights
        blend into one continuous map, marched with the Trilinear renderer's rays and samples.

        blend="linear" (the default): every sample x reads the density at x + sum_k w_k(x) (M_k x - x), M_k the voxel-space form of
        X_k^-1: linear blend skinning of the pull-back, rigid wherever one weight is 1 and the identity where all are 0.  Between
        structures with a large relative rotation it loses volume.  blend="log_euclidean": the pull-back is exp(v), v(x) =
        sum_k w_k(x) log(M_k) [x; 1] on the weight lattice's nodes, exponentiated by `steps` squarings (1..16; DESIGN.md 6m) and
        marched as render_deformed marches a field: invertible, volume-preserving between structures, and rigid wherever one
        weight is 1 (up to the squaring's error, which falls 4x per step).  It keeps `steps` lattice-sized fields for the
        backward.  motions: (K, 4, 4) shared by the poses
        or (B, K, 4, 4) world motions x -> X x as in render_structures (a tensor or a RigidTransform; it may require grad).
        weights: (K, g0, g1, g2) fp32 lattice over the volume with values in [0, 1] and sum_k <= 1, e.g. from
        polyrigid.polyrigid_weights; K <= 8.  The camera pose `*args`, calibration, n_points and alphamin / alphamax mean what they
        do in forward.

        density: a volume rendered in place of self.density (the reconstruction idiom: the module keeps the geometry, the fitted
        volume is passed in), of self.density's shape and on its device (ValueError otherwise), fp32 / fp16 / bf16.  An fp32
        density may require grad: for a fixed camera and fixed motions the render is linear in the density, and its gradient is
        the render's transpose, a backprojection along the blended samples (blend="linear": DESIGN.md 6o; blend="log_euclidean":
        render_deformed's, DESIGN.md 6l).  So one volume can be fitted to projections taken while structures move against each
        other (a knee flexion series, a spine between positions), alone or jointly with the motions and the camera.

        Gradients reach the camera pose, the calibration, the motions and a `density=` volume that requires grad; self.density
        (it must not require grad) and the weights get none.  Supported: Trilinear with default options, fp32 / fp16 / bf16
        densities, the full detector, p_subsample and patch_size; anything else raises before any launch.  No host
        synchronisation once the lattice has been seen."""
        from .polyrigid import render_polyrigid

        return render_polyrigid(self, *args, motions=motions, weights=weights, parameterization=parameterization,
                                convention=convention, degrees=degrees, calibration=calibration, n_points=n_points,
                                alphamin=alphamin, alphamax=alphamax, blend=blend, steps=steps, density=density, **kwargs)

    def polyrigid_jacobian(self, *args, motions, weights, parameterization: str = None, convention: str = None,
                           degrees: bool = False, calibration: RigidTransform = None, n_points: int = 500, alphamin=None,
                           alphamax=None, return_footprints: bool = False, blend: str = "linear", steps: int = 10, **kwargs):
        """(img, J): the render_polyrigid image (B, 1, H, W), bit for bit, and its per-pixel Jacobian J (B, K, H, W, 6) with
        respect to the increment xi_k = (omega, v) of each motion (DESIGN.md 6j), from one march.  xi_k is a left increment about
        the pivot c_k in world coordinates, X_k(xi) = T(c_k) exp(xi^) T(-c_k) X_k, c_k the weight-weighted centroid of channel k of
        the lattice (polyrigid.polyrigid_pivots).  Columns: the rotation's three, then the translation's three.  return_footprints
        adds rects (B, K, 4) int32 {w0, w1, h0, h1}: J[:, k] is zero outside rectangle k.  Arguments as in render_polyrigid; the
        same set is supported except p_subsample and patch_size, and anything else raises before any launch.  Detached results;
        no host sync once the lattice has been seen.

        blend="log_euclidean" (DESIGN.md 6p): the Jacobian of render_polyrigid(blend="log_euclidean", steps=steps), whose image it
        returns bit for bit.  The 6K velocity tangents are pushed through the `steps` squarings together and contracted in one
        march; rectangle k then bounds the pixels the exponential's spread of structure k's tangents reaches, wider than the
        support of w_k.  It holds two tangent fields of Bm * g0 * g1 * g2 * 6K * 16 bytes (201 MB at 64^3 with K = 8 and shared
        motions)."""
        from .polyrigid import polyrigid_jacobian

        return polyrigid_jacobian(self, *args, motions=motions, weights=weights, parameterization=parameterization,
                                  convention=convention, degrees=degrees, calibration=calibration, n_points=n_points,
                                  alphamin=alphamin, alphamax=alphamax, return_footprints=return_footprints, blend=blend,
                                  steps=steps, **kwargs)

    def render_deformed(self, *args, field, parameterization: str = None, convention: str = None, degrees: bool = False,
                        calibration: RigidTransform = None, n_points: int = 500, alphamin=None, alphamax=None, density=None,
                        **kwargs):
        """Deformable DRR (DESIGN.md 6i) -> (B, 1, H, W): the volume under a dense displacement field, marched with the Trilinear
        renderer's rays and samples.

        field: fp32 (3, g0, g1, g2) shared by the poses, or (B, 3, g0, g1, g2) one per pose; pull-back displacements in world mm
        (the rendered density at world point p is the CT density at p + u(p)) on a lattice over the volume whose node i of axis a
        sits at voxel coordinate (i + 1/2) D_a / g_a - 1/2, interpolated trilinearly and zero outside the lattice.  It may
        require grad.  The camera pose `*args`, calibration, n_points and alphamin / alphamax mean what they do in forward.

        density: a volume rendered in place of self.density (the reconstruction idiom: the module keeps the geometry, the fitted
        volume is passed in), of self.density's shape and on its device (ValueError otherwise), fp32 / fp16 / bf16.  An fp32
        density may require grad: its gradient is the render's transpose in the density, a backprojection along the warped
        samples (DESIGN.md 6l), so a volume can be fitted to projections taken under known per-view motion (motion-compensated
        reconstruction), alone or jointly with the field and the camera.

        Gradients reach the field, the camera pose, the calibration and a `density=` volume that requires grad; self.density gets
        none (it must not require grad).  Supported: Trilinear with default options, fp32 / fp16 / bf16 densities, the full
        detector, p_subsample and patch_size; anything else raises before any launch.  No host synchronisation."""
        from .deform import render_deformed

        return render_deformed(self, *args, field=field, parameterization=parameterization, convention=convention,
                               degrees=degrees, calibration=calibration, n_points=n_points, alphamin=alphamin,
                               alphamax=alphamax, density=density, **kwargs)

    def deformed_jvp(self, *args, field, tangent, parameterization: str = None, convention: str = None, degrees: bool = False,
                     calibration: RigidTransform = None, n_points: int = 500, alphamin=None, alphamax=None, **kwargs):
        """(img, dimg), both (B, 1, H, W): the render_deformed image, bit for bit, and its directional derivative along the field
        tangent `tangent` (DESIGN.md 6k), from one march: dimg = d/dh render_deformed(field + h tangent) at h = 0, with the rays
        and the sampling range held fixed (they do not depend on the field).  tangent: world mm, the same shape, dtype and device
        as `field`.  Arguments and coverage as in render_deformed (shared or per-pose fields, full, sub-sampled and patched
        detectors, fp32 / fp16 / bf16 densities); anything else, or a tangent that does not match the field, raises before any
        launch.  Detached results; no host synchronisation."""
        from .deform import deformed_jvp

        return deformed_jvp(self, *args, field=field, tangent=tangent, parameterization=parameterization, convention=convention,
                            degrees=degrees, calibration=calibration, n_points=n_points, alphamin=alphamin, alphamax=alphamax,
                            **kwargs)

    # ---- fused pose-in path (SURVEY.md 8f-2) ------------------------------------------------------------------
    def _pose_in_ok(self, mask_to_channels, kwargs) -> bool:
        """True when the whole pose -> rays -> Siddon chain can run as ONE kernel with in-kernel ray generation."""
        r = self.renderer
        return (isinstance(r, Siddon) and r.mode == "nearest" and r.reducefn == "sum"
                and not r.filter_intersections_outside_volume and not mask_to_channels
                and not kwargs.get("align_corners", False) and kwargs.get("mask") is None
                and self.detector.n_subsample is None and self.patch_size is None
                and self.density.is_cuda and self.density.dim() == 3 and self.density.numel() < 2**31 - 1
                and self.density.dtype in (torch.float32, torch.float16, torch.bfloat16))

    def _pose_in_trilinear_ok(self, mask_to_channels, kwargs, args) -> bool:
        """True when pose -> rays -> trilinear march can run with in-kernel ray generation: the TRAINING step (pose gradients
        wanted) of a static volume whose packed-corner copy exists; everything else takes the general path."""
        r = self.renderer
        if not (isinstance(r, Trilinear) and r.mode == "bilinear" and r.reducefn == "sum" and _TRILINEAR_POSE_IN
                and not mask_to_channels and set(kwargs) <= {"n_points"}
                and self.detector.n_subsample is None and self.patch_size is None and torch.is_grad_enabled()
                and self.density.is_cuda and self.density.dim() == 3
                and self.density.dtype in (torch.float32, torch.float16, torch.bfloat16)
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
        return self._pose_render(*self._pose_in_inputs(pose, calibration, rows), n_points)

    def _pose_in_inputs(self, pose: RigidTransform, calibration: RigidTransform | None, rows: tuple | None = None):
        """(src, G, Wd, rows, cols): the inputs of the pose-in kernels for `pose` (see _render_pose_in)."""
        det = self.detector
        if calibration is None and pose.matrix.dtype == torch.float32:
            # the whole composition below as one kernel per direction (include/b200drr.h: b200drr_pose_rays_fwd/_bwd)
            Q, r, Ainv = self._pose_constants()
            src, G, Wd = geometry.pose_rays(pose.matrix, Q, r, Ainv)
            return (src, G, Wd, *self._grid_axes(rows))
        grid = det.target.view(det.height, det.width, 3)
        if rows is not None:
            grid = grid[rows[0]:rows[1]]
        calib = det._calibration if calibration is None else calibration.matrix
        src, G, Wd = pose_in_matrices(pose.matrix, det._reorient, calib, self._affine_inverse)
        return src, G, Wd, grid[:, 0, 1], grid[0, :, 0]

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
        ).to(device=self.density.device, dtype=self.dtype)  # fp32 geometry for a 16-bit density
        # the fused path caches Q = reorient . calibration per detector: a NEW detector must never find the old constants
        # (its buffers can land on the freed addresses of a previous one; ADVICE r1)
        object.__setattr__(self, "_pose_consts", None)
        object.__setattr__(self, "_grid_axes_cache", None)

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)  # .to(device) / .float() / ... replace the buffers
        object.__setattr__(self, "_pose_consts", None)
        object.__setattr__(self, "_grid_axes_cache", None)
        object.__setattr__(self, "_structures_cache", None)  # the label copy and label boxes of render_structures
        object.__setattr__(self, "_polyrigid_cache", None)   # the packed weight lattice of render_polyrigid
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


def pose_in_matrices(P: torch.Tensor, reorient: torch.Tensor, calib: torch.Tensor, A_inv: torch.Tensor):
    """Pose matrices P (B, 4, 4) -> the pose-in kernels' (src (B, 3), G (B, 3, 4), Wd (B, 3, 4)): detector.forward
    (detector.py:144-154) + ray lengths / affine_inverse (drr.py:201-205) collapsed into two 3x4 matrices per pose."""
    M = P @ reorient                           # canonical C-arm frame -> world   (reorient.compose(extrinsic))
    T = M @ calib                              # ... including the intrinsic scaling of the detector plane
    G = (A_inv @ T)[:, :3, :]                  # A_inv: world -> voxel index
    src = (A_inv @ M)[:, :3, 3]                # the canonical source is the origin
    Wd = torch.cat([T[:, :3, :3], (T[:, :3, 3] - M[:, :3, 3]).unsqueeze(-1)], dim=-1)  # target - source, world
    return src, G, Wd


def reshape_subsampled_drr(img: torch.Tensor, detector: Detector, batch_size: int):
    """Scatter sub-sampled rays back onto the (H, W) grid, zeros elsewhere (drr.py:142-147).  The reference's own version only
    broadcasts for batch_size == 1 (it assigns a (B, 1, n) image into a (B, n) slice); here any batch / channel count works."""
    img = img.reshape(batch_size, -1, img.shape[-1])
    drr = torch.zeros(batch_size, img.shape[1], detector.height * detector.width, dtype=img.dtype, device=img.device)
    drr[:, :, detector.pick_tensor().to(img.device)] = img
    return drr.view(batch_size, img.shape[1], detector.height, detector.width)
