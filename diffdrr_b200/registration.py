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


class LevenbergMarquardt:
    """Levenberg-Marquardt steps of a `Registration` towards `target` on the global NCC loss (NormalizedCrossCorrelation2d(),
    patch_size=None), built on DRR.jacobian (DESIGN.md 6e).

    The Gauss-Newton model is the z-normalised residual r = z(img) - z(target), z(x) = (x - mean x) / sqrt(var x + eps)
    (population variance, as in metrics.py), for which |r|^2 / 2N ~= 1 - NCC.  Each step takes one Jacobian, solves the damped
    normal equations (A + lambda diag A) delta = -J_z^T r per pose in float64, renders one trial image, and keeps the trial per
    pose only if its true loss is lower (lambda / 10 on accept, x 10 on reject).  The pose Parameters are updated in place and
    keep their identity, so an optimizer can take over.  The poses are solved independently (for Trilinear with B > 1 the
    coupling through the batch-global sampling range is left out of the model; the true loss still decides).  No host sync."""

    def __init__(self, reg: Registration, target: torch.Tensor, damping: float = 1e-3, eps: float = 1e-5):
        from .metrics import NormalizedCrossCorrelation2d

        self.reg, self.eps = reg, eps
        self.target = target.detach()
        self.ncc = NormalizedCrossCorrelation2d(eps=eps)
        B = reg._rotation.shape[0]
        self.damping = torch.full((B,), float(damping), dtype=torch.float64, device=reg._rotation.device)
        self._zt = self._znorm(self.target.reshape(self.target.shape[0], -1).double())

    def _znorm(self, x):
        xc = x - x.mean(dim=1, keepdim=True)
        s = (xc.square().mean(dim=1, keepdim=True) + self.eps).sqrt()
        return xc / s

    def _loss(self, img):
        return 1.0 - self.ncc(self.target, img)

    def step(self) -> torch.Tensor:
        """One damped Gauss-Newton step; -> the per-pose 1 - NCC after it."""
        reg = self.reg
        rot, xyz = reg._rotation, reg._translation
        kw = dict(parameterization=reg.parameterization, convention=reg.convention)
        from .jacobian import drr_jacobian

        with torch.no_grad():
            # the model is of the image itself: the full derivative even if the renderer stops gradients for training
            img, J = drr_jacobian(reg.drr, rot, xyz, stop_grad=False, **kw)
            B, nr = img.shape[0], rot.shape[1]
            x = img.reshape(B, -1).double()
            Jx = J.reshape(B, x.shape[1], -1).double()
            xc = x - x.mean(dim=1, keepdim=True)
            s = (xc.square().mean(dim=1, keepdim=True) + self.eps).sqrt()
            z = xc / s
            # d z = (dI - mean dI) / s - z mean(z dI) / s
            Jz = (Jx - Jx.mean(dim=1, keepdim=True) - z.unsqueeze(-1) * (z.unsqueeze(-1) * Jx).mean(dim=1, keepdim=True)) / s.unsqueeze(-1)
            r = (z - self._zt).unsqueeze(-1)
            A = Jz.mT @ Jz
            g = Jz.mT @ r
            D = torch.diag_embed(torch.diagonal(A, dim1=-2, dim2=-1).clamp_min(1e-12))
            delta = torch.linalg.solve_ex(A + self.damping[:, None, None] * D, -g)[0].squeeze(-1).to(rot.dtype)
            rot_t, xyz_t = rot + delta[:, :nr], xyz + delta[:, nr:]
            loss, trial = self._loss(img), self._loss(reg.drr(rot_t, xyz_t, **kw))
            accept = trial < loss  # a NaN trial is rejected
            rot.copy_(torch.where(accept[:, None], rot_t, rot))
            xyz.copy_(torch.where(accept[:, None], xyz_t, xyz))
            self.damping = torch.where(accept, self.damping / 10.0, self.damping * 10.0).clamp(1e-12, 1e12)
            return torch.where(accept, trial, loss)
