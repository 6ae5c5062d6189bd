"""Image similarity used by the 2D/3D registration loop (the path's caller, SURVEY.md 8f-1).

The image losses of the reference (diffdrr/metrics.py:16-104):
- `NormalizedCrossCorrelation2d`, global (patch_size None) and patch-wise (patch_size p);
- `MultiscaleNormalizedCrossCorrelation2d`, a weighted sum of global and patch NCC;
- `GradientNormalizedCrossCorrelation2d`, NCC of the Gaussian-blurred Sobel gradients (`Sobel`).
On CUDA fp32 they run on the kernels of csrc/ncc.cu (global), csrc/local_ncc.cu (patch-wise) and csrc/sobel.cu (blur + Sobel).
CPU and fp64 inputs take the reference's torch formulas, restated here (the package does not import torchvision).
Mutual information (kornia's kernel-density histograms) and the SE(3) geodesics are not provided.

Reference quirks kept: `MultiscaleNormalizedCrossCorrelation2d` ignores its `eps` argument (every scale uses 1e-5), and
`Sobel` takes one-channel images only (its Conv2d has in_channels = 1).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import _lib


def _stream(x):
    return torch.cuda.current_stream(x.device).cuda_stream


class _NCCFunction(torch.autograd.Function):
    """score[b] = mean_{c,h,w} norm(x1) norm(x2) through b200drr_ncc_fwd / _bwd (three launches per training step instead of
    the ~40 of the reference's elementwise graph, metrics.py:21-44): the registration loop at one pose per step is launch-bound."""

    @staticmethod
    def forward(ctx, x1, x2, eps):
        x1, x2 = x1.contiguous(), x2.contiguous()
        B, C = x1.shape[0], x1.shape[1]
        N = x1[0, 0].numel()
        lib = _lib.load()
        ws = torch.empty(int(lib.b200drr_ncc_workspace_bytes(B, C, N)) // 8, dtype=torch.float64, device=x1.device)
        stats = torch.empty(B * C, 8, dtype=torch.float32, device=x1.device)
        score = torch.empty(B, dtype=torch.float32, device=x1.device)
        _lib.check(lib.b200drr_ncc_fwd(x1.data_ptr(), x2.data_ptr(), B, C, N, float(eps), ws.data_ptr(), stats.data_ptr(),
                                       score.data_ptr(), torch.cuda.current_stream(x1.device).cuda_stream), "b200drr_ncc_fwd")
        ctx.save_for_backward(x1, x2, stats)
        return score

    @staticmethod
    @once_differentiable
    def backward(ctx, gscore):
        x1, x2, stats = ctx.saved_tensors
        B, C = x1.shape[0], x1.shape[1]
        N = x1[0, 0].numel()
        need1, need2 = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need1 or need2):
            return None, None, None
        g1 = torch.empty_like(x1) if need1 else None
        g2 = torch.empty_like(x2) if need2 else None
        gscore = gscore.contiguous().float()
        _lib.check(_lib.load().b200drr_ncc_bwd(x1.data_ptr(), x2.data_ptr(), stats.data_ptr(), gscore.data_ptr(),
                                               g1.data_ptr() if need1 else None, g2.data_ptr() if need2 else None, B, C, N,
                                               torch.cuda.current_stream(x1.device).cuda_stream), "b200drr_ncc_bwd")
        return g1, g2, None


class _LocalNCCFunction(torch.autograd.Function):
    """Patch-wise NCC through b200drr_local_ncc_fwd / _bwd (box sums of the window moments instead of the reference's
    unfold of every p x p window, metrics.py:16-19): 3 launches forward, 2 backward, no (B, C H' W' p^2) copy."""

    @staticmethod
    def forward(ctx, x1, x2, patch_size, eps):
        x1, x2 = x1.contiguous(), x2.contiguous()
        B, C, H, W = x1.shape
        p = patch_size
        lib = _lib.load()
        ws = torch.empty(int(lib.b200drr_local_ncc_workspace_bytes(B, C, H, W, p)) // 8, dtype=torch.float64, device=x1.device)
        stats = torch.empty(B * C, 5, H - p + 1, W - p + 1, dtype=torch.float32, device=x1.device)
        score = torch.empty(B, dtype=torch.float32, device=x1.device)
        _lib.check(lib.b200drr_local_ncc_fwd(x1.data_ptr(), x2.data_ptr(), B, C, H, W, p, float(eps), ws.data_ptr(),
                                             stats.data_ptr(), score.data_ptr(), _stream(x1)), "b200drr_local_ncc_fwd")
        ctx.save_for_backward(x1, x2, stats)
        ctx.patch_size = p
        return score

    @staticmethod
    @once_differentiable
    def backward(ctx, gscore):
        x1, x2, stats = ctx.saved_tensors
        need1, need2 = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need1 or need2):
            return None, None, None, None
        B, C, H, W = x1.shape
        p = ctx.patch_size
        lib = _lib.load()
        ws = torch.empty(int(lib.b200drr_local_ncc_workspace_bytes(B, C, H, W, p)) // 8, dtype=torch.float64, device=x1.device)
        g1 = torch.empty_like(x1) if need1 else None
        g2 = torch.empty_like(x2) if need2 else None
        gscore = gscore.contiguous().float()
        _lib.check(lib.b200drr_local_ncc_bwd(x1.data_ptr(), x2.data_ptr(), stats.data_ptr(), gscore.data_ptr(),
                                             g1.data_ptr() if need1 else None, g2.data_ptr() if need2 else None, B, C, H, W, p,
                                             ws.data_ptr(), _stream(x1)), "b200drr_local_ncc_bwd")
        return g1, g2, None, None


class NormalizedCrossCorrelation2d(torch.nn.Module):
    """Zero-normalized cross correlation between two image batches (B, C, H, W) -> (B,).  With `patch_size` p, every stride-1
    p x p window is normalised on its own and the score is the mean over all windows (metrics.py:16-44)."""

    def __init__(self, patch_size=None, eps: float = 1e-5):
        super().__init__()
        self.patch_size = patch_size
        self.eps = eps

    @staticmethod
    def to_patches(x, patch_size: int):
        """(B, C, H, W) -> (B, C * H' * W', p, p): every p x p window (stride 1) becomes a channel (metrics.py:16-19)."""
        x = x.unfold(2, patch_size, 1).unfold(3, patch_size, 1)
        return x.reshape(x.shape[0], -1, patch_size, patch_size)

    def fused_ok(self, x1, x2) -> bool:
        """The CUDA kernels take full images (patch_size None: the patch view is a strided unfold) of fp32 on one device."""
        return (self.patch_size is None and x1.is_cuda and x2.is_cuda and x1.device == x2.device and x1.dtype == torch.float32
                and x2.dtype == torch.float32 and x1.dim() == 4 and x1.shape[0] * x1.shape[1] <= 65535 and x1.numel() > 0)

    def local_ok(self, x1, x2) -> bool:
        """The patch-wise kernels take (B, C, H, W) fp32 images on one device with 1 <= patch_size <= min(H, W)."""
        return (self.patch_size is not None and x1.is_cuda and x2.is_cuda and x1.device == x2.device
                and x1.dtype == torch.float32 and x2.dtype == torch.float32 and x1.dim() == 4 and x1.shape == x2.shape
                and x1.shape[0] * x1.shape[1] <= 65535 and x1.numel() > 0
                and 1 <= int(self.patch_size) <= min(x1.shape[2], x1.shape[3]))

    def norm(self, x):
        mu = x.mean(dim=(-1, -2), keepdim=True)
        var = x.var(dim=(-1, -2), keepdim=True, correction=0) + self.eps
        return (x - mu) / var.sqrt()

    def forward(self, x1, x2):
        if self.local_ok(x1, x2):
            with torch.cuda.device(x1.device):
                return _LocalNCCFunction.apply(x1, x2, int(self.patch_size), self.eps)
        if self.patch_size is not None:
            x1, x2 = self.to_patches(x1, self.patch_size), self.to_patches(x2, self.patch_size)
        if x1.shape != x2.shape:
            raise AssertionError("Input images must be the same size")
        _, c, h, w = x1.shape
        if self.fused_ok(x1, x2):
            with torch.cuda.device(x1.device):
                return _NCCFunction.apply(x1, x2, self.eps)
        return (self.norm(x1) * self.norm(x2)).flatten(1).sum(dim=1) / (c * h * w)


class MultiscaleNormalizedCrossCorrelation2d(torch.nn.Module):
    """sum_s weight_s * NCC_s(x1, x2) with one NormalizedCrossCorrelation2d(patch_size_s) per scale (metrics.py:47-63).

    As in the reference, `eps` is accepted and ignored: every scale uses NormalizedCrossCorrelation2d's default 1e-5."""

    def __init__(self, patch_sizes=[None], patch_weights=[1.0], eps=1e-5):  # noqa: B006 (the reference's defaults)
        super().__init__()
        if len(patch_sizes) != len(patch_weights):
            raise AssertionError("Each scale must have a weight")
        self.nccs = [NormalizedCrossCorrelation2d(patch_size) for patch_size in patch_sizes]
        self.patch_weights = patch_weights

    def forward(self, x1, x2):
        scores = [weight * ncc(x1, x2) for weight, ncc in zip(self.patch_weights, self.nccs)]
        return torch.stack(scores, dim=0).sum(dim=0)


def gaussian_kernel1d(kernel_size: int, sigma: float, dtype=torch.float32, device="cpu"):
    """torchvision's normalised 1-D Gaussian (transforms/_functional_tensor.py, _get_gaussian_kernel1d), the same ops."""
    half = (kernel_size - 1) * 0.5
    x = torch.linspace(-half, half, steps=kernel_size, dtype=dtype, device=device)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    return pdf / pdf.sum()


class _SobelFunction(torch.autograd.Function):
    """Blur + Sobel through b200drr_sobel_fwd (one launch) / b200drr_sobel_bwd (the exact adjoint, two launches)."""

    @staticmethod
    def forward(ctx, img, weights, ksize):
        x = img.contiguous()
        B, _, H, W = x.shape
        out = torch.empty(B, 2, H, W, dtype=torch.float32, device=x.device)
        _lib.check(_lib.load().b200drr_sobel_fwd(x.data_ptr(), out.data_ptr(), B, H, W, weights.data_ptr(), ksize, _stream(x)),
                   "b200drr_sobel_fwd")
        ctx.save_for_backward(weights)
        ctx.shape, ctx.ksize = (B, H, W), ksize
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        if not ctx.needs_input_grad[0]:
            return None, None, None
        (weights,) = ctx.saved_tensors
        B, H, W = ctx.shape
        gout = gout.contiguous().float()
        lib = _lib.load()
        ws = torch.empty(int(lib.b200drr_sobel_workspace_bytes(B, H, W)) // 4, dtype=torch.float32, device=gout.device)
        g = torch.empty(B, 1, H, W, dtype=torch.float32, device=gout.device)
        _lib.check(lib.b200drr_sobel_bwd(gout.data_ptr(), g.data_ptr(), B, H, W, weights.data_ptr(), ctx.ksize, ws.data_ptr(),
                                         _stream(gout)), "b200drr_sobel_bwd")
        return g, None, None


_SOBEL_TAPS = ([[1.0, 0.0, -1.0], [2.0, 0.0, -2.0], [1.0, 0.0, -1.0]], [[1.0, 2.0, 1.0], [0.0, 0.0, 0.0], [-1.0, -2.0, -1.0]])


class Sobel(torch.nn.Module):
    """Gaussian blur (sigma > 0; torchvision's gaussian_blur: kernel size int(6 sigma + 1) | 1, reflect padding) followed by
    the 3x3 Sobel filters with zero padding: (B, 1, H, W) -> (B, 2, H, W), channels (d/dx, d/dy) (metrics.py:69-93)."""

    def __init__(self, sigma: float):
        super().__init__()
        self.sigma = sigma
        self.kernel_size = (int(6 * sigma + 1) | 1) if sigma > 0 else 1
        self._weights = {}  # device -> fp32 1-D weights, copied once so that a CUDA-graph capture sees no host copy

    def weights(self, device):
        w = self._weights.get(device)
        if w is None:
            w = (gaussian_kernel1d(self.kernel_size, self.sigma) if self.sigma > 0 else torch.ones(1)).to(device)
            self._weights[device] = w
        return w

    def kernel_ok(self, img) -> bool:
        """The CUDA kernels take fp32 images on the GPU (CPU and fp64 inputs take the torch formula)."""
        return img.is_cuda and img.dtype == torch.float32 and img.numel() > 0

    def forward(self, img):
        if img.dim() != 4 or img.shape[1] != 1:
            raise RuntimeError(f"Sobel takes one-channel images (B, 1, H, W), got shape {tuple(img.shape)}")
        R = self.kernel_size // 2
        if R >= img.shape[2] or R >= img.shape[3]:
            raise RuntimeError(f"Sobel(sigma={self.sigma}): the blur's reflect padding of {R} pixels needs images larger than "
                               f"{R} x {R}, got {tuple(img.shape[2:])}")
        if self.kernel_ok(img):
            with torch.cuda.device(img.device):
                return _SobelFunction.apply(img, self.weights(img.device), self.kernel_size)
        x = img
        if self.sigma > 0:
            k1 = gaussian_kernel1d(self.kernel_size, self.sigma, x.dtype, x.device)
            x = F.conv2d(F.pad(x, [R, R, R, R], mode="reflect"), torch.mm(k1[:, None], k1[None, :])[None, None])
        return F.conv2d(x, torch.tensor(_SOBEL_TAPS, dtype=x.dtype, device=x.device).unsqueeze(1), padding=1)


class GradientNormalizedCrossCorrelation2d(NormalizedCrossCorrelation2d):
    """NCC (global, or patch-wise with `patch_size`) of the blurred Sobel gradients of both images (metrics.py:96-104)."""

    def __init__(self, patch_size=None, sigma=1.0, **kwargs):
        super().__init__(patch_size, **kwargs)
        self.sobel = Sobel(sigma)

    def forward(self, x1, x2):
        return super().forward(self.sobel(x1), self.sobel(x2))
