"""CPU checks of the image losses beyond global NCC: patch-wise NCC (csrc/local_ncc.cu), multiscale NCC and gradient NCC
(csrc/sobel.cu + the NCC kernels).  The modules' torch formulas and the kernels' arithmetic (compiled for the CPU by
tests/hostemu/hostemu_metrics.cpp) are checked against goldens recorded from the UNMODIFIED reference classes (tests/golden/make_golden_metrics.py)
and against fp64 autograd of the reference formulas."""
import ctypes
import inspect
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, relerr
from diffdrr_b200 import (GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d,
                          NormalizedCrossCorrelation2d, Sobel)
from diffdrr_b200.metrics import gaussian_kernel1d

W3 = np.array([1.0, -2.0, 0.5], np.float32)
CASES = (  # golden tag, module factory, input prefix
    ("grad_s1", lambda: GradientNormalizedCrossCorrelation2d(sigma=1.0), "x"),
    ("grad_s1_p5", lambda: GradientNormalizedCrossCorrelation2d(patch_size=5, sigma=1.0), "x"),
    ("grad_s0", lambda: GradientNormalizedCrossCorrelation2d(sigma=0.0), "x"),
    ("multiscale", lambda: MultiscaleNormalizedCrossCorrelation2d([None, 5], [0.5, 0.5]), "x"),
    ("grad_s1_small", lambda: GradientNormalizedCrossCorrelation2d(sigma=1.0), "small_x"),
)


def _golden():
    return dict(np.load(os.path.join(GOLDEN, "metrics_reference.npz")))


def local_ncc_reference(x1, x2, p, eps=1e-5):
    """Reference metrics.py:16-44 with patch_size = p, restated: every stride-1 p x p window normalised on its own."""
    def patches(x):
        x = x.unfold(2, p, 1).unfold(3, p, 1)
        return x.reshape(x.shape[0], -1, p, p)

    def norm(x):
        mu = x.mean(dim=(-1, -2), keepdim=True)
        return (x - mu) / (x.var(dim=(-1, -2), keepdim=True, correction=0) + eps).sqrt()
    a, b = norm(patches(x1)), norm(patches(x2))
    return (a * b).flatten(1).sum(dim=1) / a[0].numel()


def sobel_reference(img, sigma):
    """Reference metrics.py:69-93 (torchvision gaussian_blur: reflect padding + the outer-product kernel; 3x3 Sobel, zero
    padding), restated in plain torch ops."""
    x = img
    if sigma > 0:
        k = int(6 * sigma + 1) | 1
        k1 = gaussian_kernel1d(k, sigma, x.dtype)
        x = torch.nn.functional.conv2d(torch.nn.functional.pad(x, [k // 2] * 4, mode="reflect"),
                                       torch.mm(k1[:, None], k1[None, :])[None, None])
    G = torch.tensor([[[1, 0, -1], [2, 0, -2], [1, 0, -1]], [[1, 2, 1], [0, 0, 0], [-1, -2, -1]]], dtype=x.dtype)
    return torch.nn.functional.conv2d(x, G.unsqueeze(1), padding=1)


def test_modules_match_the_reference_goldens():
    g = _golden()
    for tag, make, src in CASES:
        for dt, suf, tol in ((torch.float32, "f32", 1e-5), (torch.float64, "f64", 1e-12)):
            x1 = torch.as_tensor(g[src + "1"]).to(dt)
            x2 = torch.as_tensor(g[src + "2"]).to(dt).requires_grad_(True)
            score = make()(x1, x2)
            (score * torch.as_tensor(W3[: x1.shape[0]]).to(dt)).sum().backward()
            assert relerr(score.detach().numpy(), g[f"{tag}_score_{suf}"]) < tol, (tag, suf)
            assert relerr(x2.grad.numpy(), g[f"{tag}_grad_x2_{suf}"]) < tol, (tag, suf)


def _emu_ncc(a, b, patch, w):
    """score and (g_a, g_b) of global (patch None; ncc.cu's math) or patch-wise NCC through the emulated kernels"""
    from hostemu import emu, emu_metrics
    if patch is None:
        return emu.ncc(a, b, w)
    return emu_metrics.local_ncc(a, b, patch, w)


def _emu_loss(tag, x1, x2, w):
    """The golden cases through the emulated kernels: Sobel forward of both images, the NCC kernels, Sobel adjoint."""
    from hostemu import emu_metrics as em
    if tag == "multiscale":
        s0, _, g0 = _emu_ncc(x1, x2, None, 0.5 * w)
        s1, _, g1 = _emu_ncc(x1, x2, 5, 0.5 * w)
        return 0.5 * s0 + 0.5 * s1, g0 + g1
    sigma = 0.0 if tag == "grad_s0" else 1.0
    wts = gaussian_kernel1d(7, 1.0).numpy() if sigma > 0 else np.ones(1, np.float32)
    patch = 5 if tag == "grad_s1_p5" else None
    score, _, gs2 = _emu_ncc(em.sobel_fwd(x1, wts), em.sobel_fwd(x2, wts), patch, w)
    return score, em.sobel_bwd(gs2, wts)


def test_emulated_kernels_match_the_reference_goldens():
    g = _golden()
    for tag, _, src in CASES:
        x1, x2 = g[src + "1"], g[src + "2"]
        score, g2 = _emu_loss(tag, x1, x2, W3[: x1.shape[0]])
        ref_err = relerr(g[f"{tag}_grad_x2_f32"], g[f"{tag}_grad_x2_f64"])
        assert relerr(score, g[f"{tag}_score_f64"]) < 5e-6, tag
        assert relerr(g2, g[f"{tag}_grad_x2_f64"]) < max(2e-4, 2 * ref_err), (tag, relerr(g2, g[f"{tag}_grad_x2_f64"]))


LOCAL_CASES = (((2, 3, 50, 47), 5, 0.0), ((1, 1, 64, 64), 13, 0.0), ((2, 2, 12, 9), 1, 0.0), ((1, 2, 7, 12), 7, 0.0),
               ((2, 1, 15, 6), 6, 0.0), ((2, 1, 30, 28), 5, 500.0))


def _autograd_reference(fn, x1, x2, wb):
    """fp64 autograd of `fn` -> (score, g1, g2), and the reference formula's own fp32-vs-fp64 error of the gradients."""
    out = []
    for dt in (torch.float64, torch.float32):
        a, b = x1.to(dt).clone().requires_grad_(True), x2.to(dt).clone().requires_grad_(True)
        s = fn(a, b)
        (s * wb.to(dt)).sum().backward()
        out.append((s.detach().double().numpy(), a.grad.double().numpy(), b.grad.double().numpy()))
    (s, g1, g2), (_, f1, f2) = out
    return s, g1, g2, max(relerr(f1, g1), relerr(f2, g2))


@pytest.mark.parametrize("shape,p,offset", LOCAL_CASES)
def test_emulated_local_ncc_matches_fp64_autograd(shape, p, offset):
    """Patch-wise NCC kernels' math: p = 1, p = min(H, W) (one row or one column of windows), several channels, and an
    intensity offset of 500 (the window variances must not cancel)."""
    from hostemu import emu_metrics
    gen = torch.Generator().manual_seed(11)
    x1 = torch.rand(*shape, generator=gen) * 3.0 + offset
    x2 = (0.5 * x1 + torch.rand(*shape, generator=gen)).contiguous()
    wb = torch.rand(shape[0], generator=gen) - 0.3
    s, g1, g2, ref_err = _autograd_reference(lambda a, b: local_ncc_reference(a, b, p), x1, x2, wb)
    score, e1, e2 = emu_metrics.local_ncc(x1.numpy(), x2.numpy(), p, wb.numpy())
    tol = max(2e-4, 2 * ref_err)
    assert relerr(score, s) < 5e-6
    assert relerr(e1, g1) < tol and relerr(e2, g2) < tol, (relerr(e1, g1), relerr(e2, g2), tol)


@pytest.mark.parametrize("shape,sigma", [((2, 1, 40, 37), 1.0), ((1, 1, 9, 11), 1.0), ((1, 1, 33, 35), 2.5), ((2, 1, 8, 5), 0.0)])
def test_emulated_sobel_matches_fp64_autograd(shape, sigma):
    """Blur + Sobel forward and its adjoint against fp64 autograd of the torch restatement: every pixel of the 9 x 11 image
    lies in the reflect band of the 7-tap blur."""
    from hostemu import emu_metrics
    gen = torch.Generator().manual_seed(4)
    x = torch.rand(*shape, generator=gen) * 2.0
    gout = torch.rand(shape[0], 2, *shape[2:], generator=gen) - 0.5
    xd = x.double().requires_grad_(True)
    ref = sobel_reference(xd, sigma)
    (ref * gout.double()).sum().backward()
    wts = gaussian_kernel1d(int(6 * sigma + 1) | 1, sigma).numpy() if sigma > 0 else np.ones(1, np.float32)
    assert relerr(emu_metrics.sobel_fwd(x.numpy(), wts), ref.detach().numpy()) < 2e-6
    assert relerr(emu_metrics.sobel_bwd(gout.numpy(), wts), xd.grad.numpy()) < 2e-6


def test_constructor_signatures_match_reference():
    # reference metrics.py:24, 50, 70, 99
    params = lambda f: [(p.name, p.default) for p in list(inspect.signature(f).parameters.values())[1:]]  # noqa: E731
    assert params(NormalizedCrossCorrelation2d.__init__) == [("patch_size", None), ("eps", 1e-5)]
    assert params(MultiscaleNormalizedCrossCorrelation2d.__init__) == [("patch_sizes", [None]), ("patch_weights", [1.0]),
                                                                        ("eps", 1e-5)]
    assert params(Sobel.__init__) == [("sigma", inspect.Parameter.empty)]
    assert list(inspect.signature(GradientNormalizedCrossCorrelation2d.__init__).parameters)[1:] == ["patch_size", "sigma", "kwargs"]
    assert inspect.signature(GradientNormalizedCrossCorrelation2d.__init__).parameters["sigma"].default == 1.0


def test_multiscale_ignores_eps_like_the_reference():
    gen = torch.Generator().manual_seed(2)
    x1, x2 = torch.rand(2, 1, 16, 16, generator=gen), torch.rand(2, 1, 16, 16, generator=gen)
    loss = MultiscaleNormalizedCrossCorrelation2d([None, 5], [0.5, 0.5], eps=0.5)
    assert all(n.eps == 1e-5 for n in loss.nccs)
    assert torch.equal(loss(x1, x2), MultiscaleNormalizedCrossCorrelation2d([None, 5], [0.5, 0.5])(x1, x2))
    with pytest.raises(AssertionError, match="weight"):
        MultiscaleNormalizedCrossCorrelation2d([None, 5], [1.0])


def test_sobel_input_validation():
    with pytest.raises(RuntimeError, match="one-channel"):
        Sobel(1.0)(torch.rand(1, 2, 16, 16))
    with pytest.raises(RuntimeError, match="reflect padding"):
        Sobel(1.0)(torch.rand(1, 1, 3, 16))  # 7-tap blur: padding 3 needs more than 3 rows
    with pytest.raises(RuntimeError, match="one-channel"):
        GradientNormalizedCrossCorrelation2d()(torch.rand(1, 3, 16, 16), torch.rand(1, 3, 16, 16))
    assert Sobel(0.0)(torch.rand(1, 1, 2, 2)).shape == (1, 2, 2, 2)  # no blur: any size


def test_new_entry_points_validate_arguments_without_gpu():
    from diffdrr_b200 import _lib
    from diffdrr_b200 import build as b200build
    b200build.build()
    lib = _lib.load()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    n = None
    assert lib.b200drr_local_ncc_workspace_bytes(1, 1, 8, 8, 3) > 0
    assert lib.b200drr_local_ncc_workspace_bytes(1, 1, 8, 8, 9) == 0
    assert lib.b200drr_local_ncc_fwd(n, n, 1, 1, 8, 8, 3, 1e-5, n, n, n, n) == -1
    assert lib.b200drr_local_ncc_bwd(n, n, n, n, n, n, 1, 1, 8, 8, 3, n, n) == -1
    assert lib.b200drr_local_ncc_fwd(p, p, 1, 1, 8, 6, 7, 1e-5, p, p, p, n) == -1   # p > min(H, W)
    assert lib.b200drr_local_ncc_fwd(p, p, 1, 1, 8, 8, 0, 1e-5, p, p, p, n) == -1   # p < 1
    assert lib.b200drr_local_ncc_fwd(p, p, 70000, 1, 8, 8, 3, 1e-5, p, p, p, n) == -1  # B * C > 65535
    assert lib.b200drr_local_ncc_bwd(p, p, p, p, n, n, 1, 1, 8, 8, 3, p, n) == -1   # no gradient requested
    assert lib.b200drr_local_ncc_bwd(p, p, p, p, p, p, 1, 1, 8, 8, 9, p, n) == -1
    assert lib.b200drr_sobel_workspace_bytes(2, 8, 8) == 2 * 8 * 8 * 4
    assert lib.b200drr_sobel_fwd(n, n, 1, 8, 8, n, 7, n) == -1
    assert lib.b200drr_sobel_bwd(n, n, 1, 8, 8, n, 7, n, n) == -1
    assert lib.b200drr_sobel_fwd(p, p, 1, 8, 8, p, 6, n) == -1   # even kernel size
    assert lib.b200drr_sobel_fwd(p, p, 1, 8, 8, p, 0, n) == -1   # non-positive kernel size
    assert lib.b200drr_sobel_fwd(p, p, 1, 8, 8, p, -3, n) == -1
    assert lib.b200drr_sobel_fwd(p, p, 1, 3, 8, p, 7, n) == -1   # reflect padding 3 needs H > 3
    assert lib.b200drr_sobel_bwd(p, p, 1, 8, 8, p, 4, p, n) == -1
