"""CPU checks of the NCC normal equations (csrc/ncc_normal.cu, the Gauss-Newton system of LevenbergMarquardt): the kernels' math
compiled for the host against a float64 torch statement that builds the normalised Jacobian of every window explicitly, g against
fp64 autograd of the Gauss-Newton objective, exact results (p = 1, symmetry, positive semidefiniteness), argument validation of
the new entry points, and the loss rejections that need no device."""
import ctypes

import numpy as np
import pytest
import torch

from hostemu import emu_ncc_normal


def _windows(a, p):
    """(B, C, H, W, ...) -> (B, C, windows, n, ...): every stride-1 p x p window (p None: the whole image)."""
    B, C, H, W = a.shape[:4]
    rest = a.shape[4:]
    if p is None:
        return a.reshape(B, C, 1, H * W, *rest)
    a = a.movedim((2, 3), (-2, -1)).unfold(-2, p, 1).unfold(-2, p, 1)  # (B, C, ..., H', W', p, p)
    a = a.reshape(B, C, *rest, (H - p + 1) * (W - p + 1), p * p)
    return a.movedim((-2, -1), (2, 3)) if rest else a


def reference(x, t, J, p, eps=1e-5):
    """(A (B, P, P), g (B, P)) = sum over channels and windows of Jz^T Jz and Jz^T r in float64, r = z(x) - z(t) per window
    and Jz = dz(x)/dtheta built explicitly per (window, pixel).  x, t (B, C, H, W); J (B, C, H, W, P)."""
    x, t, J = x.double(), t.double(), J.double()
    xw, tw, Jw = _windows(x, p), _windows(t, p), _windows(J, p)

    def norm(a):
        mu = a.mean(-1, keepdim=True)
        s = (((a - mu) ** 2).mean(-1, keepdim=True) + eps).sqrt()
        return (a - mu) / s, s

    z, s = norm(xw)
    zt, _ = norm(tw)
    Jz = (Jw - Jw.mean(-2, keepdim=True) - z[..., None] * (z[..., None] * Jw).mean(-2, keepdim=True)) / s[..., None]
    return torch.einsum("bcwqk,bcwql->bkl", Jz, Jz), torch.einsum("bcwqk,bcwq->bk", Jz, z - zt)


def make_case(B, C, H, W, P, offset=0.0, constant=False, seed=0):
    gen = torch.Generator().manual_seed(seed)
    x = torch.rand(B, C, H, W, generator=gen) * 3.0 + offset
    t = 0.5 * x + torch.rand(B, C, H, W, generator=gen)
    if constant:  # one constant window of x and of t at every patch size up to 4
        x[..., :4, :4] = offset + 1.0
        t[..., 2:6, 3:7] = 2.0
    J = torch.randn(B, P, C, H, W, generator=gen)  # the Sobel-plane layout: strides (P C H W, H W, C H W, 1)
    return x, t, J


def sobel_strides(B, C, H, W, P):
    return (P * C * H * W, H * W, C * H * W, 1)


def relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


CASES = [(shape, p, C, P) for shape in ((9, 11), (16, 16)) for p in (1, 3, "min", None) for C in (1, 2) for P in (1, 6, 9, 16)]


def _p(shape, p):
    return min(shape) if p == "min" else p


@pytest.mark.parametrize("shape,p,C,P", CASES)
def test_emulated_kernels_match_explicit_fp64_reference(shape, p, C, P):
    H, W = shape
    p = _p(shape, p)
    B = 2
    x, t, J = make_case(B, C, H, W, P, offset=500.0 if P in (6, 16) else 0.0, constant=P != 1, seed=P + 7 * C)
    A, g = emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), J.numpy(), sobel_strides(B, C, H, W, P), P, 0 if p is None else p)
    Ar, gr = reference(x, t, J.permute(0, 2, 3, 4, 1), p)
    if p == 1:  # one-pixel windows: z = 0, r = 0, Jz = 0
        assert not A.any() and not g.any() and float(Ar.abs().max()) == 0.0
        return
    # the moment form differs from the explicit one by the one-pass variance's cancellation (an offset of 500 costs ~6 digits)
    bound = 1e-9
    assert relerr(A, Ar.numpy()) < bound and relerr(g, gr.numpy()) < bound, (relerr(A, Ar.numpy()), relerr(g, gr.numpy()))
    assert np.array_equal(A, A.transpose(0, 2, 1))
    ev = np.linalg.eigvalsh(A)
    assert ev.min() >= -1e-12 * ev.max()


def test_drr_jacobian_layout_matches_sobel_layout():
    """DRR.jacobian's (B, H W, P) goes in with strides (H W P, 0, 1, P) and gives the system of the same J in plane layout."""
    B, C, H, W, P = 3, 1, 9, 11, 6
    x, t, J = make_case(B, C, H, W, P, seed=4)
    Jd = J[:, :, 0].reshape(B, P, H * W).transpose(1, 2).contiguous()
    for p in (0, 4):
        a = emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), J.numpy(), sobel_strides(B, C, H, W, P), P, p)
        b = emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), Jd.numpy(), (H * W * P, 0, 1, P), P, p)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("C", [1, 2])
def test_g_is_the_gradient_of_the_gauss_newton_objective(C):
    """Independent of the moment algebra: Phi = sum_s w_s / (2 N_s) sum_w |z(x_w) - z(t_w)|^2 with x = x0 + J theta, the
    windows normalised as metrics.py does, differentiated by fp64 autograd at theta = 0."""
    B, H, W, P = 2, 12, 10, 7
    x, t, J = make_case(B, C, H, W, P, offset=20.0, seed=9)
    scales = [(None, 0.5), (3, 0.3), (5, 0.2)]
    theta = torch.zeros(B, P, dtype=torch.float64, requires_grad=True)
    xs = x.double() + torch.einsum("bkchw,bk->bchw", J.double(), theta)
    phi = 0.0
    g = np.zeros((B, P))
    for p, w in scales:
        N = C * H * W if p is None else C * (H - p + 1) * (W - p + 1) * p * p
        xw, tw = _windows(xs, p), _windows(t.double(), p)
        z = lambda a: (a - a.mean(-1, keepdim=True)) / (a.var(-1, keepdim=True, correction=0) + 1e-5).sqrt()  # noqa: E731
        phi = phi + w / (2 * N) * ((z(xw) - z(tw)) ** 2).sum(dim=(1, 2, 3))
        g += emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), J.numpy(), sobel_strides(B, C, H, W, P), P,
                                       0 if p is None else p, weight=w / N)[1]
    (gt,) = torch.autograd.grad(phi.sum(), theta)
    assert relerr(g, gt.numpy()) < 1e-9


def test_weight_scales_and_calls_accumulate():
    B, C, H, W, P = 2, 2, 9, 11, 6
    x, t, J = make_case(B, C, H, W, P, seed=2)
    st = sobel_strides(B, C, H, W, P)
    A1, g1 = emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), J.numpy(), st, P, 3)
    A2, g2 = emu_ncc_normal.ncc_normal(x.numpy(), t.numpy(), J.numpy(), st, P, 3, weight=0.25)
    assert np.allclose(A2, 0.25 * A1, rtol=1e-15, atol=0) and np.allclose(g2, 0.25 * g1, rtol=1e-15, atol=0)


def test_entry_points_reject_bad_arguments_without_gpu():
    from diffdrr_b200 import _lib
    from diffdrr_b200 import build as b200build

    b200build.build()
    lib = _lib.load()
    buf = (ctypes.c_double * 64)()
    q, n = ctypes.cast(buf, ctypes.c_void_p), None
    ok_dims = (1, 1, 8, 8, 3, 6)
    assert lib.b200drr_ncc_normal_workspace_bytes(*ok_dims) > 0
    assert lib.b200drr_ncc_normal_workspace_bytes(1, 1, 8, 8, 0, 6) > 0  # global
    for dims in ((1, 1, 8, 8, 9, 6), (1, 1, 8, 8, -1, 6), (1, 1, 8, 8, 3, 0), (1, 1, 8, 8, 3, 17), (0, 1, 8, 8, 3, 6),
                 (1, 0, 8, 8, 3, 6), (1, 1, 0, 8, 0, 6), (1, 1, 8, -2, 0, 6), (70000, 1, 8, 8, 3, 6), (300, 300, 8, 8, 3, 6)):
        assert lib.b200drr_ncc_normal_workspace_bytes(*dims) == 0, dims
        assert lib.b200drr_ncc_normal(q, q, q, 1, 1, 1, 1, *dims[:4], dims[4], dims[5], 1e-5, 1.0, q, q, q, n) == -1, dims
    ptrs = [q] * 3
    tail = [q] * 3
    for i in range(6):  # any single null pointer: x, t, J, workspace, A, g
        a, b = list(ptrs), list(tail)
        if i < 3:
            a[i] = None
        else:
            b[i - 3] = None
        assert lib.b200drr_ncc_normal(*a, 1, 0, 1, 1, *ok_dims, 1e-5, 1.0, *b, n) == -1, i
    for s in range(4):  # negative strides
        st = [1, 0, 1, 1]
        st[s] = -1
        assert lib.b200drr_ncc_normal(q, q, q, *st, *ok_dims, 1e-5, 1.0, q, q, q, n) == -1, s
    assert lib.b200drr_ncc_normal(q, q, q, 1, 0, 1, 1, *ok_dims, -1e-5, 1.0, q, q, q, n) == -1  # negative eps


def test_levenberg_marquardt_rejects_unsupported_losses_without_gpu():
    from diffdrr_b200 import (DRR, GradientNormalizedCrossCorrelation2d, LevenbergMarquardt, MultiscaleNormalizedCrossCorrelation2d,
                              MutualInformation, NormalizedCrossCorrelation2d, Registration, synthetic)
    from diffdrr_b200.metrics import LogGeodesicSE3

    drr = DRR(synthetic.make_subject(synthetic.make_volume(16, "smooth")), **synthetic.detector_kwargs(12))
    rot, xyz = synthetic.make_poses(1)
    reg = Registration(drr, rot, xyz, "euler_angles", "ZXY")
    target = torch.rand(1, 1, 12, 12)
    for loss in (MutualInformation(), LogGeodesicSE3(), torch.nn.MSELoss(), lambda a, b: (a * b).mean()):
        with pytest.raises(TypeError, match="sum of squares"):
            LevenbergMarquardt(reg, target, loss=loss)

    class MyNCC(NormalizedCrossCorrelation2d):  # a subclass may change forward: its model is unknown
        pass

    with pytest.raises(TypeError, match="sum of squares"):
        LevenbergMarquardt(reg, target, loss=MyNCC())
    for loss in (NormalizedCrossCorrelation2d(patch_size=13), NormalizedCrossCorrelation2d(patch_size=0),
                 MultiscaleNormalizedCrossCorrelation2d([None, 20], [0.5, 0.5]), GradientNormalizedCrossCorrelation2d(patch_size=13)):
        with pytest.raises(ValueError, match="patch_size"):
            LevenbergMarquardt(reg, target, loss=loss)
    with pytest.raises(ValueError, match="reflect padding"):
        LevenbergMarquardt(reg, target, loss=GradientNormalizedCrossCorrelation2d(sigma=4.0))
    with pytest.raises(ValueError, match="one-channel"):
        LevenbergMarquardt(reg, torch.rand(1, 2, 12, 12))
    with pytest.raises(ValueError, match="batch"):
        LevenbergMarquardt(reg, torch.rand(3, 1, 12, 12))
    with pytest.raises(ValueError, match="CUDA"):  # the supported losses still need the GPU
        LevenbergMarquardt(reg, target, loss=GradientNormalizedCrossCorrelation2d(patch_size=5))
