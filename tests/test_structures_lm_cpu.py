"""CPU checks of Levenberg-Marquardt over structures (DESIGN.md 6g): the block-sparse normal equations of
csrc/ncc_normal_structures.cu compiled for the host against a float64 torch statement with the dense composite Jacobian and an
explicit Jz, g against fp64 autograd of the Gauss-Newton objective, the footprint kernel's host build against the culling of the
structures render, the motion tangents against float64 central differences, the ABI's argument checks and every refusal."""
import ctypes

import numpy as np
import pytest
import torch

from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, StructuresLevenbergMarquardt, _lib, synthetic
from diffdrr_b200.drr import pose_in_matrices
from diffdrr_b200.metrics import MultiscaleNormalizedCrossCorrelation2d, MutualInformation, GradientNormalizedCrossCorrelation2d
from diffdrr_b200.pose import RigidTransform, convert
from diffdrr_b200.structures import _rigid_inverse, _translation, motion_tangents, se3_exp, twist_matrix
from hostemu import emu_ncc_normal_structures as emu
from hostemu import emu_structures

KW = dict(parameterization="euler_angles", convention="ZXY")


def relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def reference(x, t, Jd, eps=1e-5):
    """(A (B, P, P), g (B, P)) of the global NCC in float64 with the dense composite Jacobian Jd (B, H*W, P) and the explicit
    Jz = (J - mean J - z mean(z J)) / s, r = z(x) - z(t)."""
    x, t, Jd = x.double().flatten(1), t.double().flatten(1), Jd.double()

    def norm(a):
        mu = a.mean(-1, keepdim=True)
        s = (((a - mu) ** 2).mean(-1, keepdim=True) + eps).sqrt()
        return (a - mu) / s, s

    z, s = norm(x)
    zt, _ = norm(t)
    Jz = (Jd - Jd.mean(1, keepdim=True) - z[..., None] * (z[..., None] * Jd).mean(1, keepdim=True)) / s[..., None]
    return torch.einsum("bqk,bql->bkl", Jz, Jz), torch.einsum("bqk,bq->bk", Jz, z - zt)


def make_case(B, K, H, W, overlap, offset=0.0, constant=False, t_batch=None, seed=0):
    """x (B, H, W), t, per-slot J (B, K + 1, H*W, 6) zero outside rects (B, K + 1, 4) (the background slot: whole detector,
    zero J), and the dense composite (B, H*W, 6K)."""
    gen = torch.Generator().manual_seed(seed)
    S = K + 1
    x = torch.rand(B, H, W, generator=gen) * 3.0 + offset
    t = 0.5 * x + torch.rand(B, H, W, generator=gen)
    if t_batch == 1:
        t = t[:1].contiguous()
    if constant:
        x[:] = offset + 1.0
    rects = torch.zeros(B, S, 4, dtype=torch.int32)
    J = torch.zeros(B, S, H, W, 6)
    for b in range(B):
        for k in range(K):
            if overlap:   # random rectangles: some pairs overlap, some do not
                w0, h0 = (int(v) for v in torch.randint(0, W - 3, (1,), generator=gen).tolist() + torch.randint(
                    0, H - 3, (1,), generator=gen).tolist())
                w1 = min(W - 1, w0 + int(torch.randint(1, W // 2, (1,), generator=gen)))
                h1 = min(H - 1, h0 + int(torch.randint(1, H // 2, (1,), generator=gen)))
            else:         # disjoint vertical strips
                w0, w1 = k * W // K, (k + 1) * W // K - 1
                h0, h1 = 1, H - 2
            rects[b, k] = torch.tensor([w0, w1, h0, h1], dtype=torch.int32)
            J[b, k, h0:h1 + 1, w0:w1 + 1] = torch.randn(h1 - h0 + 1, w1 - w0 + 1, 6, generator=gen)
        rects[b, K] = torch.tensor([0, W - 1, 0, H - 1], dtype=torch.int32)
    J = J.reshape(B, S, H * W, 6)
    Jd = J[:, :K].permute(0, 2, 1, 3).reshape(B, H * W, 6 * K)
    return x, t, J, rects, Jd


def strides(J):
    return tuple(J.stride())   # (B, S, H*W, 6): (pose, structure, pixel, parameter)


CASES = [(B, K, overlap, offset, constant) for B, K in ((1, 1), (2, 3), (2, 4), (1, 9)) for overlap in (False, True)
         for offset, constant in ((0.0, False), (500.0, False), (0.0, True))]


@pytest.mark.parametrize("B,K,overlap,offset,constant", CASES)
def test_emulated_kernel_matches_the_dense_fp64_statement(B, K, overlap, offset, constant):
    H, W = 13, 17
    x, t, J, rects, Jd = make_case(B, K, H, W, overlap, offset, constant, seed=K + 10 * B + int(overlap))
    A, g = emu.ncc_normal_structures(x.numpy(), t.numpy(), J.numpy(), strides(J), rects.numpy(), K, K + 1)
    Ar, gr = reference(x, t, Jd)
    # the moment form differs from the explicit one by the one-pass variance's cancellation (an offset of 500 costs digits)
    assert relerr(A, Ar.numpy()) < 1e-9 and relerr(g, gr.numpy()) < 1e-9, (relerr(A, Ar.numpy()), relerr(g, gr.numpy()))
    assert np.array_equal(A, A.transpose(0, 2, 1))
    ev = np.linalg.eigvalsh(A)
    assert ev.min() >= -1e-12 * ev.max()


def test_a_shared_target_and_weights_accumulate():
    B, K, H, W = 3, 3, 11, 12
    x, t, J, rects, Jd = make_case(B, K, H, W, True, t_batch=1, seed=5)
    A1, g1 = emu.ncc_normal_structures(x.numpy(), t.numpy(), J.numpy(), strides(J), rects.numpy(), K, K + 1)
    Ar, gr = reference(x, t.expand(B, H, W), Jd)
    assert relerr(A1, Ar.numpy()) < 1e-9 and relerr(g1, gr.numpy()) < 1e-9
    A2, g2 = emu.ncc_normal_structures(x.numpy(), t.numpy(), J.numpy(), strides(J), rects.numpy(), K, K + 1, weight=0.25)
    assert np.allclose(A2, 0.25 * A1, rtol=1e-15, atol=0) and np.allclose(g2, 0.25 * g1, rtol=1e-15, atol=0)


def test_pairs_without_overlap_have_zero_blocks():
    B, K, H, W = 1, 4, 12, 16
    x, t, J, rects, Jd = make_case(B, K, H, W, False, seed=3)
    A, _ = emu.ncc_normal_structures(x.numpy(), t.numpy(), J.numpy(), strides(J), rects.numpy(), K, K + 1)
    # disjoint footprints: block (j, k) is only the rank-2 correction -a a^T - b b^T, which the dense statement reproduces
    Ar, _ = reference(x, t, Jd)
    assert relerr(A, Ar.numpy()) < 1e-9


def test_g_is_the_gradient_of_the_gauss_newton_objective():
    """Independent of the moment algebra: Phi = 1/(2N) |z(x0 + J theta) - z(t)|^2 differentiated by fp64 autograd at 0."""
    B, K, H, W = 2, 3, 10, 12
    x, t, J, rects, Jd = make_case(B, K, H, W, True, offset=20.0, seed=9)
    N = H * W
    theta = torch.zeros(B, 6 * K, dtype=torch.float64, requires_grad=True)
    xs = x.double().flatten(1) + torch.einsum("bqp,bp->bq", Jd.double(), theta)
    z = lambda a: (a - a.mean(-1, keepdim=True)) / (a.var(-1, keepdim=True, correction=0) + 1e-5).sqrt()  # noqa: E731
    phi = ((z(xs) - z(t.double().flatten(1))) ** 2).sum() / (2 * N)
    (gt,) = torch.autograd.grad(phi, theta)
    _, g = emu.ncc_normal_structures(x.numpy(), t.numpy(), J.numpy(), strides(J), rects.numpy(), K, K + 1, weight=1.0 / N)
    assert relerr(g, gt.numpy()) < 1e-9


def _scene(H=20):
    shape = (24, 20, 28)
    vol = synthetic.make_volume(shape, "phantom", seed=2)
    lab = np.zeros(shape, np.float32)
    lab[3:9, 4:12, 5:15] = 3
    lab[12:20, 8:16, 14:24] = 7
    lab[14:18, 2:6, 2:8] = 12
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(H))
    return drr, vol, lab


def _motions(K, B=None, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    shape = (K,) if B is None else (B, K)
    rot = (torch.rand(*shape, 3, generator=g) * 2 - 1) * 0.2 * scale
    xyz = (torch.rand(*shape, 3, generator=g) * 2 - 1) * 20.0 * scale
    return convert(rot.reshape(-1, 3), xyz.reshape(-1, 3), parameterization="euler_angles", convention="XYZ").matrix.reshape(
        *shape, 4, 4)


@pytest.mark.parametrize("B", [1, 3])
def test_footprint_kernel_host_build_equals_the_render_culling(B):
    drr, vol, lab = _scene()
    labels = (3, 7, 12)
    K, S = 3, 4
    rot, xyz = synthetic.make_poses(B, seed=4)
    P = convert(rot, xyz, **KW).matrix
    X = _motions(K, B, seed=B, scale=3.0)
    Ps = torch.cat([_rigid_inverse(X) @ P[:, None], P[:, None]], dim=1).reshape(B * S, 4, 4)
    det = drr.detector
    src, G, Wd = pose_in_matrices(Ps, det._reorient, det._calibration, drr._affine_inverse)
    grid = det.target.view(det.height, det.width, 3)
    rows, cols = grid[:, 0, 1], grid[0, :, 0]
    boxes = emu_structures.label_boxes(lab.astype(np.uint8))
    box = np.concatenate([boxes[list(labels)], [[0, 0, 0, *vol.shape]]]).astype(np.int32)
    slot_of_label = np.full(256, K, np.int32)
    slot_of_label[list(labels)] = np.arange(K)
    args = [a.detach().numpy() for a in (src, G, Wd, rows, cols)]
    ref = emu_structures.structures(vol, lab, *args, slot_of_label, box, S, sens=False)["rect"]
    got = emu.footprints(args[0], args[1], args[3], args[4], box, S)
    assert np.array_equal(got, ref)
    assert (got[:, 1] - got[:, 0] < 19).any()   # some footprints are smaller than the detector


@pytest.mark.parametrize("per_pose,calibration", [(False, False), (True, False), (True, True)])
def test_motion_tangents_match_fp64_central_differences(per_pose, calibration):
    """d(src, G, Wd)/d xi_k of X_k(xi) = T(c_k) exp(xi^) T(-c_k) X_k, with exp the matrix exponential, by central differences."""
    drr, _, _ = _scene()
    B, K = 2, 3
    rot, xyz = synthetic.make_poses(B, seed=6)
    P = convert(rot, xyz, **KW).matrix
    X = _motions(K, B if per_pose else None, seed=7)
    pivots = torch.randn(K, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(1)) * 30.0
    det = drr.detector
    calib = None
    if calibration:
        C = det._calibration.reshape(1, 4, 4).repeat(B, 1, 1)
        C[:, 0, 0] *= torch.tensor([1.03, 0.97])
        calib = RigidTransform(C)
    dsrc, dG, dWd = motion_tangents(drr, P, X, pivots, K, True, calib)
    S = K + 1
    assert dsrc.shape == (B * S, 6, 3) and dG.shape == (B * S, 6, 3, 4) and dWd.shape == (B * S, 6, 3, 4)
    dsrc, dG, dWd = (d.view(B, S, 6, *d.shape[2:]) for d in (dsrc, dG, dWd))
    assert not dsrc[:, K].any() and not dG[:, K].any() and not dWd[:, K].any()   # the background does not move
    Cm = (det._calibration if calib is None else calib.matrix).double().reshape(-1, 4, 4)
    Xd = X.double().expand(B, K, 4, 4)
    h = 1e-6

    def inputs(k, i, s):
        xi = torch.zeros(6, dtype=torch.float64)
        xi[i] = s
        Xk = _translation(pivots[k]) @ torch.linalg.matrix_exp(twist_matrix(xi)) @ _translation(-pivots[k]) @ Xd[:, k]
        return pose_in_matrices(_rigid_inverse(Xk) @ P.double(), det._reorient.double(), Cm, drr._affine_inverse.double())

    for k in range(K):
        for i in range(6):
            fd = [(a - b) / (2 * h) for a, b in zip(inputs(k, i, h), inputs(k, i, -h))]
            for got, ref in zip((dsrc[:, k, i], dG[:, k, i], dWd[:, k, i]), fd):
                assert relerr(got.numpy(), ref.numpy()) < 1e-6, (k, i)


def test_closed_form_exponential_is_the_matrix_exponential_of_the_twist():
    xi = torch.tensor([[0.3, -0.2, 0.1, 5.0, -3.0, 2.0], [1e-6, 2e-5, -3e-6, 1.0, 2.0, 3.0], [0.0] * 6,
                       [2.5, 0.4, -1.0, -7.0, 0.5, 11.0]], dtype=torch.float64)
    E = se3_exp(xi)
    assert relerr(E.numpy(), torch.linalg.matrix_exp(twist_matrix(xi)).numpy()) < 1e-13
    R = E[:, :3, :3]
    assert torch.allclose(R @ R.mT, torch.eye(3, dtype=torch.float64).expand(4, 3, 3), atol=1e-12)


def test_structures_jacobian_refusals_before_any_launch():
    drr, _, _ = _scene()
    rot, xyz = synthetic.make_poses(1)
    X = torch.eye(4).expand(2, 4, 4)
    with pytest.raises(ValueError, match="labels"):
        drr.structures_jacobian(rot, xyz, motions=X, labels=(), **KW)
    with pytest.raises(ValueError, match="motions"):
        drr.structures_jacobian(rot, xyz, motions=torch.eye(4).expand(3, 4, 4), labels=(3, 7), **KW)
    with pytest.raises(ValueError, match="do not occur"):
        drr.structures_jacobian(rot, xyz, motions=X, labels=(3, 99), **KW)
    with pytest.raises(NotImplementedError, match="renderer options"):
        drr.structures_jacobian(rot, xyz, motions=X, labels=(3, 7), mask=drr.mask, **KW)
    with pytest.raises(_lib.B200DRRError, match="CUDA"):
        drr.structures_jacobian(rot, xyz, motions=X, labels=(3, 7), **KW)
    tri = DRR(synthetic.make_subject(synthetic.make_volume(16, "smooth"), mask=torch.ones(16, 16, 16)),
              **synthetic.detector_kwargs(12), renderer="trilinear")
    with pytest.raises(NotImplementedError, match="Siddon"):
        tri.structures_jacobian(rot, xyz, motions=torch.eye(4)[None], labels=(1,), **KW)


def test_structures_levenberg_marquardt_refusals():
    drr, _, _ = _scene()
    rot, xyz = synthetic.make_poses(2, seed=1)
    X = torch.eye(4).repeat(2, 1, 1)
    target = torch.rand(1, 1, 20, 20)
    for loss in (MutualInformation(), torch.nn.MSELoss(), NormalizedCrossCorrelation2d(patch_size=5),
                 MultiscaleNormalizedCrossCorrelation2d([None, 5], [0.5, 0.5]), GradientNormalizedCrossCorrelation2d()):
        with pytest.raises(TypeError, match="global NCC"):
            StructuresLevenbergMarquardt(drr, rot, xyz, X, (3, 7), target, loss=loss, **KW)

    class MyNCC(NormalizedCrossCorrelation2d):
        pass

    with pytest.raises(TypeError, match="global NCC"):
        StructuresLevenbergMarquardt(drr, rot, xyz, X, (3, 7), target, loss=MyNCC(), **KW)
    with pytest.raises(ValueError, match="one-channel"):
        StructuresLevenbergMarquardt(drr, rot, xyz, X, (3, 7), torch.rand(1, 2, 20, 20), **KW)
    with pytest.raises(ValueError, match="detector"):
        StructuresLevenbergMarquardt(drr, rot, xyz, X, (3, 7), torch.rand(1, 1, 20, 21), **KW)
    with pytest.raises(ValueError, match="batch"):
        StructuresLevenbergMarquardt(drr, rot, xyz, X, (3, 7), torch.rand(3, 1, 20, 20), **KW)
    with pytest.raises(ValueError, match="motions"):
        StructuresLevenbergMarquardt(drr, rot, xyz, RigidTransform(X), (3, 7), target, **KW)
    with pytest.raises(ValueError, match="motions"):
        StructuresLevenbergMarquardt(drr, rot, xyz, torch.eye(4).repeat(3, 1, 1), (3, 7), target, **KW)
    for labels in ((), (3, 3), (3, 99), (3, 300)):
        with pytest.raises(ValueError, match="labels"):
            StructuresLevenbergMarquardt(drr, rot, xyz, X[:max(len(set(labels)), 1)] if labels else X, labels, target, **KW)
    with pytest.raises(_lib.B200DRRError, match="CUDA"):   # a CPU density: the only refusal left for good arguments
        StructuresLevenbergMarquardt(drr, rot, xyz, X, (3, 7), target, **KW)


def test_entry_points_reject_bad_arguments_without_gpu():
    from diffdrr_b200 import build as b200build

    b200build.build()
    lib = _lib.load()
    buf = (ctypes.c_double * 64)()
    q, n = ctypes.cast(buf, ctypes.c_void_p), None
    assert lib.b200drr_ncc_normal_structures_workspace_bytes(1, 1, 8, 8) > 0
    assert lib.b200drr_ncc_normal_structures_workspace_bytes(16, 255, 256, 256) > 0
    bad = ((0, 2, 8, 8), (1, 0, 8, 8), (1, 256, 8, 8), (70000, 2, 8, 8), (1, 2, 0, 8), (1, 2, 8, -1))
    for dims in bad:
        B, K, H, W = dims
        assert lib.b200drr_ncc_normal_structures_workspace_bytes(*dims) == 0, dims
        assert lib.b200drr_ncc_normal_structures(q, q, 1, q, 1, 1, 1, 1, q, B, K, K + 1, H, W, 1e-5, 1.0, q, q, q, n) == -1, dims
    ok = (2, 3, 4, 8, 8)   # B, K, S, H, W

    def call(ptrs=(q,) * 7, t_batch=1, st=(1, 1, 1, 1), dims=ok, eps=1e-5):
        x, t, J, rects, ws, A, g = ptrs
        return lib.b200drr_ncc_normal_structures(x, t, t_batch, J, *st, rects, *dims, eps, 1.0, ws, A, g, n)

    for i in range(7):   # any single null pointer: x, t, J, rects, workspace, A, g
        ptrs = [q] * 7
        ptrs[i] = None
        assert call(ptrs) == -1, i
    for s in range(4):
        st = [1, 1, 1, 1]
        st[s] = -1
        assert call(st=tuple(st)) == -1, s
    assert call(t_batch=3) == -1 and call(t_batch=0) == -1
    assert call(dims=(2, 3, 2, 8, 8)) == -1 and call(dims=(2, 3, 257, 8, 8)) == -1   # S < K, S > 256
    assert call(eps=-1e-5) == -1
    fp = lambda *a: lib.b200drr_structure_footprints(*a, n)  # noqa: E731
    assert fp(None, q, q, q, q, q, 1, 2, 8, 8, 0.5) == -1 and fp(q, q, q, q, q, None, 1, 2, 8, 8, 0.5) == -1
    for dims in ((0, 2, 8, 8), (1, 0, 8, 8), (1, 257, 8, 8), (1, 2, 0, 8), (1, 2, 8, 0)):
        assert fp(q, q, q, q, q, q, *dims, 0.5) == -1, dims
