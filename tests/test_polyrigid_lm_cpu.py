"""The blended-rigid render's per-pixel motion Jacobian and its Levenberg-Marquardt on the CPU (DESIGN.md 6j): the B200_HD march of
csrc/polyrigid_math.cuh (polyrigid_ray_jac, poly_jac_entry) compiled for the host against a per-ray fp64 reference built here from
polyrigid_oracle's per-sample quantities, the tangents and pivots of diffdrr_b200.polyrigid against central differences and by
construction, and every refusal that needs no GPU.  Runs without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

import polyrigid_cases as pc
import polyrigid_oracle as po
import trilinear_cases as tc
from conftest import relerr
from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, PolyrigidLevenbergMarquardt, _lib, synthetic
from diffdrr_b200.metrics import GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d, MutualInformation
from diffdrr_b200.polyrigid import polyrigid_jacobian, polyrigid_pivots, polyrigid_tangents, voxel_maps
from diffdrr_b200.pose import convert
from diffdrr_b200.structures import _rigid_inverse, _translation, apply_increments, twist_matrix
from hostemu import emu_polyrigid as emu
from hostemu import emu_polyrigid_jac as emu_jac

FLOOR = 1e-4
KW = dict(parameterization="euler_angles", convention="ZXY")


def grid_of(c):
    """(H, W) the Jacobian is taken on: the case's detector grid, or its ragged ray set as one row."""
    return (c["H"], c["W"]) if c["H"] else (1, c["tgt"].shape[1])


def case_tangents(c, seed=0):
    """T (Bm, K, 6, 3, 4) of the case's voxel maps under a left increment about random pivots near the volume centre (the
    affine is the identity here): T_i = -(M_k T(c_k) E_i T(-c_k))[:3], the form polyrigid_tangents takes in world space."""
    rng = np.random.default_rng(seed)
    M = c["M"].astype(np.float64)
    Bm, K = M.shape[:2]
    Mh = np.concatenate([M, np.broadcast_to([0.0, 0.0, 0.0, 1.0], (Bm, K, 1, 4))], axis=-2)
    piv = (np.asarray(c["vol"].shape) - 1) / 2 + rng.normal(size=(K, 3)) * 5
    E = twist_matrix(torch.eye(6, dtype=torch.float64)).numpy()
    Tc, Tm = _translation(torch.from_numpy(piv)).numpy(), _translation(torch.from_numpy(-piv)).numpy()
    T = -np.einsum("bkij,kjl,qlm,kmn->bkqin", Mh, Tc, E, Tm)
    return np.ascontiguousarray(T[..., :3, :]).astype(np.float32)


def jac_reference(vol, src, tgt, raylen, M, weights, T, n_points, amin, amax, dtype=np.float64):
    """Per-ray J (B, K, N, 6) from polyrigid_oracle._march's per-sample quantities: dI/dM_k = A_k (x) [s; 1] + B_k (x) [d; 0] with
    A_k = L step sum_m w_k G_m and B_k = L step sum_m alpha_m w_k G_m, contracted with T."""
    q = po._march(vol, src, tgt, M, weights, n_points, amin, amax, 0.5, 1e-8, dtype)
    step = dtype(amax - amin) / dtype(n_points - 1)
    c = np.asarray(raylen, dtype) * step                                        # (B, N)
    G, w, alpha, d = q["G"], q["w"], q["alpha"], q["d"]
    A = c[..., None, None] * np.einsum("bnpk,bnpi->bnki", w, G)
    Bv = c[..., None, None] * np.einsum("bnpk,bnpi->bnki", w * alpha[..., None], G)
    s = np.asarray(src, dtype)
    dM = np.zeros(A.shape + (4,), dtype)
    dM[..., :3] = A[..., None] * s[:, None, None, None, :] + Bv[..., None] * d[:, :, None, None, :]
    dM[..., 3] = A
    Tb = np.broadcast_to(np.asarray(T, dtype), (tgt.shape[0],) + T.shape[1:])
    return np.einsum("bnkij,bkqij->bknq", dM, Tb)


@pytest.fixture(scope="module", params=sorted(pc.CASES))
def case(request):
    c = pc.CASES[request.param]()
    c["T"] = case_tangents(c)
    a = pc.args(c)
    c["jref"] = jac_reference(*a[:6], c["T"], *a[6:])
    c["j32"] = jac_reference(*a[:6], c["T"], *a[6:], dtype=np.float32)
    return c


def emulate(c, packed=False):
    H, W = grid_of(c)
    a = pc.args(c)
    return emu_jac.polyrigid_jac(*a[:6], c["T"], H, W, *a[6:], packed=packed)


def smooth_rays(c):
    """Rays whose derivative is two-sided: all but the axis case's rays on an integer plane (tc.axis_kinks)."""
    return slice(None) if c["kinks"] is None else ~c["kinks"]


@pytest.mark.parametrize("packed", [False, True])
def test_emulated_jacobian_matches_fp64_reference(case, packed):
    c = case
    got = emulate(c, packed)["J"]
    sm = smooth_rays(c)
    ref, r32 = c["jref"][:, :, sm], c["j32"][:, :, sm]
    assert np.abs(ref).max() > 0
    assert relerr(got[:, :, sm], ref) <= tc.tol(r32, ref, FLOOR)


def test_emulated_image_is_the_forward_bitwise_and_gathers_agree(case):
    c = case
    a, b = emulate(c), emulate(c, packed=True)
    assert np.array_equal(a["img"], emu.polyrigid(*pc.args(c))["out"])
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_footprints_contain_every_nonzero_column(case):
    c = case
    H, W = grid_of(c)
    got = emulate(c)
    J, rects = got["J"].reshape(*got["J"].shape[:2], H, W, 6), got["rects"]
    assert J.any()
    for b in range(J.shape[0]):
        for k in range(J.shape[1]):
            w0, w1, h0, h1 = rects[b, k]
            nz = np.argwhere(np.abs(J[b, k]).max(-1) > 0)
            if nz.size == 0:
                continue
            assert h0 <= nz[:, 0].min() and nz[:, 0].max() <= h1 and w0 <= nz[:, 1].min() and nz[:, 1].max() <= w1, (b, k)
            assert 0 <= w0 <= w1 < W and 0 <= h0 <= h1 < H


def test_footprints_are_empty_for_zero_weights_and_tight_on_a_small_support():
    c = pc.CASES["k3_per_pose"]()
    c["T"] = case_tangents(c)
    a = pc.args(c)
    got = emu_jac.polyrigid_jac(*a[:5], np.zeros_like(c["weights"]), c["T"], c["H"], c["W"], *a[6:])
    assert not got["J"].any()
    assert (got["rects"] == np.array([c["W"], -1, c["H"], -1])).all()
    w = np.zeros_like(c["weights"])
    w[1, 3, 4, 2] = 0.5                                                       # one node of channel 1
    got = emu_jac.polyrigid_jac(*a[:5], w, c["T"], c["H"], c["W"], *a[6:])
    r = got["rects"]
    assert (r[:, [0, 2]] == np.array([c["W"], -1, c["H"], -1])).all()          # channels 0 and 2 are empty
    assert (r[:, 1, 0] <= r[:, 1, 1]).all()
    assert ((r[:, 1, 1] - r[:, 1, 0] + 1) * (r[:, 1, 3] - r[:, 1, 2] + 1) < c["H"] * c["W"]).any()


def test_column_sums_are_the_backward_g_M_contracted_with_the_tangents(case):
    """sum_n gout_n J[b, k, n, i] = g_M[bm, k] : T[bm, k, i] of the emulated backward (summed over the views for shared maps)."""
    c = case
    H, W = grid_of(c)
    J = emulate(c)["J"].astype(np.float64)
    gM = emu.polyrigid(*pc.args(c), gout=c["gout"])["g_M"].astype(np.float64)
    lhs = np.einsum("bn,bknq->bkq", c["gout"].astype(np.float64), J)
    if gM.shape[0] == 1:
        lhs = lhs.sum(0, keepdims=True)
    rhs = np.einsum("bkij,bkqij->bkq", gM, c["T"].astype(np.float64))
    assert relerr(lhs, rhs) <= 1e-5


# ---- host algebra: tangents, pivots -------------------------------------------------------------------------------------------
def _drr(shape=(24, 20, 28), H=12, **kw):
    vol = synthetic.make_volume(shape, "phantom", seed=2)
    return DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear", **kw)


def _motions(K, B=None, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    shape = (K,) if B is None else (B, K)
    rot = (torch.rand(*shape, 3, generator=g) * 2 - 1) * 0.2 * scale
    xyz = (torch.rand(*shape, 3, generator=g) * 2 - 1) * 20.0 * scale
    return convert(rot.reshape(-1, 3), xyz.reshape(-1, 3), parameterization="euler_angles", convention="XYZ").matrix.reshape(
        *shape, 4, 4)


def _maps64(drr, X):
    """voxel_maps in float64 (voxel_maps itself returns fp32): (A^-1 X^-1 A)[:3]."""
    A = drr._affine.reshape(4, 4).double()
    return (torch.linalg.inv(A) @ _rigid_inverse(X.double()) @ A)[..., :3, :]


@pytest.mark.parametrize("per_pose", [False, True])
def test_tangents_match_fp64_central_differences(per_pose):
    drr = _drr()
    K, B = 3, 2
    X = _motions(K, B if per_pose else None, seed=3).double()
    pivots = torch.randn(K, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(4)) * 30.0
    T = polyrigid_tangents(drr, X, pivots)
    assert T.dtype == torch.float32 and T.shape == ((B if per_pose else 1), K, 6, 3, 4)
    assert relerr(voxel_maps(drr, X).numpy(), _maps64(drr, X).float().numpy()) == 0.0   # the fp64 restatement is voxel_maps
    h = 1e-6
    for k in range(K):
        for i in range(6):
            xi = torch.zeros(*X.shape[:-2], 6, dtype=torch.float64)
            xi[..., k, i] = h
            fd = (_maps64(drr, apply_increments(X, xi, pivots)) - _maps64(drr, apply_increments(X, -xi, pivots))) / (2 * h)
            fd = fd if fd.dim() == 4 else fd[None]
            assert relerr(T[:, k, i].numpy(), fd[:, k].numpy()) < 1e-6, (k, i)


def test_pivots_of_a_one_hot_lattice_land_on_the_node():
    drr = _drr()
    D = drr.density.shape
    g = (5, 7, 4)
    w = torch.zeros(3, *g)
    w[0, 1, 5, 2] = 0.7
    w[2, 4, 0, 3] = 0.2
    w[2, 4, 6, 3] = 0.2                                                        # two nodes: their midpoint
    A = drr._affine.reshape(4, 4).double()

    def world(v):
        return torch.tensor(v, dtype=torch.float64) @ A[:3, :3].mT + A[:3, 3]

    def node(i):
        return [(i[a] + 0.5) * D[a] / g[a] - 0.5 for a in range(3)]

    got = polyrigid_pivots(drr, w)
    assert got.dtype == torch.float64 and got.shape == (3, 3)
    assert relerr(got[0].numpy(), world(node((1, 5, 2))).numpy()) < 1e-14
    assert relerr(got[1].numpy(), world([(d - 1) / 2 for d in D]).numpy()) < 1e-14      # all-zero channel: the volume centre
    assert relerr(got[2].numpy(), world(node((4, 3, 3))).numpy()) < 1e-14


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def test_polyrigid_jacobian_refusals_before_any_launch():
    drr = _drr()
    rot, xyz = synthetic.make_poses(2, seed=1)
    X = torch.eye(4).expand(2, 4, 4)
    W = torch.full((2, 4, 4, 4), 0.25)
    with pytest.raises(NotImplementedError, match="full detector"):
        _drr(p_subsample=0.5).polyrigid_jacobian(rot, xyz, motions=X, weights=W, **KW)
    with pytest.raises(NotImplementedError, match="full detector"):
        _drr(patch_size=4).polyrigid_jacobian(rot, xyz, motions=X, weights=W, **KW)
    siddon = DRR(synthetic.make_subject(synthetic.make_volume((24, 20, 28), "phantom", seed=2)), **synthetic.detector_kwargs(12))
    with pytest.raises(NotImplementedError, match="Trilinear renderer"):
        siddon.polyrigid_jacobian(rot, xyz, motions=X, weights=W, **KW)
    with pytest.raises(NotImplementedError, match="no renderer options"):
        drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, mask_to_channels=True, **KW)
    with pytest.raises(NotImplementedError, match="at most 8"):
        drr.polyrigid_jacobian(rot, xyz, motions=torch.eye(4).expand(9, 4, 4), weights=torch.zeros(9, 4, 4, 4), **KW)
    with pytest.raises(ValueError, match="motions must be"):
        drr.polyrigid_jacobian(rot, xyz, motions=X[:1].expand(3, 4, 4), weights=W, **KW)
    with pytest.raises(ValueError, match="fp32 lattice"):
        drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W.double(), **KW)
    with pytest.raises(NotImplementedError, match="blend weights"):
        drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W.clone().requires_grad_(True), **KW)
    with pytest.raises(_lib.B200DRRError, match="CUDA"):   # a CPU density: the only refusal left for good arguments
        polyrigid_jacobian(drr, rot, xyz, motions=X, weights=W, **KW)


def test_polyrigid_levenberg_marquardt_refusals():
    drr = _drr()
    rot, xyz = synthetic.make_poses(2, seed=1)
    X = torch.eye(4).repeat(2, 1, 1)
    W = torch.full((2, 4, 4, 4), 0.25)
    target = torch.rand(1, 1, 12, 12)
    for loss in (MutualInformation(), torch.nn.MSELoss(), NormalizedCrossCorrelation2d(patch_size=5),
                 MultiscaleNormalizedCrossCorrelation2d([None, 5], [0.5, 0.5]), GradientNormalizedCrossCorrelation2d()):
        with pytest.raises(TypeError, match="global NCC"):
            PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, loss=loss, **KW)

    class MyNCC(NormalizedCrossCorrelation2d):
        pass

    with pytest.raises(TypeError, match="global NCC"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, loss=MyNCC(), **KW)
    with pytest.raises(ValueError, match="one-channel"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, torch.rand(1, 2, 12, 12), **KW)
    with pytest.raises(ValueError, match="detector"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, torch.rand(1, 1, 12, 13), **KW)
    with pytest.raises(ValueError, match="batch"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, torch.rand(3, 1, 12, 12), **KW)
    with pytest.raises(ValueError, match="motions"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X[0], W, target, **KW)
    with pytest.raises(ValueError, match="motions"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, torch.eye(4).repeat(3, 1, 1), W, target, **KW)
    with pytest.raises(NotImplementedError, match="full detector"):
        PolyrigidLevenbergMarquardt(_drr(p_subsample=0.5), rot, xyz, X, W, target, **KW)
    with pytest.raises(NotImplementedError, match="at most 8"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, torch.eye(4).repeat(9, 1, 1), torch.zeros(9, 4, 4, 4), target, **KW)
    with pytest.raises(_lib.B200DRRError, match="CUDA"):   # a CPU density: the only refusal left for good arguments
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, **KW)


def test_entry_points_reject_bad_arguments_without_a_gpu():
    from diffdrr_b200 import build as b200build

    b200build.build()
    lib = _lib.load()
    buf = (ctypes.c_float * 64)()
    p, n = ctypes.cast(buf, ctypes.c_void_p), None

    def call(vol=p, packed=n, ptrs=(p,) * 10, Bm=1, K=3, B=1, H=4, W=4, n_points=10):
        src, tgt, raylen, M, weights, T, img, J, rects, arange = ptrs
        return lib.b200drr_polyrigid_jac(vol, packed, 4, 4, 4, src, tgt, raylen, M, Bm, K, weights, 2, 2, 2, T, img, J, rects, B, H,
                                         W, 0.5, 1e-8, n_points, arange, n)

    for i in range(10):   # any single null pointer: src, tgt, raylen, M, weights, T, img, J, rects, alpha_range
        ptrs = [p] * 10
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1, i
    assert call(vol=n) == -1 and call(packed=p) == -1                  # exactly one of vol / packed
    assert call(H=0) == -1 and call(W=0) == -1 and call(H=-2, W=-2) == -1   # H * W = 0: full grids only
    assert call(Bm=2) == -1 and call(K=0) == -1 and call(n_points=1) == -1
    assert call(K=9) == -2                                              # K > 8
    v16 = lambda vol_type, **kw: lib.b200drr_polyrigid_jac_v16(p, n, vol_type, 4, 4, 4, p, p, p, p, 1, 3, p, 2, 2, 2, p, p, p, p,  # noqa: E731
                                                               1, kw.get("H", 4), 4, 0.5, 1e-8, 10, p, n)
    assert v16(0) == -1 and v16(7) == -1 and v16(1, H=0) == -1
