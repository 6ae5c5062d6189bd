"""The log-Euclidean blended-rigid motion Jacobian on the CPU (DESIGN.md 6p): the velocity's Dlog tangent against central
differences of se3_log_matrix, the library's velocity tangents against torch.func.jacfwd of the fp64 velocity, the fp64 oracle
Jacobian (log_euclidean_jac_oracle.py) against central differences of the fp64 render, the B200_HD P-tangent squaring step
compiled for the host slice by slice against the single-tangent step (bit for bit) and svf_jvp_oracle, the B200_HD Jacobian march
against the oracle, the emulated forward (its image, bit for bit), its footprints and the emulated field scatter, and the C ABI's
refusals.  Runs without a GPU."""
import ctypes
import types

import numpy as np
import pytest
import torch

import log_euclidean_jac_oracle as lo
import svf_jvp_oracle as sj
import svf_oracle as so
import trilinear_cases as tc
from conftest import relerr
from hostemu import emu_deform
from hostemu import emu_log_euclidean_jac as emu
from hostemu import emu_svf_jvp
from diffdrr_b200 import svf
from diffdrr_b200.structures import twist_matrix

DIMS = (21, 25, 17)
STEPS = 4


def _rot(axis, angle):
    w = torch.zeros(6, dtype=torch.float64)
    w[:3] = torch.tensor(axis, dtype=torch.float64) / np.linalg.norm(axis) * angle
    w[3:] = torch.tensor([0.7, -0.4, 0.3], dtype=torch.float64) * angle
    return torch.linalg.matrix_exp(twist_matrix(w))


def _weights(K, g, seed):
    """K smooth bumps on a (g0, g1, g2) lattice, scaled to sum to at most 1."""
    rng = np.random.default_rng(seed)
    x = np.stack(np.meshgrid(*[(np.arange(n) + 0.5) / n for n in g], indexing="ij"), -1)
    w = np.stack([np.exp(-((x - rng.uniform(0.3, 0.7, 3)) ** 2).sum(-1) / 0.08) for _ in range(K)])
    return (w / np.maximum(w.sum(0), 1.0)).astype(np.float32)


def _case(K, per_pose, seed=0, g=(6, 7, 5), H=5, W=6, B=2):
    src, tgt, raylen = tc.miss(DIMS, H, W, B, seed=seed)
    amin, amax = tc.range_of(DIMS, src, tgt)
    rng = np.random.default_rng(seed)
    Bm = B if per_pose else 1
    M = torch.stack([torch.stack([_rot(rng.normal(size=3), rng.uniform(0.05, 0.2)) for _ in range(K)]) for _ in range(Bm)])
    M[..., :3, 3] += torch.as_tensor(rng.normal(size=(Bm, K, 3)))
    w = _weights(K, g, seed)
    piv = torch.as_tensor(rng.uniform(4, 14, size=(K, 3)))
    c = dict(vol=tc.volume(DIMS), src=src, tgt=np.ascontiguousarray(tgt), raylen=np.ascontiguousarray(raylen), n_points=60,
             amin=float(amin), amax=float(amax), H=H, W=W, K=K, M=M, w=w, piv=piv,
             gout=rng.normal(size=raylen.shape).astype(np.float32))
    c["U"], c["T"] = lo.tangents(M, w, piv, STEPS, DIMS)
    c["J"] = lo.jacobian(c, c["U"], c["T"], K)
    return c


CASES = {"shared_k2": lambda: _case(2, False, 1), "per_pose_k3": lambda: _case(3, True, 2), "shared_k5": lambda: _case(5, False, 3)}


@pytest.fixture(scope="module", params=sorted(CASES))
def case(request):
    return CASES[request.param]()


@pytest.mark.parametrize("angle", [0.0, 0.5, 2.5])
def test_dlog_tangent_matches_central_differences(angle):
    Y = _rot([0.3, -1.0, 0.5], angle)
    for i in range(6):
        dY = -(Y @ twist_matrix(torch.eye(6, dtype=torch.float64)[i]))
        got = svf.se3_log_tangents(Y, dY)
        h = 1e-6
        fd = (svf.se3_log_matrix(Y + h * dY) - svf.se3_log_matrix(Y - h * dY)) / (2 * h)
        assert torch.isfinite(got).all()
        assert float((got - fd).abs().max()) <= 1e-7 * max(1.0, float(fd.abs().max())), (i, angle)


@pytest.mark.parametrize("per_pose", [False, True])
def test_velocity_tangents_match_jacfwd_of_the_velocity(per_pose):
    K, g = 3, (4, 5, 3)
    rng = np.random.default_rng(7)
    B = 2 if per_pose else 1
    Minv = torch.stack([torch.stack([_rot(rng.normal(size=3), 0.4 + 0.3 * k) for k in range(K)]) for _ in range(B)])
    X = torch.linalg.inv(Minv)
    w = _weights(K, g, 7)
    piv = torch.as_tensor(rng.uniform(4, 14, size=(K, 3)))
    drr = types.SimpleNamespace(_affine=torch.eye(4), density=torch.empty(DIMS))
    got = svf.velocity_tangents(drr, X if per_pose else X[0], torch.as_tensor(w), piv)
    assert got.shape == (B, *g, 6 * K, 4) and got.dtype == torch.float32 and not got[..., 3].any()
    for b in range(B):
        want = torch.func.jacfwd(lambda xi: lo.velocity(Minv[b:b + 1], w, piv, xi[None], DIMS)[0])(torch.zeros(K, 6,
                                                                                                           dtype=torch.float64))
        want = want.reshape(*g, 3, 6 * K).movedim(-1, -2)
        assert float((got[b, ..., :3].double() - want).abs().max()) <= 2e-6 * float(want.abs().max())


def test_oracle_jacobian_matches_central_differences():
    c = _case(2, True, 4)
    B, K = c["src"].shape[0], c["K"]
    for b, k, i in ((0, 0, 0), (1, 1, 4), (0, 1, 2), (1, 0, 5)):
        h = 1e-6
        fd = []
        for sgn in (1, -1):
            xi = torch.zeros(B, K, 6, dtype=torch.float64)
            xi[b, k, i] = sgn * h
            U = torch.stack([so.exp(lo.velocity(c["M"][j:j + 1], c["w"], c["piv"], xi[j:j + 1], DIMS), STEPS, DIMS)[0]
                             for j in range(B)])
            fd.append(lo.image(c, U)[b])
        fd = (fd[0] - fd[1]) / (2 * h)
        assert np.abs(fd).max() > 0
        assert relerr(c["J"][b, k, :, i], fd) <= 1e-5, (b, k, i)


@pytest.mark.parametrize("s", [1.0 / 16, 1.0])
@pytest.mark.parametrize("P", [1, 6, 13])
def test_emulated_tangent_step_is_the_single_tangent_step_slice_by_slice(P, s):
    rng = np.random.default_rng(P)
    g = (5, 6, 4)
    u = (3.0 * rng.normal(size=(2, *g, 3))).astype(np.float32)
    T = rng.normal(size=(2, *g, P, 3)).astype(np.float32)
    got, lane3, out = emu.square_tangents(u, T, s, DIMS)
    assert not lane3.any()
    for p in range(P):
        want, _, want_out = emu_svf_jvp.square_jvp(u, T[..., p, :], s, DIMS)
        assert np.array_equal(got[..., p, :], want), p
        assert np.array_equal(out, want_out)
        ref = sj.square_jvp(u.astype(np.float64), T[..., p, :].astype(np.float64), s, DIMS).numpy()
        assert np.abs(got[..., p, :] - ref).max() <= 2e-6 * np.abs(ref).max()
    assert emu.square_tangents(u, T, s, DIMS, primal=False)[2] is None


def _emu(c, packed=False):
    U, T = c["U"].numpy().astype(np.float32), c["T"].numpy().astype(np.float32)
    return emu.deform_jac(c["vol"], c["src"], c["tgt"], c["raylen"], U, T, c["K"], c["H"], c["W"], c["n_points"], c["amin"],
                          c["amax"], packed=packed)


def test_emulated_march_matches_the_oracle(case):
    c = case
    got = _emu(c)
    J32 = lo.jacobian(c, c["U"].numpy().astype(np.float32), c["T"].numpy().astype(np.float32), c["K"])
    assert np.abs(c["J"]).max() > 0
    # the oracle's own fp32 error: the fp32-rounded field and tangents marched in fp64 cover the inputs' rounding only, so the
    # rule's floor carries the march's fp32 sums
    assert relerr(got["J"], c["J"]) <= tc.tol(J32, c["J"], 1e-4)


def test_emulated_image_is_the_forward_bitwise_and_gathers_agree(case):
    c = case
    a, b = _emu(c), _emu(c, packed=True)
    U = np.moveaxis(c["U"].numpy().astype(np.float32), -1, 1)
    fwd = emu_deform.deform(c["vol"], c["src"], c["tgt"], c["raylen"], U, c["n_points"], c["amin"], c["amax"])["out"]
    assert np.array_equal(a["img"], fwd)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_jacobian_is_zero_outside_the_footprints(case):
    c = case
    got = _emu(c)
    B, K, H, W = got["J"].shape[0], c["K"], c["H"], c["W"]
    J = got["J"].reshape(B, K, H, W, 6)
    for b in range(B):
        for k in range(K):
            w0, w1, h0, h1 = got["rects"][b, k]
            inside = np.zeros((H, W), bool)
            if w0 <= w1:
                inside[h0:h1 + 1, w0:w1 + 1] = True
            else:
                assert (w0, w1, h0, h1) == (W, -1, H, -1)
            assert not J[b, k][~inside].any()
    assert (got["flushes"] > 0).any()


def test_march_is_the_transpose_of_the_field_scatter(case):
    """sum_n gout_n J[.][n][p] = <g_field, t_p> with g_field the emulated deform backward's field gradient for gout."""
    c = case
    got = _emu(c)
    U = np.moveaxis(c["U"].numpy().astype(np.float32), -1, 1)
    gU = emu_deform.deform(c["vol"], c["src"], c["tgt"], c["raylen"], U, c["n_points"], c["amin"], c["amax"],
                           gout=c["gout"])["g_U"].astype(np.float64)                       # (Bf, 3, g0, g1, g2)
    T = c["T"].numpy().astype(np.float32).astype(np.float64)                             # (Bf, g0, g1, g2, P, 3)
    K = got["J"].shape[1]
    lhs = np.einsum("bn,bknp->bkp", c["gout"].astype(np.float64), got["J"].astype(np.float64))
    rhs = np.einsum("bxyza,bxyzpa->bp", np.moveaxis(gU, 1, -1), T).reshape(-1, K, 6)
    if rhs.shape[0] == 1:
        lhs = lhs.sum(0, keepdims=True)
    assert np.abs(rhs).max() > 0
    assert np.abs(lhs - rhs).max() <= 1e-5 * np.abs(rhs).max()


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    from diffdrr_b200 import _lib

    lib = _lib.load()
    n = None
    bufs = [(ctypes.c_float * 256)() for _ in range(4)]
    p, t, o, r = (ctypes.c_void_p((ctypes.cast(b, ctypes.c_void_p).value + 15) // 16 * 16) for b in bufs)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    st = lib.b200drr_svf_square_tangents
    ok = (1, 6, 2, 2, 2, 4, 4, 4, 1.0, n)
    assert st(n, t, o, r, *ok) == -1                                  # field
    assert st(p, n, o, r, *ok) == -1                                  # tangents
    assert st(p, t, n, r, *ok) == -1                                  # tout
    for P in (0, 49, -1):
        assert st(p, t, o, r, 1, P, 2, 2, 2, 4, 4, 4, 1.0, n) == -1   # P outside 1..48
    assert st(p, t, o, r, 0, 6, 2, 2, 2, 4, 4, 4, 1.0, n) == -1      # Bf
    assert st(p, t, o, r, 1, 6, 2, 2, 2, 4, 4, 4, 0.0, n) == -1      # scale
    for a in ((q, t, o, r), (p, q, o, r), (p, t, q, r), (p, t, o, q)):   # alignment
        assert st(*a, *ok) == -1
    for tout, out in ((p, r), (t, r), (o, p), (o, t), (o, o)):         # aliasing
        assert st(p, t, tout, out, *ok) == -1
    assert st(p, t, o, r, 1, 48, 256, 256, 256, 4, 4, 4, 1.0, n) == -2   # 2^31 floats of tangents per pose
    assert st(p, t, o, r, 1, 1, 1024, 1024, 512, 4, 4, 4, 1.0, n) == -2

    def jac(*change, v16=False, **kw):
        a = dict(vol=p, packed=n, D0=4, D1=4, D2=4, src=p, tgt=p, raylen=p, field=p, Bf=1, g0=2, g1=2, g2=2, tangents=t, P=12, K=2,
                 img=o, J=r, rects=r, B=1, H=2, W=2, shift=0.5, eps=1e-8, n_points=10, arange=p, stream=n)
        a.update(kw)
        args = list(a.values())
        if v16:
            return lib.b200drr_deform_jac_v16(*args[:2], 1, *args[2:])
        return lib.b200drr_deform_jac(*args)

    for v16 in (False, True):
        for kw in (dict(vol=n), dict(tangents=n), dict(img=n), dict(J=n), dict(rects=n), dict(H=0), dict(W=0), dict(P=0),
                   dict(P=49), dict(P=6, K=2), dict(P=12, K=1), dict(tangents=q), dict(img=t), dict(J=t), dict(vol=p, packed=p),
                   dict(Bf=3), dict(B=0), dict(n_points=1)):
            assert jac(v16=v16, **kw) == -1, kw
        assert jac(v16=v16, K=9, P=54) == -1                            # P outside 1..48 first
        assert jac(v16=v16, g0=512, g1=512, g2=512, P=6, K=1) == -2     # 2^31 floats of tangents per pose
        assert jac(v16=v16, g0=1024, g1=1024, g2=512, P=6, K=1) == -2
    assert lib.b200drr_deform_jac_v16(p, n, 7, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, t, 12, 2, o, r, r, 1, 2, 2, 0.5, 1e-8, 10, p, n) == -1
