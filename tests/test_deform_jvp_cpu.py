"""The field-tangent (JVP) march on the CPU: the B200_HD math of csrc/deform_math.cuh (deform_ray_jvp) compiled for the host against
a float64 restatement built on deform_oracle's march, the restatement against central differences of deform_oracle.fwd, the
adjoint relation with the field scatter, the image against the forward bit for bit, and the host-side algebra of
DeformableLevenbergMarquardt (the NCC Jacobian, the smoothness term and the batched conjugate gradients) against torch.  Runs
without a GPU."""
import numpy as np
import pytest
import torch

import deform_cases as dc
import deform_oracle as do
import trilinear_cases as tc
from conftest import relerr
from hostemu import emu_deform
from hostemu import emu_deform_jvp as emu
from polyrigid_oracle import _tri
from diffdrr_b200.registration import batched_cg, field_smoothness, field_smoothness_grad, ncc_z, ncc_z_jvp

FLOOR = 1e-4


def jvp_ref(c, V, U=None, dtype=np.float64):
    """L step sum_m G_m . v(x_m) on every sample of every ray (B, N): G_m and v are zero where deform_ray_jvp skips a sample (y_m
    outside the padded volume, x_m outside the lattice's support), so no sample needs masking."""
    U = c["U"] if U is None else U
    q = do._march(c["vol"], c["src"], c["tgt"], U, c["n_points"], c["amin"], c["amax"], 0.5, 1e-8, dtype)
    V = np.asarray(V, dtype)
    v = np.stack([_tri(V[b if V.shape[0] > 1 else 0], q["q"][b])[0] for b in range(q["q"].shape[0])])
    step = dtype(c["amax"] - c["amin"]) / dtype(c["n_points"] - 1)
    return np.asarray(c["raylen"], dtype) * step * (q["G"] * v).sum((-1, -2))


def tangent(c, seed):
    return dc.smooth_field(np.random.default_rng(seed), c["U"].shape[0], c["U"].shape[2:], 1.0)


@pytest.fixture(scope="module", params=sorted(dc.CASES))
def case(request):
    c = dc.CASES[request.param]()
    c["V"] = tangent(c, 100)
    c["ref"] = jvp_ref(c, c["V"])
    c["r32"] = jvp_ref(c, c["V"], dtype=np.float32)
    return c


@pytest.mark.parametrize("packed", [False, True])
def test_emulated_jvp_matches_fp64_restatement(case, packed):
    c = case
    got = emu.deform_jvp(*dc.args(c), c["V"], packed=packed)
    assert np.abs(c["ref"]).max() > 0
    smooth = slice(None) if c["kinks"] is None else ~c["kinks"]   # a ray on an integer plane has a one-sided derivative
    assert relerr(got["jv"][:, smooth], c["ref"][:, smooth]) <= tc.tol(c["r32"][:, smooth], c["ref"][:, smooth], FLOOR)


def test_image_is_the_forward_bitwise_and_gathers_agree(case):
    c = case
    a = emu.deform_jvp(*dc.args(c), c["V"], packed=False)
    b = emu.deform_jvp(*dc.args(c), c["V"], packed=True)
    fwd = emu_deform.deform(*dc.args(c))["out"]
    assert np.array_equal(a["img"], fwd)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_zero_tangent_gives_exact_zeros(case):
    got = emu.deform_jvp(*dc.args(case), np.zeros_like(case["V"]))
    assert np.all(got["jv"] == 0) and not np.signbit(got["jv"]).any()


def test_jvp_is_the_transpose_of_the_field_scatter(case):
    """sum_n w_n (J v)_n = <g_U(w), v>, g_U the emulated backward's field gradient for gout = w: the two marches share the
    samples and G_m, and differ only in the order of the fp32 sums."""
    c = case
    jv = emu.deform_jvp(*dc.args(c), c["V"])["jv"].astype(np.float64)
    gU = emu_deform.deform(*dc.args(c), gout=c["gout"])["g_U"].astype(np.float64)
    lhs = float((c["gout"].astype(np.float64) * jv).sum())
    rhs = float((gU * c["V"]).sum())
    assert lhs != 0 and abs(lhs - rhs) <= 1e-5 * abs(rhs), (lhs, rhs)


@pytest.mark.parametrize("name", ["per_pose", "out_and_back", "source_inside", "shared"])
def test_restatement_matches_central_differences(name):
    c = dc.CASES[name]()
    a = [np.asarray(x, np.float64) for x in dc.args(c)[:5]]
    for seed in (1, 2):
        V = tangent(c, seed).astype(np.float64)
        h = 1e-6
        fd = (do.fwd(*a[:4], a[4] + h * V, c["n_points"], c["amin"], c["amax"]) -
              do.fwd(*a[:4], a[4] - h * V, c["n_points"], c["amin"], c["amax"])) / (2 * h)
        assert np.abs(fd).max() > 0 and relerr(jvp_ref(c, V), fd) <= 1e-6


# ---- DeformableLevenbergMarquardt's host algebra ---------------------------------------------------------------------------------
def test_ncc_jacobian_matches_autograd():
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(3, 50, generator=g, dtype=torch.float64), torch.randn(3, 50, generator=g, dtype=torch.float64)
    eps = 1e-2   # large enough that the eps term is exercised
    _, want = torch.autograd.functional.jvp(lambda t: ncc_z(t, eps)[0], x, y)
    z, sigma = ncc_z(x, eps)
    assert torch.allclose(ncc_z_jvp(y, z, sigma), want, rtol=1e-12, atol=1e-12)
    w = torch.randn(3, 50, generator=g, dtype=torch.float64)   # symmetric: <w, M y> = <M w, y>
    assert torch.allclose((w * ncc_z_jvp(y, z, sigma)).sum(-1), (ncc_z_jvp(w, z, sigma) * y).sum(-1), rtol=1e-12)


@pytest.mark.parametrize("shape", [(1, 3, 5, 4, 6), (2, 3, 4, 1, 3)])
def test_smoothness_gradient_and_product_match_autograd(shape):
    g = torch.Generator().manual_seed(1)
    U, v = torch.randn(*shape, generator=g, dtype=torch.float64), torch.randn(*shape, generator=g, dtype=torch.float64)
    Ur = U.clone().requires_grad_(True)
    field_smoothness(Ur).sum().backward()
    assert torch.allclose(field_smoothness_grad(U), Ur.grad, rtol=1e-12, atol=1e-14)
    _, Hv = torch.autograd.functional.hvp(lambda t: field_smoothness(t).sum(), U, v)
    assert torch.allclose(field_smoothness_grad(v), Hv, rtol=1e-12, atol=1e-14)
    # the test suite's Adam term on a (3, g0, g1, g2) field is the same function
    smooth = sum(((U[0].diff(dim=a)) ** 2).mean() for a in (1, 2, 3) if U.shape[a + 1] > 1)
    assert torch.allclose(field_smoothness(U[:1])[0], smooth)


@pytest.mark.parametrize("S", [1, 3])
def test_batched_cg_solves_small_spd_systems(S):
    g = torch.Generator().manual_seed(2)
    n = 6
    Q = torch.randn(S, n, n, generator=g, dtype=torch.float64)
    A = Q @ Q.transpose(1, 2) + 0.1 * torch.eye(n, dtype=torch.float64)
    b = torch.randn(S, 2, 3, generator=g, dtype=torch.float64)   # the vectors keep their own shape
    mu = torch.rand(S, generator=g, dtype=torch.float64)
    H = lambda p: (A @ p.reshape(S, n, 1)).reshape(p.shape)      # noqa: E731
    x = batched_cg(H, b, mu, iters=n)
    want = torch.linalg.solve(A + mu[:, None, None] * torch.eye(n, dtype=torch.float64), b.reshape(S, n, 1)).reshape(b.shape)
    assert torch.allclose(x, want, rtol=1e-8, atol=1e-10)
    zero = batched_cg(H, torch.zeros_like(b), mu, iters=n)       # a zero right-hand side: zeros, no NaN
    assert torch.equal(zero, torch.zeros_like(b))
    b[0] = 0   # one system done from the start, the others still solved
    x = batched_cg(H, b, mu, iters=n)
    assert torch.equal(x[0], torch.zeros_like(x[0])) and torch.isfinite(x).all()


def test_batched_cg_stops_on_nonpositive_curvature():
    b = torch.tensor([[1.0, 0.0], [1.0, 1.0]], dtype=torch.float64)
    H = lambda p: -p      # noqa: E731  (p^T H p < 0: the system is not SPD)
    x = batched_cg(H, b, torch.zeros(2, dtype=torch.float64), iters=4)
    assert torch.equal(x, torch.zeros_like(x))


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    import ctypes

    from diffdrr_b200 import _lib
    lib = _lib.load()
    n = None
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    assert lib.b200drr_deform_jvp(n, n, 4, 4, 4, n, n, n, n, 1, 2, 2, 2, n, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_deform_jvp_v16(n, n, 1, 4, 4, 4, n, n, n, n, 1, 2, 2, 2, n, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_deform_jvp_v16(p, n, 7, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1  # vol_type
    assert lib.b200drr_deform_jvp(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, n, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # no tangent
    assert lib.b200drr_deform_jvp(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, n, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # no jv
    assert lib.b200drr_deform_jvp(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, q, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # alignment
    assert lib.b200drr_deform_jvp(p, p, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # vol AND packed
    assert lib.b200drr_deform_jvp(p, n, 4, 4, 4, p, p, p, p, 2, 2, 2, 2, p, p, p, 3, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # Bf
    assert lib.b200drr_deform_jvp(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, p, 1, 4, 2, 3, 0.5, 1e-8, 10, p, n) == -1   # H * W != N
    assert lib.b200drr_deform_jvp(p, n, 4, 4, 4, p, p, p, p, 1, 1024, 1024, 512, p, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -2  # 2^31
