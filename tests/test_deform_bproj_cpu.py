"""The deformable render's transpose in the density on the CPU: the B200_HD math of csrc/deform_math.cuh (deform_ray_bproj) compiled
for the host against the float64 backprojection of deform_bproj_oracle, the oracle against differences of deform_oracle.fwd in
the density (the render is linear in it, so these are exact up to rounding), the adjoint relation with the emulated forward, and
the C ABI's argument checks.  Runs without a GPU."""
import numpy as np
import pytest

import deform_bproj_oracle as bo
import deform_cases as dc
import deform_oracle as do
import trilinear_cases as tc
from conftest import relerr
from hostemu import emu_deform
from hostemu import emu_deform_bproj as emu

FLOOR = 1e-4


def _bproj_args(c):
    return (c["src"], c["tgt"], c["raylen"], c["U"], c["n_points"], c["amin"], c["amax"], c["gout"])


@pytest.fixture(scope="module", params=sorted(dc.CASES))
def case(request):
    c = dc.CASES[request.param]()
    a = (c["vol"], c["src"], c["tgt"], c["raylen"], c["U"], c["gout"], c["n_points"], c["amin"], c["amax"])
    c["ref"] = bo.bproj(*a)
    c["r32"] = bo.bproj(*a, dtype=np.float32)
    return c


def test_emulated_bproj_matches_fp64_oracle(case):
    c = case
    got = emu.deform_bproj(c["vol"].shape, *_bproj_args(c))
    assert np.abs(c["ref"]).max() > 0
    assert relerr(got, c["ref"]) <= tc.tol(c["r32"], c["ref"], FLOOR)


def test_oracle_matches_differences_of_the_forward(case):
    """sum_n gout_n (fwd(V + dV) - fwd(V - dV))_n / 2 = <g_V, dV> along random directions and on single voxels, in float64."""
    c = case
    a = [np.asarray(x, np.float64) for x in dc.args(c)[:5]]
    gout = c["gout"].astype(np.float64)
    rng = np.random.default_rng(11)

    def diff(dV):
        plus = do.fwd(a[0] + dV, *a[1:], c["n_points"], c["amin"], c["amax"])
        minus = do.fwd(a[0] - dV, *a[1:], c["n_points"], c["amin"], c["amax"])
        return float((gout * (plus - minus)).sum()) / 2

    for _ in range(2):
        dV = rng.normal(size=a[0].shape)
        want = float((c["ref"] * dV).sum())
        assert want != 0 and abs(diff(dV) - want) <= 1e-9 * np.abs(c["ref"]).sum() * np.abs(dV).max(), (diff(dV), want)
    hit = np.flatnonzero(c["ref"])
    for k in list(rng.choice(hit, 3, replace=False)) + [int(np.abs(c["ref"]).argmax())]:
        e = np.zeros(a[0].size)
        e[k] = 1.0
        assert abs(diff(e.reshape(a[0].shape)) - c["ref"].reshape(-1)[k]) <= 1e-9 * np.abs(c["ref"]).max()


def test_bproj_is_the_transpose_of_the_emulated_forward(case):
    """sum_n w_n fwd(dV)_n = <bproj(w), dV> with both sides from the host-compiled kernels' math: the two marches share the
    samples and the trilinear weights, and differ only in the order of the fp32 sums."""
    c = case
    dV = np.random.default_rng(12).normal(size=c["vol"].shape).astype(np.float32)
    img = emu_deform.deform(dV, *dc.args(c)[1:])["out"].astype(np.float64)
    g = emu.deform_bproj(c["vol"].shape, *_bproj_args(c)).astype(np.float64)
    lhs = float((c["gout"].astype(np.float64) * img).sum())
    rhs = float((g * dV).sum())
    scale = float((np.abs(c["gout"]).astype(np.float64) * emu_deform.deform(np.abs(dV), *dc.args(c)[1:])["out"]).sum())
    assert lhs != 0 and abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


def test_zero_upstream_gradient_gives_exact_zeros(case):
    c = dict(case, gout=np.zeros_like(case["gout"]))
    got = emu.deform_bproj(c["vol"].shape, *_bproj_args(c))
    assert np.all(got == 0) and not np.signbit(got).any()


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    import ctypes

    from diffdrr_b200 import _lib
    lib = _lib.load()
    n = None
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    assert lib.b200drr_deform_bproj(4, 4, 4, n, n, n, n, 1, 2, 2, 2, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, p, 1, 2, 2, 2, n, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # no gout
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, n, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # no g_vol
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, q, 1, 2, 2, 2, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # alignment
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, p, 2, 2, 2, 2, p, p, 3, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # Bf
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, 1, 4, 2, 3, 0.5, 1e-8, 10, p, n) == -1   # H * W != N
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, 1, 4, 0, 0, 0.5, 1e-8, 1, p, n) == -1    # n_points
    assert lib.b200drr_deform_bproj(4, 0, 4, p, p, p, p, 1, 2, 2, 2, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # dims
    assert lib.b200drr_deform_bproj(4, 4, 4, p, p, p, p, 1, 1024, 1024, 512, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -2  # 2^31
