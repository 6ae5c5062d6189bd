"""The blended-rigid render's transpose in the density on the CPU: the B200_HD math of csrc/polyrigid_math.cuh (polyrigid_ray_bproj)
compiled for the host against the float64 backprojection of polyrigid_bproj_oracle, the oracle against differences of
polyrigid_oracle.fwd in the density (the render is linear in it, so these are exact up to rounding), the adjoint relation with the
emulated forward, and the C ABI's argument checks.  Runs without a GPU."""
import numpy as np
import pytest

import polyrigid_bproj_oracle as bo
import polyrigid_cases as pc
import polyrigid_oracle as po
import trilinear_cases as tc
from conftest import relerr
from hostemu import emu_polyrigid
from hostemu import emu_polyrigid_bproj as emu

FLOOR = 1e-4


def _bproj_args(c):
    return (c["src"], c["tgt"], c["raylen"], c["M"], c["weights"], c["n_points"], c["amin"], c["amax"], c["gout"])


@pytest.fixture(scope="module", params=sorted(pc.CASES))
def case(request):
    c = pc.CASES[request.param]()
    a = pc.args(c)
    c["ref"] = bo.bproj(*a[:6], c["gout"], *a[6:])
    c["r32"] = bo.bproj(*a[:6], c["gout"], *a[6:], dtype=np.float32)
    return c


def test_emulated_bproj_matches_fp64_oracle(case):
    c = case
    got = emu.polyrigid_bproj(c["vol"].shape, *_bproj_args(c))
    assert np.abs(c["ref"]).max() > 0
    assert relerr(got, c["ref"]) <= tc.tol(c["r32"], c["ref"], FLOOR)


def test_oracle_matches_differences_of_the_forward(case):
    """sum_n gout_n (fwd(V + dV) - fwd(V - dV))_n / 2 = <g_V, dV> along random directions and on single voxels, in float64."""
    c = case
    a = [np.asarray(x, np.float64) for x in pc.args(c)[:6]]
    gout = c["gout"].astype(np.float64)
    rng = np.random.default_rng(21)

    def diff(dV):
        plus = po.fwd(a[0] + dV, *a[1:], c["n_points"], c["amin"], c["amax"])
        minus = po.fwd(a[0] - dV, *a[1:], c["n_points"], c["amin"], c["amax"])
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
    dV = np.random.default_rng(22).normal(size=c["vol"].shape).astype(np.float32)
    rest = pc.args(c)[1:]
    img = emu_polyrigid.polyrigid(dV, *rest)["out"].astype(np.float64)
    g = emu.polyrigid_bproj(c["vol"].shape, *_bproj_args(c)).astype(np.float64)
    lhs = float((c["gout"].astype(np.float64) * img).sum())
    rhs = float((g * dV).sum())
    scale = float((np.abs(c["gout"]).astype(np.float64) * emu_polyrigid.polyrigid(np.abs(dV), *rest)["out"]).sum())
    assert lhs != 0 and abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


def test_zero_upstream_gradient_gives_exact_zeros(case):
    c = dict(case, gout=np.zeros_like(case["gout"]))
    got = emu.polyrigid_bproj(c["vol"].shape, *_bproj_args(c))
    assert np.all(got == 0) and not np.signbit(got).any()


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    import ctypes

    from diffdrr_b200 import _lib
    lib = _lib.load()
    f = lib.b200drr_polyrigid_bproj
    n = None
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    ok = (4, 4, 4, p, p, p, p, 1, 2, p, 2, 2, 2, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n)

    def call(**kw):
        a = list(ok)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return f(*a)

    assert f(4, 4, 4, n, n, n, n, 1, 2, n, 2, 2, 2, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert call(a13=n) == -1                # no gout
    assert call(a14=n) == -1                # no g_vol
    for i in (3, 4, 5, 6, 9, 22):           # src, tgt, raylen, M, the lattice, the range
        assert call(**{f"a{i}": n}) == -1, i
    assert call(a9=q) == -1                 # lattice alignment
    assert call(a7=2, a15=3) == -1          # Bm neither 1 nor B
    assert call(a8=0) == -1                 # K
    assert call(a17=2, a18=3) == -1         # H * W != N
    assert call(a21=1) == -1                # n_points
    assert call(a1=0) == -1                 # dims
    assert call(a11=0) == -1                # lattice dims
    assert call(a8=9) == -2                 # K > 8
    assert call(a10=1024, a11=1024, a12=512) == -2   # a lattice of 2^31 floats
    assert call(a8=9, a13=n) == -1          # EINVAL before EUNSUPPORTED
