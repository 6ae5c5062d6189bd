"""The deformable march on the CPU: the B200_HD math of csrc/deform_math.cuh compiled for the host (its field scatter a plain add)
against the fp64 reference of deform_oracle.py, the reference's backward against central differences of its own fp64 forward, the
zero-field identity with the Trilinear march, and the C ABI's refusals.  Runs without a GPU."""
import numpy as np
import pytest

import deform_cases as dc
import deform_oracle as do
import trilinear_cases as tc
from conftest import relerr
from hostemu import emu_deform as emu
from hostemu import emu_polyrigid

FLOOR = 1e-4


@pytest.fixture(scope="module", params=sorted(dc.CASES))
def case(request):
    c = dc.CASES[request.param]()
    c["ref"] = do.fwd(*dc.args(c))
    c["gref"] = do.bwd(*dc.args(c)[:5], c["gout"], *dc.args(c)[5:])
    c["g32"] = do.bwd(*dc.args(c)[:5], c["gout"], *dc.args(c)[5:], dtype=np.float32)
    return c


@pytest.mark.parametrize("packed", [False, True])
def test_emulated_march_matches_fp64_reference(case, packed):
    c = case
    got = emu.deform(*dc.args(c), gout=c["gout"], packed=packed)
    assert np.abs(c["ref"]).max() > 0
    assert relerr(got["out"], c["ref"]) <= 1e-4
    ref, r32 = c["gref"], c["g32"]
    assert relerr(got["g_raylen"], ref["g_raylen"]) <= tc.tol(r32["g_raylen"], ref["g_raylen"], FLOOR)
    assert np.all(got["lane3"] == 0)
    smooth = slice(None) if c["kinks"] is None else ~c["kinks"]   # a ray on an integer plane has a one-sided derivative
    assert relerr(got["g_tgt"][:, smooth], ref["g_tgt"][:, smooth]) <= tc.tol(r32["g_tgt"][:, smooth], ref["g_tgt"][:, smooth], FLOOR)
    if c["kinks"] is not None:
        return   # the sums over rays below include the kink rays
    for key in ("g_src", "g_U"):
        assert np.abs(ref[key]).max() > 0
        assert relerr(got[key], ref[key]) <= tc.tol(r32[key], ref[key], FLOOR), key
    scale = tc.alpha_scale(ref["g_raylen"], c["raylen"], c["amin"], c["amax"])
    for key in ("g_alphamin", "g_alphamax"):
        assert abs(got[key] - ref[key]) / scale <= tc.tol(r32[key], ref[key], FLOOR, scale=scale), key


def test_plain_and_packed_gathers_agree_bitwise(case):
    a = emu.deform(*dc.args(case), gout=case["gout"], packed=False)
    b = emu.deform(*dc.args(case), gout=case["gout"], packed=True)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_skipping_the_scatter_changes_nothing_else(case):
    a = emu.deform(*dc.args(case), gout=case["gout"])
    b = emu.deform(*dc.args(case), gout=case["gout"], scatter=False)
    assert b["g_U"] is None and not b["flushes"].any()
    for key in ("out", "g_src", "g_tgt", "g_raylen", "g_alphamin", "g_alphamax"):
        assert np.array_equal(a[key], b[key]), key


def test_run_length_scatter_flushes_once_per_lattice_cell(case):
    """A ray flushes its registers once per run of samples in one lattice cell: at most once per sample, and far fewer on a coarse
    lattice (a straight ray crosses at most g0 + g1 + g2 cells)."""
    c = case
    got = emu.deform(*dc.args(c), gout=c["gout"])
    assert got["flushes"].max() > 0 and got["flushes"].max() <= c["n_points"]
    if c["name"] in ("shared", "per_pose", "source_inside"):
        assert got["flushes"].max() <= sum(c["U"].shape[2:])


@pytest.mark.parametrize("name", ["per_pose", "out_and_back", "source_inside"])
def test_reference_backward_matches_central_differences(name):
    """d sum(gout * I) along random directions of U, s, t, a few single field nodes and the range ends, by central differences
    of the fp64 forward."""
    c = dc.CASES[name]()
    rng = np.random.default_rng(11)
    a = [np.asarray(x, np.float64) for x in dc.args(c)[:5]]
    g = do.bwd(*a, c["gout"], c["n_points"], c["amin"], c["amax"])

    def loss(src=a[1], tgt=a[2], U=a[4], amin=c["amin"], amax=c["amax"]):
        return float((c["gout"] * do.fwd(a[0], src, tgt, a[3], U, c["n_points"], amin, amax)).sum())

    def check(analytic, f, h):
        fd = (f(h) - f(-h)) / (2 * h)
        assert abs(fd - analytic) <= 1e-6 * max(abs(analytic), abs(fd)) + 1e-9 * abs(loss()), (fd, analytic)

    dU, ds, dt = rng.normal(size=a[4].shape), rng.normal(size=a[1].shape), rng.normal(size=a[2].shape)
    check((g["g_U"] * dU).sum(), lambda h: loss(U=a[4] + h * dU), 1e-6)
    big = np.argsort(np.abs(g["g_U"]).ravel())[-3:]      # the nodes with the largest gradients, one at a time
    for i in big:
        e = np.zeros(a[4].size)
        e[i] = 1.0
        check(g["g_U"].ravel()[i], lambda h: loss(U=a[4] + h * e.reshape(a[4].shape)), 1e-5)
    check((g["g_src"] * ds).sum(), lambda h: loss(src=a[1] + h * ds), 2e-6)
    check((g["g_tgt"] * dt).sum(), lambda h: loss(tgt=a[2] + h * dt), 1e-4)
    check(g["g_alphamin"], lambda h: loss(amin=c["amin"] + h), 1e-8)
    check(g["g_alphamax"], lambda h: loss(amax=c["amax"] + h), 1e-8)


def test_zero_field_is_the_trilinear_march_bitwise(case):
    c = case
    got = emu.deform(c["vol"], c["src"], c["tgt"], c["raylen"], np.zeros_like(c["U"]), c["n_points"], c["amin"], c["amax"])["out"]
    assert np.array_equal(got, emu_polyrigid.trilinear(c["vol"], c["src"], c["tgt"], c["raylen"], c["n_points"], c["amin"], c["amax"]))


def test_constant_field_is_the_trilinear_march_on_shifted_rays():
    """u = c everywhere the lattice reaches: y = x + c, so inside the lattice's support the image is the Trilinear renderer's on
    the rays (s + c, t + c).  The density is cut to a core that no sample outside the support can reach."""
    c = dc.CASES["shared"]()
    shift = np.array([1.25, -2.5, 0.75], np.float32)
    U = np.broadcast_to(shift[None, :, None, None, None], c["U"].shape).copy()
    core = np.zeros_like(c["vol"])
    core[9:-9, 9:-9, 9:-9] = c["vol"][9:-9, 9:-9, 9:-9]
    amin, amax = c["amin"], c["amax"]
    got = emu.deform(core, c["src"], c["tgt"], c["raylen"], U, c["n_points"], amin, amax)["out"]
    want = emu_polyrigid.trilinear(core, c["src"] + shift, c["tgt"] + shift, c["raylen"], c["n_points"], amin, amax)
    assert np.abs(want).max() > 0 and relerr(got, want) <= 1e-5


def test_cases_cover_what_they_claim():
    c = dc.CASES["out_and_back"]()
    q = do._march(c["vol"], c["src"], c["tgt"], c["U"], c["n_points"], c["amin"], c["amax"], 0.5, 1e-8, np.float64)
    D = np.asarray(c["vol"].shape)
    inside_y = np.all((q["y"] > -1) & (q["y"] < D), -1)          # (B, N, P)
    flips = np.abs(np.diff(inside_y.astype(int), axis=-1)).sum(-1)
    assert np.any(flips >= 3)                                   # some ray's pulled-back samples leave and re-enter the volume
    c = dc.CASES["source_inside"]()
    assert np.all((c["src"] > 0) & (c["src"] < D - 1))
    c = dc.CASES["per_pose"]()
    assert c["U"].shape[0] == c["src"].shape[0] > 1 and any(d % g for d, g in zip(c["vol"].shape, c["U"].shape[2:]))
    c = dc.CASES["per_pose_ragged"]()
    assert c["H"] == 0 and c["tgt"].shape[1] % 128 != 0


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    import ctypes

    from diffdrr_b200 import _lib
    lib = _lib.load()
    n = None
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    assert lib.b200drr_deform_fwd(n, n, 4, 4, 4, n, n, n, n, 1, 2, 2, 2, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_deform_bwd(n, n, 4, 4, 4, n, n, n, n, 1, 2, 2, 2, n, n, n, n, n, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_deform_fwd_v16(p, n, 7, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # vol_type
    assert lib.b200drr_deform_fwd(p, p, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # vol AND packed
    assert lib.b200drr_deform_fwd(p, n, 4, 4, 4, p, p, p, p, 2, 2, 2, 2, p, 3, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # Bf not in {1, B}
    assert lib.b200drr_deform_fwd(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, 1, 4, 2, 3, 0.5, 1e-8, 10, p, n) == -1   # H * W != N
    assert lib.b200drr_deform_fwd(p, n, 4, 4, 4, p, p, p, q, 1, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # field alignment
    assert lib.b200drr_deform_fwd(p, n, 4, 4, 4, p, p, p, p, 1, 2, 0, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # empty lattice
    assert lib.b200drr_deform_fwd(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 1, p, n) == -1    # n_points < 2
    assert lib.b200drr_deform_bwd(p, n, 4, 4, 4, p, p, p, p, 1, 2, 2, 2, p, p, p, p, q, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1  # g_field
    assert lib.b200drr_deform_fwd(p, n, 4, 4, 4, p, p, p, p, 1, 1024, 1024, 512, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -2  # 2^31 floats
    assert lib.b200drr_deform_scratch_floats(2, 300, 0, 0) == 2 * 3 * 5            # 128 rays per CTA
    assert lib.b200drr_deform_scratch_floats(2, 20 * 17, 20, 17) == 2 * 2 * 3 * 5   # 16 x 8 pixel tiles
    assert lib.b200drr_deform_scratch_floats(2, 300, 7, 0) == 0
