"""The blended-rigid (skinned) march on the CPU: the B200_HD math of csrc/polyrigid_math.cuh compiled for the host against the
fp64 reference of polyrigid_oracle.py, the reference's backward against central differences of its own fp64 forward, and the three
identities that tie the march to the Trilinear renderer.  Runs without a GPU."""
import numpy as np
import pytest

import polyrigid_cases as pc
import polyrigid_oracle as po
import trilinear_cases as tc
from conftest import relerr
from hostemu import emu_polyrigid as emu

FLOOR = 1e-4


@pytest.fixture(scope="module", params=sorted(pc.CASES))
def case(request):
    c = pc.CASES[request.param]()
    c["ref"] = po.fwd(*pc.args(c))
    c["gref"] = po.bwd(*pc.args(c)[:6], c["gout"], *pc.args(c)[6:])
    c["g32"] = po.bwd(*pc.args(c)[:6], c["gout"], *pc.args(c)[6:], dtype=np.float32)
    return c


@pytest.mark.parametrize("packed", [False, True])
def test_emulated_march_matches_fp64_reference(case, packed):
    c = case
    got = emu.polyrigid(*pc.args(c), gout=c["gout"], packed=packed)
    assert np.abs(c["ref"]).max() > 0
    assert relerr(got["out"], c["ref"]) <= 1e-4
    ref, r32 = c["gref"], c["g32"]
    assert relerr(got["g_raylen"], ref["g_raylen"]) <= tc.tol(r32["g_raylen"], ref["g_raylen"], FLOOR)
    smooth = slice(None) if c["kinks"] is None else ~c["kinks"]   # a ray on an integer plane has a one-sided derivative
    assert relerr(got["g_tgt"][:, smooth], ref["g_tgt"][:, smooth]) <= tc.tol(r32["g_tgt"][:, smooth], ref["g_tgt"][:, smooth], FLOOR)
    if c["kinks"] is not None:
        return   # the sums over rays below include the kink rays
    for key in ("g_src", "g_M"):
        assert np.abs(ref[key]).max() > 0
        assert relerr(got[key], ref[key]) <= tc.tol(r32[key], ref[key], FLOOR), key
    scale = tc.alpha_scale(ref["g_raylen"], c["raylen"], c["amin"], c["amax"])
    for key in ("g_alphamin", "g_alphamax"):
        assert abs(got[key] - ref[key]) / scale <= tc.tol(r32[key], ref[key], FLOOR, scale=scale), key


def test_plain_and_packed_gathers_agree_bitwise(case):
    a = emu.polyrigid(*pc.args(case), gout=case["gout"], packed=False)
    b = emu.polyrigid(*pc.args(case), gout=case["gout"], packed=True)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


@pytest.mark.parametrize("name", ["k3_per_pose", "k8_shared", "source_inside"])
def test_reference_backward_matches_central_differences(name):
    """d sum(gout * I) along random directions of M, s, t and the range ends, by central differences of the fp64 forward."""
    c = pc.CASES[name]()
    rng = np.random.default_rng(11)
    a = [np.asarray(x, np.float64) for x in pc.args(c)[:6]]
    g = po.bwd(*a, c["gout"], c["n_points"], c["amin"], c["amax"])

    def loss(src=a[1], tgt=a[2], M=a[4], amin=c["amin"], amax=c["amax"]):
        return float((c["gout"] * po.fwd(a[0], src, tgt, a[3], M, a[5], c["n_points"], amin, amax)).sum())

    def check(analytic, f, h):
        fd = (f(h) - f(-h)) / (2 * h)
        assert abs(fd - analytic) <= 1e-6 * max(abs(analytic), abs(fd)) + 1e-9 * abs(loss()), (fd, analytic)

    dM, ds, dt = rng.normal(size=a[4].shape), rng.normal(size=a[1].shape), rng.normal(size=a[2].shape)
    check((g["g_M"] * dM).sum(), lambda h: loss(M=a[4] + h * dM), 1e-6)
    check((g["g_src"] * ds).sum(), lambda h: loss(src=a[1] + h * ds), 1e-5)
    check((g["g_tgt"] * dt).sum(), lambda h: loss(tgt=a[2] + h * dt), 1e-4)
    check(g["g_alphamin"], lambda h: loss(amin=c["amin"] + h), 1e-8)
    check(g["g_alphamax"], lambda h: loss(amax=c["amax"] + h), 1e-8)


def test_identity_motions_are_the_trilinear_march_bitwise(case):
    c = case
    M = np.broadcast_to(np.eye(3, 4, dtype=np.float32), c["M"].shape)
    got = emu.polyrigid(c["vol"], c["src"], c["tgt"], c["raylen"], M, c["weights"], c["n_points"], c["amin"], c["amax"])["out"]
    assert np.array_equal(got, emu.trilinear(c["vol"], c["src"], c["tgt"], c["raylen"], c["n_points"], c["amin"], c["amax"]))


def test_zero_weights_are_the_trilinear_march_bitwise(case):
    c = case
    got = emu.polyrigid(c["vol"], c["src"], c["tgt"], c["raylen"], c["M"], np.zeros_like(c["weights"]), c["n_points"], c["amin"],
                        c["amax"])["out"]
    assert np.array_equal(got, emu.trilinear(c["vol"], c["src"], c["tgt"], c["raylen"], c["n_points"], c["amin"], c["amax"]))


def test_one_structure_with_unit_weight_is_the_trilinear_march_on_the_moved_rays():
    """K = 1, w = 1: y = M x, so the image is the Trilinear renderer's on the rays (M s, M t) with the same explicit range (raylen
    is an input and stays).  A lattice of ones is 1 up to half a lattice cell from the volume's faces and falls to 0 beyond, so the
    density is cut to a core that no sample with w < 1 can reach (the maps move a point by less than 6 voxels)."""
    c = pc.CASES["k1_shared"]()
    M = c["M"].astype(np.float64)[0, 0]
    core = np.zeros_like(c["vol"])
    core[9:-9, 9:-9, 9:-9] = c["vol"][9:-9, 9:-9, 9:-9]
    c["vol"] = core
    amin, amax = c["amin"], c["amax"]
    got = emu.polyrigid(c["vol"], c["src"], c["tgt"], c["raylen"], c["M"], np.ones_like(c["weights"]), c["n_points"], amin, amax)["out"]
    src = c["src"].astype(np.float64) @ M[:, :3].T + M[:, 3]
    tgt = c["tgt"].astype(np.float64) @ M[:, :3].T + M[:, 3]
    want = emu.trilinear(c["vol"], src, tgt, c["raylen"], c["n_points"], amin, amax)
    assert np.abs(want).max() > 0 and relerr(got, want) <= 1e-5


def test_cases_cover_what_they_claim():
    c = pc.CASES["pushed_out"]()
    D = np.asarray(c["vol"].shape, np.float64)
    centre = (D - 1) / 2
    moved = c["M"][0, 0].astype(np.float64) @ np.append(centre, 1.0)
    assert np.any((moved < -1) | (moved > D))                      # the volume centre is pulled from outside the volume
    c = pc.CASES["source_inside"]()
    assert np.all((c["src"] > 0) & (c["src"] < D - 1))
    c = pc.CASES["k3_per_pose"]()
    assert c["M"].shape[0] == c["src"].shape[0] > 1 and any(d % g for d, g in zip(c["vol"].shape, c["weights"].shape[1:]))
    c = pc.CASES["k8_per_pose_ragged"]()
    assert c["H"] == 0 and c["tgt"].shape[1] % 128 != 0 and c["M"].shape[1] == 8
    for name in pc.CASES:
        w = pc.CASES[name]()["weights"]
        assert w.min() >= 0 and w.sum(0).max() <= 1 + 1e-5


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    import ctypes

    from diffdrr_b200 import _lib
    lib = _lib.load()
    n = None
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.b200drr_polyrigid_fwd(n, n, 4, 4, 4, n, n, n, n, 1, 1, n, 2, 2, 2, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_polyrigid_bwd(n, n, 4, 4, 4, n, n, n, n, 1, 1, n, 2, 2, 2, n, n, n, n, n, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, n) == -1
    assert lib.b200drr_polyrigid_fwd_v16(p, n, 7, 4, 4, 4, p, p, p, p, 1, 1, p, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # vol_type
    assert lib.b200drr_polyrigid_fwd(p, p, 4, 4, 4, p, p, p, p, 1, 1, p, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # vol AND packed
    assert lib.b200drr_polyrigid_fwd(p, n, 4, 4, 4, p, p, p, p, 2, 1, p, 2, 2, 2, p, 3, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -1   # Bm not in {1, B}
    assert lib.b200drr_polyrigid_fwd(p, n, 4, 4, 4, p, p, p, p, 1, 1, p, 2, 2, 2, p, 1, 4, 2, 3, 0.5, 1e-8, 10, p, n) == -1   # H * W != N
    assert lib.b200drr_polyrigid_fwd(p, n, 4, 4, 4, p, p, p, p, 1, 9, p, 2, 2, 2, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, n) == -2   # K > 8
    assert lib.b200drr_polyrigid_pack_weights(p, 9, 2, 2, 2, p, n) == -2 and lib.b200drr_polyrigid_pack_weights(n, 3, 2, 2, 2, p, n) == -1
    assert lib.b200drr_polyrigid_weight_floats(3, 5, 6, 7) == 5 * 6 * 7 * 4 and lib.b200drr_polyrigid_weight_floats(5, 5, 6, 7) == 5 * 6 * 7 * 8
    assert lib.b200drr_polyrigid_scratch_floats(2, 300, 0, 0, 3) == 2 * 3 * (4 * 12 + 5)        # 128 rays per CTA
    assert lib.b200drr_polyrigid_scratch_floats(2, 20 * 17, 20, 17, 8) == 2 * 2 * 3 * (8 * 12 + 5)   # 16 x 8 pixel tiles
