"""The scaling-and-squaring exponential on the CPU: the B200_HD step and adjoint of csrc/svf_math.cuh compiled for the host (its
vector reductions plain adds) against the fp64 reference of svf_oracle.py, that reference's adjoint against central differences of
its own forward, the exact affine identity of trilinear squaring, the volume a twisted two-structure blend keeps, the SE(3) log the
log-Euclidean blend takes, and the C ABI's refusals.  Runs without a GPU."""
import ctypes

import numpy as np
import pytest
import scipy.linalg as sl
import torch

import svf_oracle as so
from hostemu import emu_svf as emu

# (D, g, Bf, displacement scale in voxels): anisotropic D / g, shared and per-pose fields, and fields large enough that many
# lookups land outside the node range and are clamped
CASES = {
    "aniso_shared": ((20, 13, 9), (6, 5, 4), 1, 2.0),
    "aniso_per_pose": ((17, 24, 11), (5, 7, 3), 3, 1.5),
    "outside": ((12, 12, 12), (4, 4, 4), 2, 8.0),
    "flat_axis": ((10, 8, 6), (5, 1, 3), 2, 2.0),   # one node along axis 1: the lookup is constant there
}
SCALES = [1.0 / 16, 1.0]


def _case(name, seed=0):
    D, g, Bf, amp = CASES[name]
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    return D, rng.normal(size=(Bf, *g, 3)) * amp, rng.normal(size=(Bf, *g, 3))


def _clamped_share(u, s, D):
    g = u.shape[1:4]
    q = np.stack(np.meshgrid(*[np.arange(n) for n in g], indexing="ij"), -1) + s * u * (np.array(g) / np.array(D))
    return np.mean((q < 0) | (q > np.array(g) - 1))


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_step_and_adjoint_match_fp64_reference(name, s):
    D, u, gp = _case(name)
    ref = so.square(torch.tensor(u), s, D).numpy()
    got, lane3 = emu.square(u, s, D)
    assert np.all(lane3 == 0)
    assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()
    gref = so.square_bwd(u, gp, s, D).numpy()
    gg, lane3 = emu.square_bwd(u, gp, s, D)
    assert np.all(lane3 == 0)
    # per node: one product with s, a 3 x 3 product with J, and up to 9 fp32 adds from the scatter
    assert np.abs(gg - gref).max() <= 2e-6 * np.abs(gref).max()


def test_cases_cover_what_they_claim():
    D, u, _ = _case("outside")
    assert _clamped_share(u, 1.0, D) > 0.2
    D, u, _ = _case("aniso_shared")
    assert 0 < _clamped_share(u, 1.0, D) < 0.5 and any(d % n for d, n in zip(D, u.shape[1:4]))
    assert _case("aniso_per_pose")[1].shape[0] > 1


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_adjoint_matches_central_differences(name, s):
    D, u, gp = _case(name)
    u, gp = torch.tensor(u), torch.tensor(gp)
    g = so.square_bwd(u, gp, s, D)
    rng = np.random.default_rng(1)
    for _ in range(3):
        d = torch.tensor(rng.normal(size=u.shape))
        h = 1e-6
        fd = ((so.square(u + h * d, s, D) - so.square(u - h * d, s, D)) * gp).sum() / (2 * h)
        assert abs(float((g * d).sum()) - float(fd)) <= 1e-6 * max(1.0, abs(float(fd)))


def test_exp_adjoint_is_the_adjoint_of_the_composition():
    D, u, gp = _case("aniso_per_pose")
    v = torch.tensor(u * 0.5, requires_grad=True)
    (so.exp(v, 4, D) * torch.tensor(gp)).sum().backward()
    g = so.exp_bwd(v.detach(), gp, 4, D)
    assert torch.allclose(g, v.grad, rtol=1e-10, atol=1e-12)


def _affine_case(steps):
    g = D = (32, 32, 32)
    c = np.full(3, 15.5)
    W = np.array([[0.0, -0.3, 0.1], [0.3, 0.0, -0.05], [-0.1, 0.05, 0.02]])   # a rotation by ~0.32 rad and a slight stretch
    L = np.concatenate([W, (-W @ c)[:, None]], 1)
    x = so.node_coords(g, D).numpy()
    v = (np.concatenate([x, np.ones(g + (1,))], -1) @ L.T)[None]
    inner = np.linalg.norm(x - c, axis=-1) <= 9.0
    return D, L, x, v, inner


@pytest.mark.parametrize("steps", [4, 8, 10])
def test_affine_velocity_gives_the_exact_affine_identity(steps):
    """v = L [x; 1] with one structure at weight 1: trilinear interpolation reproduces affine maps, so wherever the trajectories
    stay inside the lattice N squarings give ((I + L / 2^N)^(2^N) - I) [x; 1] exactly; the emulated fp32 steps match it to
    round-off at every node within 9 voxels of the centre."""
    D, L, x, v, inner = _affine_case(steps)
    ident = so.affine_identity(L, steps, torch.tensor(x)).numpy()
    ref = so.exp(torch.tensor(v), steps, D).numpy()[0]
    assert np.abs(ref - ident)[inner].max() <= 1e-11   # the fp64 reference: the identity holds there
    got = emu.exp(v, steps, D)[0]
    scale = np.abs(ident[inner]).max()
    assert np.abs(got - ident)[inner].max() <= 2e-6 * scale
    # and against the exact flow exp(L) the error falls ~4x per squaring
    E = sl.expm(np.vstack([L, np.zeros(4)]))
    exact = np.concatenate([x, np.ones(x.shape[:-1] + (1,))], -1) @ (E - np.eye(4))[:3].T
    err = np.abs(ident - exact)[inner].max()
    assert err <= 600.0 * 4.0**-steps   # 4.4e-4 voxel at N = 10


def _twist(theta):
    g = D = (32, 32, 32)
    c = np.full(3, 15.5)
    x = so.node_coords(g, D).numpy()
    w1 = 1.0 / (1.0 + np.exp(-(x[..., 0] - c[0]) / 2.0))   # two structures split along axis 0, a logistic of width 2
    xh = np.concatenate([x, np.ones(g + (1,))], -1)
    gens = []
    for t in (theta, -theta):
        W = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, -t], [0.0, t, 0.0]])   # a twist about axis 0 through the centre
        gens.append(np.concatenate([W, (-W @ c)[:, None]], 1))
    v = sum(w[..., None] * (xh @ L.T) for w, L in zip((w1, 1 - w1), gens))[None]
    lin = sum(w[..., None] * (xh @ sl.expm(np.vstack([L, np.zeros(4)]))[:3].T - x) for w, L in zip((w1, 1 - w1), gens))[None]
    near = (np.hypot(x[..., 1] - c[1], x[..., 2] - c[2]) <= 10.0)[1:-1, 1:-1, 1:-1]
    return D, v, lin, near


def test_twisted_blend_keeps_its_volume():
    """Two structures twisted +-1.2 rad about axis 0 on a 32^3 lattice (the voxel grid), split by a logistic weight of width 2.
    The log-Euclidean field (10 emulated squarings) has det grad phi in [0.83, 1.002] over the lattice's interior nodes and within
    2e-3 of 1 within 10 cells of the axis; the linear blend of the same weights and motions falls to cos^2(1.2) = 0.13 there
    (the candy wrapper)."""
    D, v, lin, near = _twist(1.2)
    det_le = so.jacobian_det(torch.tensor(emu.exp(v, 10, D), dtype=torch.float64), D).numpy()[0]
    det_lin = so.jacobian_det(torch.tensor(lin), D).numpy()[0]
    assert det_le.min() > 0
    assert np.abs(det_le[near] - 1).max() < 1e-2
    assert det_lin[near].min() < 0.5


def test_se3_log_inverts_the_exponential_with_a_finite_derivative_at_the_identity():
    from diffdrr_b200.pose import axis_angle_to_matrix
    from diffdrr_b200.svf import se3_log_matrix

    rng = np.random.default_rng(3)
    aa = torch.tensor(rng.normal(size=(4, 3)) * [[0.0], [1e-6], [0.5], [2.5]])
    X = torch.eye(4, dtype=torch.float64).repeat(4, 1, 1)
    X[:, :3, :3] = axis_angle_to_matrix(aa)
    X[:, :3, 3] = torch.tensor(rng.normal(size=(4, 3)) * 20)
    assert torch.allclose(torch.linalg.matrix_exp(se3_log_matrix(X)), X, atol=1e-10)
    assert torch.equal(se3_log_matrix(torch.eye(4, dtype=torch.float64)), torch.zeros(4, 4, dtype=torch.float64))

    def f(xi):   # the log along a twist path through X0: at xi = 0 the derivative must be the generator's
        return se3_log_matrix(torch.linalg.matrix_exp(_twist_matrix(xi)) @ X0)

    for X0 in (torch.eye(4, dtype=torch.float64), X[2]):
        xi = torch.zeros(6, dtype=torch.float64, requires_grad=True)
        J = torch.autograd.functional.jacobian(f, xi)
        assert torch.isfinite(J).all()
        h = 1e-6
        fd = torch.stack([(f(h * e) - f(-h * e)) / (2 * h) for e in torch.eye(6, dtype=torch.float64)], -1)
        assert torch.allclose(J, fd, atol=1e-7)
    xi = torch.zeros(6, dtype=torch.float64)
    X0 = torch.eye(4, dtype=torch.float64)
    Jid = torch.autograd.functional.jacobian(f, xi)
    assert torch.allclose(Jid, torch.stack([_twist_matrix(e) for e in torch.eye(6, dtype=torch.float64)], -1), atol=1e-12)


def _twist_matrix(xi):
    w, v = xi[:3], xi[3:]
    z = torch.zeros((), dtype=xi.dtype)
    top = torch.stack([torch.stack([z, -w[2], w[1], v[0]]), torch.stack([w[2], z, -w[0], v[1]]),
                       torch.stack([-w[1], w[0], z, v[2]])])
    return torch.cat([top, torch.zeros(1, 4, dtype=xi.dtype)])


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    from diffdrr_b200 import _lib

    lib = _lib.load()
    n = None
    buf = (ctypes.c_float * 64)()
    buf2 = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    p = ctypes.c_void_p((p.value + 15) // 16 * 16)
    o = ctypes.cast(buf2, ctypes.c_void_p)
    o = ctypes.c_void_p((o.value + 15) // 16 * 16)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    assert lib.b200drr_svf_square(n, n, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1
    assert lib.b200drr_svf_square_bwd(n, n, n, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1
    assert lib.b200drr_svf_square(p, o, 0, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # Bf
    assert lib.b200drr_svf_square(p, o, 1, 2, 0, 2, 4, 4, 4, 1.0, n) == -1     # empty lattice
    assert lib.b200drr_svf_square(p, o, 1, 2, 2, 2, 4, -4, 4, 1.0, n) == -1    # volume
    assert lib.b200drr_svf_square(p, o, 1, 2, 2, 2, 4, 4, 4, 0.0, n) == -1     # scale
    assert lib.b200drr_svf_square(q, o, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # alignment
    assert lib.b200drr_svf_square(p, p, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # in place
    assert lib.b200drr_svf_square_bwd(p, o, p, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1   # gin aliases the field
    assert lib.b200drr_svf_square_bwd(p, q, o, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1   # gout alignment
    assert lib.b200drr_svf_square(p, o, 1, 1024, 1024, 512, 4, 4, 4, 1.0, n) == -2  # 2^31 floats
