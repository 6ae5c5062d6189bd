"""The tangent of the scaling-and-squaring exponential on the CPU: the fp64 closed form of svf_jvp_oracle.py against
torch.func.jvp of svf_oracle's exponential and against central differences away from cell boundaries and clamp edges; the B200_HD
tangent step of csrc/svf_math.cuh compiled for the host against that reference on test_svf_cpu.py's cases, its primal output
against the emulated forward bit for bit, exact zeros for a zero tangent, the transpose relation with the emulated adjoint per step
and through ten levels, and the C ABI's refusals.  Runs without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

import svf_jvp_oracle as sj
import svf_oracle as so
from hostemu import emu_svf as emu
from hostemu import emu_svf_jvp as emu_jvp
from test_svf_cpu import CASES, SCALES, _case


def _tangent(name, seed=5):
    D, u, _ = _case(name)
    return np.random.default_rng(seed + sum(map(ord, name))).normal(size=u.shape)


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_tangent_is_the_forward_derivative(name):
    """The closed form against torch.func.jvp of svf_oracle's step, per scale and through four squarings."""
    D, u, _ = _case(name)
    u, t = torch.tensor(u), torch.tensor(_tangent(name))
    for s in SCALES:
        _, want = torch.func.jvp(lambda x: so.square(x, s, D), (u,), (t,))
        got = sj.square_jvp(u, t, s, D)
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12 * float(want.abs().max()))
    v = 0.5 * u
    want_u, want_t = torch.func.jvp(lambda x: so.exp(x, 4, D), (v,), (t,))
    got_u, got_t = sj.exp_jvp(v, t, 4, D)
    assert torch.equal(got_u, so.exp(v, 4, D))
    assert torch.allclose(got_u, want_u, rtol=0, atol=1e-12 * float(want_u.abs().max()))
    assert torch.allclose(got_t, want_t, rtol=1e-10, atol=1e-10 * float(want_t.abs().max()))


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_tangent_matches_central_differences(name, s):
    """Per node, away from cell boundaries and clamp edges (the lookup is only piecewise smooth): h = 1e-6 in fp64."""
    D, u, _ = _case(name)
    u, t = torch.tensor(u), torch.tensor(_tangent(name))
    g = u.shape[1:4]
    sc = torch.tensor([g[a] / D[a] for a in range(3)], dtype=u.dtype)
    idx = torch.stack(torch.meshgrid(*[torch.arange(n, dtype=u.dtype) for n in g], indexing="ij"), -1)
    q = idx + s * u * sc
    qd = s * t * sc   # dq along t
    near = torch.zeros(q.shape[:-1], dtype=torch.bool)
    for a in range(3):
        if g[a] > 1:   # an axis of one node has no kink: its lookup is constant
            near |= ((q[..., a] - q[..., a].round()).abs() <= 1e-4 + 1e-6 * qd[..., a].abs())
    h = 1e-6
    fd = (so.square(u + h * t, s, D) - so.square(u - h * t, s, D)) / (2 * h)
    got = sj.square_jvp(u, t, s, D)
    smooth = ~near
    assert smooth.float().mean() > 0.9
    assert float((got - fd)[smooth].abs().max()) <= 1e-6 * max(1.0, float(fd.abs().max()))


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_tangent_matches_fp64_reference_and_its_primal_is_the_step(name, s):
    D, u, _ = _case(name)
    t = _tangent(name)
    ref = sj.square_jvp(u, t, s, D).numpy()
    got, lane3, out = emu_jvp.square_jvp(u, t, s, D)
    assert np.all(lane3 == 0)
    # per node: the step's 3 x 3 product with J, one trilinear lookup of t and two adds
    assert np.abs(got - ref).max() <= 2e-6 * np.abs(ref).max()
    fwd, fwd3 = emu.square(u, s, D)
    assert np.array_equal(out[..., :3], fwd) and np.array_equal(out[..., 3], fwd3)
    alone = emu_jvp.square_jvp(u, t, s, D, primal=False)
    assert np.array_equal(alone[0], got) and alone[2] is None


@pytest.mark.parametrize("name", sorted(CASES))
def test_zero_tangent_gives_exact_zeros(name):
    D, u, _ = _case(name)
    for s in SCALES:
        got, lane3, _ = emu_jvp.square_jvp(u, np.zeros_like(u), s, D)
        assert not np.any(got) and not np.any(lane3)


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_exp_tangent_matches_fp64_reference(name):
    D, u, _ = _case(name)
    v, t = 0.5 * u, _tangent(name)
    ref_u, ref_t = sj.exp_jvp(v, t, 4, D)
    got_u, got_t = emu_jvp.exp_jvp(v, t, 4, D)
    assert np.array_equal(got_u, emu.exp(v, 4, D))
    assert np.abs(got_t - ref_t.numpy()).max() <= 2e-5 * np.abs(ref_t.numpy()).max()


def _dot(a, b):
    return float((np.asarray(a, np.float64) * np.asarray(b, np.float64)).sum())


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", sorted(CASES))
def test_tangent_is_the_transpose_of_the_emulated_adjoint(name, s):
    """<w, J t> = <J^T w, t> with J^T the emulated b200drr_svf_square_bwd."""
    D, u, w = _case(name)
    t = _tangent(name)
    jt = emu_jvp.square_jvp(u, t, s, D, primal=False)[0]
    jtw = emu.square_bwd(u, w, s, D)[0]
    lhs, rhs = _dot(w, jt), _dot(jtw, t)
    assert lhs != 0 and abs(lhs - rhs) <= 1e-5 * abs(rhs), (lhs, rhs)


@pytest.mark.parametrize("name", sorted(CASES))
def test_tangent_chain_is_the_transpose_of_the_adjoint_chain(name):
    """The same relation through ten squarings over one set of emulated levels, as the velocity LM chains them."""
    D, u, w = _case(name)
    steps = 10
    levels = [0.5 * u.astype(np.float32)]
    for k in range(steps - 1):
        levels.append(emu.square(levels[-1], 2.0**-steps if k == 0 else 1.0, D)[0])
    t = _tangent(name).astype(np.float32)
    jt = t
    for k in range(steps):
        jt = emu_jvp.square_jvp(levels[k], jt, 2.0**-steps if k == 0 else 1.0, D, primal=False)[0]
    g = w.astype(np.float32)
    for k in reversed(range(steps)):
        g = emu.square_bwd(levels[k], g, 2.0**-steps if k == 0 else 1.0, D)[0]
    lhs, rhs = _dot(w, jt), _dot(g, t)
    assert lhs != 0 and abs(lhs - rhs) <= 1e-5 * abs(rhs), (lhs, rhs)


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    from diffdrr_b200 import _lib

    lib = _lib.load()
    n = None
    bufs = [(ctypes.c_float * 64)() for _ in range(4)]
    p, t, o, r = (ctypes.c_void_p((ctypes.cast(b, ctypes.c_void_p).value + 15) // 16 * 16) for b in bufs)
    q = ctypes.c_void_p(p.value + 4)   # not 16-byte aligned
    jvp = lib.b200drr_svf_square_jvp
    assert jvp(n, t, o, r, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # field
    assert jvp(p, n, o, r, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # tangent
    assert jvp(p, t, n, r, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # tout
    assert jvp(p, t, o, r, 0, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # Bf
    assert jvp(p, t, o, r, 1, 2, 0, 2, 4, 4, 4, 1.0, n) == -1     # empty lattice
    assert jvp(p, t, o, r, 1, 2, 2, 2, 4, -4, 4, 1.0, n) == -1    # volume
    assert jvp(p, t, o, r, 1, 2, 2, 2, 4, 4, 4, 0.0, n) == -1     # scale
    assert jvp(q, t, o, r, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # field alignment
    assert jvp(p, q, o, r, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # tangent alignment
    assert jvp(p, t, q, r, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # tout alignment
    assert jvp(p, t, o, q, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1     # out alignment
    for tout, out in ((p, r), (t, r), (o, p), (o, t), (o, o)):      # aliasing
        assert jvp(p, t, tout, out, 1, 2, 2, 2, 4, 4, 4, 1.0, n) == -1
    assert jvp(p, t, o, r, 1, 1024, 1024, 512, 4, 4, 4, 1.0, n) == -2   # 2^31 floats
    assert jvp(p, t, o, n, 1, 1024, 1024, 512, 4, 4, 4, 1.0, n) == -2
