"""The log-Euclidean blended-rigid motion Jacobian and its Levenberg-Marquardt on the GPU (DRR.polyrigid_jacobian(blend=
"log_euclidean"), PolyrigidLevenbergMarquardt(blend="log_euclidean"); DESIGN.md 6p): b200drr_svf_square_tangents slice by slice
against b200drr_svf_square_jvp (bit for bit) and the fp64 closed form, b200drr_deform_jac column by column against the composition
of exp_velocity's tangent chain and b200drr_deform_jvp, its image against render_polyrigid bit for bit, its transpose against
autograd, one column against an fp64 central difference, the normal equations, and the registration: monotone, free of host syncs,
and its convergence on the two-structure scene."""
import numpy as np
import pytest
import torch

import deform_oracle as do
import svf_jvp_oracle as sj
import svf_oracle as so
import trilinear_cases as tc
from conftest import relerr
from diffdrr_b200 import NormalizedCrossCorrelation2d, PolyrigidLevenbergMarquardt, synthetic
from diffdrr_b200 import _lib, svf
from diffdrr_b200 import polyrigid as pr
from diffdrr_b200.deform import _marches, field_jvp
from diffdrr_b200.pose import convert
from diffdrr_b200.registration import ncc_normal_structures_equations
from diffdrr_b200.renderers import _ptr, _stream
from diffdrr_b200.structures import _rigid_inverse, apply_increments, se3_exp
from test_gpu_polyrigid_lm import DIMS, KW, _scene, _twists, _two_structures
from test_gpu_structures_lm import _about, _dense, _moved, registration_errors

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LE = dict(blend="log_euclidean", steps=8)


def _weights(K, g=(12, 14, 10), seed=0):
    """K smooth bumps on the lattice, scaled to sum to at most 1 (any K up to 8, unlike the three labels of _scene)."""
    rng = np.random.default_rng(seed)
    x = np.stack(np.meshgrid(*[(np.arange(n) + 0.5) / n for n in g], indexing="ij"), -1)
    w = np.stack([np.exp(-((x - rng.uniform(0.25, 0.75, 3)) ** 2).sum(-1) / 0.03) for _ in range(K)])
    w[w < 1e-3] = 0.0
    return torch.from_numpy((w / np.maximum(w.sum(0), 1.0)).astype(np.float32)).to(DEV)


def test_tangent_step_slices_are_the_single_tangent_step_bitwise():
    lib = _lib.load()
    g, P, D = (9, 11, 7), 13, DIMS
    gen = torch.Generator().manual_seed(0)
    u = torch.nn.functional.pad(3.0 * torch.randn(2, *g, 3, generator=gen), (0, 1)).to(DEV).contiguous()
    T = torch.nn.functional.pad(torch.randn(2, *g, P, 3, generator=gen), (0, 1)).to(DEV).contiguous()
    for s in (1.0 / 256, 1.0):
        tout, out = torch.empty_like(T), torch.empty_like(u)
        _lib.check(lib.b200drr_svf_square_tangents(_ptr(u), _ptr(T), _ptr(tout), _ptr(out), 2, P, *g, *D, s, _stream()), "tangents")
        again = torch.empty_like(T)
        _lib.check(lib.b200drr_svf_square_tangents(_ptr(u), _ptr(T), _ptr(again), None, 2, P, *g, *D, s, _stream()), "tangents")
        assert torch.equal(tout, again)
        prim = torch.empty_like(u)
        _lib.check(lib.b200drr_svf_square(_ptr(u), _ptr(prim), 2, *g, *D, s, _stream()), "square")
        assert torch.equal(out, prim)
        for p in range(P):
            Tp = T[..., p, :].contiguous()
            one = torch.empty_like(u)
            _lib.check(lib.b200drr_svf_square_jvp(_ptr(u), _ptr(Tp), _ptr(one), None, 2, *g, *D, s, _stream()), "jvp")
            assert torch.equal(tout[..., p, :], one), p
            ref = sj.square_jvp(u[..., :3].double().cpu(), Tp[..., :3].double().cpu(), s, D)
            assert relerr(tout[..., p, :3].cpu().numpy(), ref.numpy()) <= 2e-6


def _setup(drr, W, rot, xyz, X, steps, n_points):
    """The composition's pieces in voxel units: (levels, exp(v), the 6K velocity tangents, the rays of the one march)."""
    dims = tuple(drr.density.shape)
    v = svf.polyrigid_velocity(drr, X, W)
    levels, U = svf.square_chain(v, steps, dims)
    T0 = svf.velocity_tangents(drr, X, W, pr.polyrigid_pivots(drr, W))
    source, [(tgt, lens, arange, grid)] = _marches(drr, (rot, xyz), rot.shape[0], KW["parameterization"], KW["convention"], False,
                                                   None, None, None)
    return v, levels, U, T0, (source, tgt, lens, arange, grid)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("per_pose", [False, True])
def test_every_column_is_the_composition_of_existing_pieces(per_pose, K, dtype):
    """J[:, k, ..., i] against exp_velocity's tangent chain (square_chain_jvp) along velocity tangent p = 6k + i, marched by
    b200drr_deform_jvp; img against render_polyrigid(blend="log_euclidean") bit for bit, and the footprints hold J."""
    _, drr, _ = _scene(H=24)
    if dtype != torch.float32:
        drr.density = drr.density.to(dtype)
    W = _weights(K, seed=K)
    B = 2
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(B, seed=1))
    X = se3_exp(_twists(K, B if per_pose else None, seed=2)).float()
    img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=120, return_footprints=True, **LE, **KW)
    with torch.no_grad():
        ref = drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=120, **LE, **KW)
        assert torch.equal(img, ref)
        again = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=120, return_footprints=True, **LE, **KW)
        assert torch.equal(again[1], J) and torch.equal(again[2], rects)
        v, levels, U, T0, (source, tgt, lens, arange, grid) = _setup(drr, W, rot, xyz, X, LE["steps"], 120)
        packed = drr.renderer._packed_volume(drr.density)
        worst = 0.0
        for p in range(6 * K):
            _, Tp = svf.square_chain_jvp(levels, T0[..., p, :].contiguous(), tuple(drr.density.shape))
            col = field_jvp(drr, packed, source, tgt, lens, U, Tp, arange, 120, grid).view(B, 24, 24)
            got = J[:, p // 6, ..., p % 6]
            scale = float(col.abs().max())
            if scale > 0:
                worst = max(worst, float((got - col).abs().max()) / scale)
            else:
                assert not got.any()
        print(f"K={K} per_pose={per_pose} {dtype}: worst column error {worst:.2e} of the column's max-abs")
        assert worst <= 1e-4
    Jr = J.reshape(B, K, 24, 24, 6)
    for b in range(B):
        for k in range(K):
            w0, w1, h0, h1 = rects[b, k].tolist()
            mask = torch.ones(24, 24, dtype=torch.bool, device=DEV)
            if w0 <= w1:
                mask[h0:h1 + 1, w0:w1 + 1] = False
            assert not Jr[b, k][mask].any()


@pytest.mark.parametrize("per_pose", [False, True])
def test_columns_are_the_render_backward(per_pose):
    """sum_n gout_n J[b, k, n] equals autograd's gradient of sum(gout * render_polyrigid(blend="log_euclidean")) with respect to
    the increments xi at xi = 0 (apply_increments' left increment about polyrigid_pivots)."""
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=1))
    X = se3_exp(_twists(3, 2 if per_pose else None, seed=2)).float()
    _, J = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=150, **LE, **KW)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(3)).to(DEV)
    lhs = torch.einsum("bhw,bkhwi->bki", gout[:, 0].double(), J.double())
    if not per_pose:
        lhs = lhs.sum(0)
    xi = torch.zeros(*X.shape[:-2], 6, dtype=torch.float64, device=DEV, requires_grad=True)
    out = drr.render_polyrigid(rot, xyz, motions=_moved(X, xi, pr.polyrigid_pivots(drr, W)), weights=W, n_points=150, **LE, **KW)
    (gout * out).sum().backward()
    assert float(xi.grad.abs().max()) > 0
    err = relerr(lhs.cpu().numpy(), xi.grad.cpu().numpy())
    print(f"per_pose={per_pose}: transpose against autograd {err:.2e}")
    # J repeats bit for bit; autograd's side sums the field scatter and the squarings' adjoints with atomics, so it moves between
    # runs.  Per-pose motions measured 9.7e-6 to 1.09e-5 over three H100 runs (shared: 1.6e-6 to 1.7e-6), hence the wider bound.
    assert err <= (2e-5 if per_pose else 1e-5)


def test_jacobian_column_matches_an_fp64_central_difference():
    """Independent of every fp32 kernel: the velocity formed in float64, svf_oracle's exponential and deform_oracle's forward on
    the module's rays, differenced along omega_y and v_z of structure 1."""
    vol, drr, W = _scene(H=24)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(1, seed=4))
    X = se3_exp(_twists(3, seed=5)).float()
    _, J = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=120, **LE, **KW)
    with torch.no_grad():
        source, target = drr.detector(convert(rot, xyz, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = drr.affine_inverse(source)[:, 0], drr.affine_inverse(target)
    src, tgt, raylen = (t.double().cpu().numpy() for t in (src, tgt, raylen))
    amin, amax = tc.range_of(DIMS, src.astype(np.float32), tgt.astype(np.float32))
    g = 1.0 + torch.rand(24, 24, generator=torch.Generator().manual_seed(6)).double()
    A = drr._affine.reshape(4, 4).double().cpu()
    pivots = pr.polyrigid_pivots(drr, W).cpu()
    Wn = W.double().cpu()
    x = torch.nn.functional.pad(so.node_coords(tuple(W.shape[1:]), DIMS), (0, 1), value=1.0)
    h = 1e-6

    def f(k, col, s):
        xi = torch.zeros(3, 6, dtype=torch.float64)
        xi[k, col] = s
        Xk = apply_increments(X.cpu().double(), xi, pivots)
        L = (torch.linalg.inv(A) @ svf.se3_log_matrix(_rigid_inverse(Xk)) @ A)[:, :3, :]
        v = torch.einsum("kxyz,krc,xyzc->xyzr", Wn, L, x)[None]
        U = so.exp(v, LE["steps"], DIMS).numpy()
        img = do.fwd(vol, src, tgt, raylen, np.moveaxis(U, -1, 1), 120, float(amin), float(amax))
        return float((g.numpy().reshape(1, -1) * img).sum())

    for k, col in ((1, 1), (1, 5)):
        an = float((g.to(DEV) * J[0, k, ..., col].double()).sum())
        fd = (f(k, col, h) - f(k, col, -h)) / (2 * h)
        print(f"column ({k}, {col}): {an:.6e} against fp64 {fd:.6e}")
        assert abs(fd) > 0 and abs(an - fd) < 1e-3 * abs(fd), (k, col, an, fd)


def test_normal_equations_on_the_jacobian_equal_the_dense_statement():
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=7))
    X = se3_exp(_twists(3, seed=8)).float()
    img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=150, return_footprints=True, **LE, **KW)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=se3_exp(_twists(3, seed=9, scale=0.5)).float(), weights=W, n_points=150,
                                      **LE, **KW)
    B, K = 2, 3
    x, t = img.reshape(B, 40, 40).contiguous(), target.reshape(B, 40, 40).contiguous()
    area = (rects[..., 1] - rects[..., 0] + 1) * (rects[..., 3] - rects[..., 2] + 1)
    print(f"footprint areas {area.tolist()} of {40 * 40} pixels")
    assert (area < 40 * 40).any()   # footprints do cull
    A = torch.zeros(B, 6 * K, 6 * K, dtype=torch.float64, device=DEV)
    g = torch.zeros(B, 6 * K, dtype=torch.float64, device=DEV)
    ncc_normal_structures_equations(x, t, J, rects, 1e-5, 1.0, A, g)
    Ar, gr = _dense(x, t, J.reshape(B, K, 40 * 40, 6), K)
    assert relerr(A.cpu().numpy(), Ar.cpu().numpy()) <= 1e-9 and relerr(g.cpu().numpy(), gr.cpu().numpy()) <= 1e-9


@pytest.mark.parametrize("per_pose", [False, True])
def test_lm_never_increases_the_loss_and_makes_no_host_sync(per_pose):
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(3, seed=10))
    X_true = se3_exp(_twists(3, 3 if per_pose else None, seed=11, scale=0.5)).float()
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=X_true, weights=W, n_points=150, **LE, **KW)
    X = torch.eye(4, device=DEV).expand(*X_true.shape).clone()
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=150, **LE, **KW)
    hist = [lm.step()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(5):
            hist.append(lm.step())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    h = torch.stack(hist).cpu()
    assert h.shape == ((6, 3) if per_pose else (6,))
    assert (h[1:] <= h[:-1]).all(), h
    assert (h[-1] < h[0]).all(), h


def test_refusals_come_before_any_launch():
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(1, seed=1))
    X = torch.eye(4, device=DEV).expand(3, 4, 4).clone()
    target = torch.zeros(1, 1, 40, 40, device=DEV)
    for bad in (0, 17, 2.5, True):
        with pytest.raises(ValueError, match="steps must be"):
            drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, blend="log_euclidean", steps=bad, **KW)
        with pytest.raises(ValueError, match="steps must be"):
            PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, blend="log_euclidean", steps=bad, **KW)
    with pytest.raises(ValueError, match="blend must be"):
        drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, blend="dual_quaternion", **KW)
    with pytest.raises(ValueError, match="blend must be"):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, blend="dual_quaternion", **KW)
    with pytest.raises(TypeError):
        PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, loss=NormalizedCrossCorrelation2d(patch_size=8), **LE, **KW)
    _, sub, _ = _scene(p_subsample=0.5)
    with pytest.raises(NotImplementedError, match="full detector"):
        sub.polyrigid_jacobian(rot, xyz, motions=X, weights=W, **LE, **KW)
    with pytest.raises(NotImplementedError):
        PolyrigidLevenbergMarquardt(sub, rot, xyz, X, W, target, **LE, **KW)


# ---- convergence on the two-structure scene -------------------------------------------------------------------------------------
def _run_lm(X, steps, rad, mm):
    """test_gpu_polyrigid_lm's two-structure scene with the target rendered by the log-Euclidean blend (test_gpu_svf.
    test_registration_recovers_two_structures' problem; Adam needs 500 steps there) and the same blend fitted."""
    drr, rot, xyz, W, _, X_true, centre, w_true, t_true = _two_structures()
    le = dict(blend="log_euclidean", steps=10)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=X_true, weights=W, n_points=250, **le, **KW)
    X = X(centre, w_true, t_true) if callable(X) else X
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=250, **le, **KW)
    for k in range(1, steps + 1):
        loss = lm.step()
        err_r, err_t = registration_errors(X, X_true, centre)
        print(f"step {k}: rotation error {err_r:.3e} rad, centroid error {err_t:.3e} mm, loss {float(loss):.3e}")
        if err_r < rad and err_t < mm:
            return k, err_r, err_t, float(loss)
    raise AssertionError(f"after {steps} steps: rotation error {err_r:.4f} rad, centroid error {err_t:.3f} mm, loss {float(loss):.3g}")


def test_lm_converges_quadratically_near_the_solution():
    """From 80 % of the way there (rotations at 0.8 x, translations at 0.98 x the truth): 1e-3 rad and 0.02 mm within 6 steps."""
    steps, err_r, err_t, loss = _run_lm(lambda c, w, t: _about(0.8 * w, 0.98 * t, c), 6, 1e-3, 0.02)
    print(f"log-Euclidean LM from 80 % of the way: {steps} steps, {err_r:.2e} rad, {err_t:.3f} mm, loss {loss:.3g}")


def test_lm_recovers_two_structures():
    """From the identity: 0.02 rad and 2 mm within 40 steps."""
    steps, err_r, err_t, loss = _run_lm(torch.eye(4, device=DEV).expand(2, 4, 4).clone(), 40, 0.02, 2.0)
    print(f"log-Euclidean LM recovered both structures in {steps} steps: {err_r:.2e} rad, {err_t:.3f} mm, loss {loss:.3g}")
