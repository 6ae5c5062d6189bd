"""Stationary velocity fields on the GPU (exp_velocity, DRR.render_polyrigid(blend="log_euclidean"); DESIGN.md 6m): the squaring
kernels and their adjoint against the fp64 reference of svf_oracle.py, the identities (zero velocity, zero weights, identity
motions, the affine identity of one rigid structure), autograd to the camera pose and the motions against the fp64 chain of the
oracle exponential and deform_oracle.py, the detector variants, the refusals, CUDA-graph capture and two registrations."""
import math

import numpy as np
import pytest
import torch

import deform_oracle as do
import svf_oracle as so
import trilinear_cases as tc
from conftest import relerr
from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, exp_velocity, polyrigid_weights, synthetic
from diffdrr_b200 import _lib
from diffdrr_b200 import svf
from diffdrr_b200.pose import convert
from diffdrr_b200.structures import _rigid_inverse, se3_exp, twist_matrix
from test_gpu_polyrigid import _about, _rays, _scene, _twists
from test_svf_cpu import CASES, _case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
DIMS = (48, 56, 40)


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=DEV)


def _pad(u):
    return torch.nn.functional.pad(_t(u), (0, 1)).contiguous()


@pytest.mark.parametrize("name", sorted(CASES))
def test_kernels_match_fp64_reference(name):
    D, u, gp = _case(name)
    steps = 4
    v = (u * 0.5)
    ref = so.exp(torch.tensor(v), steps, D).numpy()
    V = _pad(v).requires_grad_(True)
    out = svf._SquaringFunction.apply(V, steps, D)
    assert torch.all(out[..., 3] == 0)
    got = out[..., :3].detach().cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()
    out.backward(_pad(gp))
    gref = so.exp_bwd(v, gp, steps, D).numpy()
    g = V.grad[..., :3].cpu().numpy()
    assert torch.all(V.grad[..., 3] == 0)
    # the emulated adjoint is within 2e-6 of the reference per step; 4 steps compound it
    assert np.abs(g - gref).max() <= 2e-5 * np.abs(gref).max()
    again = svf._SquaringFunction.apply(V.detach(), steps, D)
    assert torch.equal(again, out.detach())   # one write per node: the forward repeats bit for bit


def _velocity(B=None, grid=(10, 12, 9), seed=0, amp=6.0):
    rng = np.random.default_rng(seed)
    coarse = rng.normal(size=(1 if B is None else B, 3, 3, 3, 3)) * amp
    v = torch.nn.functional.interpolate(torch.tensor(coarse), size=grid, mode="trilinear", align_corners=True)
    return _t(v[0] if B is None else v)


@pytest.mark.parametrize("per_pose", [False, True])
def test_exp_velocity_and_its_gradient_match_fp64_autograd(per_pose):
    _, drr, _ = _scene()
    v0 = _velocity(2 if per_pose else None, seed=1)
    gout = torch.randn(v0.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    v = v0.clone().requires_grad_(True)
    u = exp_velocity(drr, v, steps=8)
    assert u.shape == v.shape
    (u * gout).sum().backward()
    A = drr._affine.reshape(4, 4)[:3, :3].double().cpu()
    Ainv = torch.linalg.inv(A)
    w = v0.detach().double().cpu().requires_grad_(True)
    wb = w if w.dim() == 5 else w[None]
    vox = torch.einsum("ij,bjxyz->bxyzi", Ainv, wb)
    ref = torch.einsum("ij,bxyzj->bixyz", A, so.exp(vox, 8, DIMS))
    ref = ref if w.dim() == 5 else ref[0]
    (ref * gout.double().cpu()).sum().backward()
    assert relerr(u.detach().cpu().numpy(), ref.detach().numpy()) <= 1e-5
    assert relerr(v.grad.cpu().numpy(), w.grad.numpy()) <= 2e-5


def test_identities():
    vol, drr, W = _scene()
    zero = exp_velocity(drr, torch.zeros(3, 10, 12, 9, device=DEV))
    assert torch.equal(zero, torch.zeros_like(zero))
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=3))
    plain = drr(rot, xyz, n_points=150, **KW)
    X = se3_exp(_twists(3, seed=4))
    le = dict(weights=W, n_points=150, blend="log_euclidean", **KW)
    assert torch.equal(drr.render_polyrigid(rot, xyz, motions=X, **{**le, "weights": torch.zeros_like(W)}), plain)
    eye = torch.eye(4, device=DEV).expand(3, 4, 4).contiguous()
    assert torch.equal(drr.render_polyrigid(rot, xyz, motions=eye, **le), plain)
    # the linear blend is untouched by the new option
    lin = drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=150, **KW)
    assert torch.equal(drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=150, blend="linear", **KW), lin)
    # small motions: the two blends agree to first order
    Xs = se3_exp(_twists(3, seed=4, scale=0.05))
    a = drr.render_polyrigid(rot, xyz, motions=Xs, **le).cpu().numpy()
    b = drr.render_polyrigid(rot, xyz, motions=Xs, weights=W, n_points=150, **KW).cpu().numpy()
    assert relerr(a, b) <= 2e-2


def test_one_rigid_structure_is_the_affine_identity():
    """One structure at weight 1 on the whole lattice: the velocity is L [x; 1] with L = log(M), and the kernels' exponential is
    ((I + L / 2^N)^(2^N) - I) [x; 1] at every node whose trajectory stays inside the lattice."""
    _, drr, _ = _scene()
    g, steps = (24, 28, 20), 10
    X = se3_exp(_twists(1, seed=5, scale=0.5))
    U = svf._SquaringFunction.apply(svf.polyrigid_velocity(drr, X, torch.ones(1, *g, device=DEV)), steps, DIMS)
    A = drr._affine.reshape(4, 4).double().cpu()
    L = (torch.linalg.inv(A) @ svf.se3_log_matrix(_rigid_inverse(X[0].double().cpu())) @ A)[:3]
    x = so.node_coords(g, DIMS)
    ident = so.affine_identity(L, steps, x)
    v = torch.cat([x, torch.ones(*g, 1, dtype=torch.float64)], -1) @ L.T
    ref = so.exp(v[None], steps, DIMS)[0]
    inside = (ref - ident).abs().amax(-1) <= 1e-9   # the fp64 reference's own test of "stays inside"
    assert inside.float().mean() > 0.3
    got = U[0, ..., :3].double().cpu()
    assert float((got - ident).abs().amax(-1)[inside].max()) <= 1e-5 * float(ident.abs().max())
    # and close to the exact rigid map there (the squaring's error, 4x smaller per step)
    M = torch.linalg.inv(A) @ _rigid_inverse(X[0].double().cpu()) @ A
    exact = torch.cat([x, torch.ones(*g, 1, dtype=torch.float64)], -1) @ (M - torch.eye(4, dtype=torch.float64))[:3].T
    assert float((ident - exact).abs()[inside].max()) <= 1e-2


@pytest.mark.parametrize("at_identity", [False, True])
def test_autograd_to_pose_and_motions_matches_fp64_chain(at_identity):
    """rot, xyz and the twists of the motions, blend="log_euclidean": autograd against the fp64 chain of the same host algebra,
    svf_oracle's exponential and deform_oracle's march.  At the identity motions the log's derivative must still be finite."""
    vol, drr, W = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=6))
    xi0 = torch.zeros(2, 3, 6, device=DEV) if at_identity else _twists(3, 2, seed=7)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(8)).to(DEV)
    rot, xyz, xi = (t.clone().requires_grad_(True) for t in (rot0, xyz0, xi0))
    steps = 8
    # at xi = 0 the motions come from torch.linalg.matrix_exp: se3_exp's own derivative is not finite exactly there
    motion = (lambda t: torch.linalg.matrix_exp(twist_matrix(t))) if at_identity else se3_exp
    img = drr.render_polyrigid(rot, xyz, motions=motion(xi).float(), weights=W, n_points=150, blend="log_euclidean",
                               steps=steps, **KW)
    (img * gout).sum().backward()

    def chain(dtype):
        host = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(torch.float64)
        r, x, t = (v.detach().cpu().double().requires_grad_(True) for v in (rot0, xyz0, xi0))
        source, target = host.detector(convert(r, x, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = host.affine_inverse(source)[:, 0], host.affine_inverse(target)
        A = host._affine.reshape(4, 4)
        L = (torch.linalg.inv(A) @ svf.se3_log_matrix(_rigid_inverse(motion(t))) @ A)[..., :3, :]   # (2, 3, 3, 4)
        g = W.shape[1:]
        xh = torch.cat([so.node_coords(g, DIMS), torch.ones(*g, 1, dtype=torch.float64)], -1)
        v = torch.einsum("kxyz,bkij,xyzj->bxyzi", W.double().cpu(), L, xh)
        Uv = so.exp(v, steps, DIMS).permute(0, 4, 1, 2, 3)
        dims = torch.tensor(DIMS, dtype=torch.float64)
        from diffdrr_b200.renderers import _get_alpha_minmax
        amin, amax = _get_alpha_minmax(src[:, None], tgt, dims, 0.5, 1e-8)
        amin, amax = amin.min(), amax.max()
        q = do.bwd(vol, src.detach().numpy(), tgt.detach().numpy(), raylen.detach().numpy(), Uv.detach().numpy(),
                   gout.cpu().numpy().reshape(2, -1), 150, float(amin), float(amax), dtype=dtype)
        total = sum((torch.from_numpy(np.asarray(q[k], np.float64)) * val).sum() for k, val in
                    (("g_src", src), ("g_tgt", tgt), ("g_raylen", raylen), ("g_U", Uv)))
        (total + q["g_alphamin"] * amin + q["g_alphamax"] * amax).backward()
        return [val.grad.numpy() for val in (r, x, t)]

    ref, r32 = chain(np.float64), chain(np.float32)
    for got, want, w32, name in zip((rot.grad, xyz.grad, xi.grad), ref, r32, ("rot", "xyz", "twists")):
        assert torch.isfinite(got).all(), name
        assert np.abs(want).max() > 0
        assert relerr(got.cpu().numpy(), want) <= max(tc.tol(w32, want, 1e-3), 2e-3), name


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_per_pose_16bit_and_detector_variants_render_the_same_pixels(dtype):
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=9))
    amin, amax = _rays(drr, rot, xyz)[3]
    kw = dict(weights=W, n_points=120, alphamin=amin, alphamax=amax, blend="log_euclidean", **KW)
    X = se3_exp(_twists(3, 2, seed=10))
    full = drr.render_polyrigid(rot, xyz, motions=X, **kw)
    for b in range(2):   # per-pose motions: each pose renders as that pose alone with its own motions (the velocity's
        one = drr.render_polyrigid(rot[b:b + 1], xyz[b:b + 1], motions=X[b], **kw)   # batched product may round differently)
        assert relerr(one.cpu().numpy(), full[b:b + 1].cpu().numpy()) <= 1e-6
    _, patched, _ = _scene(patch_size=10)
    assert torch.equal(patched.render_polyrigid(rot, xyz, motions=X, **kw), full)
    _, sub, _ = _scene(p_subsample=0.3)
    got = sub.render_polyrigid(rot, xyz, motions=X, **kw)
    pick = sub.detector.pick_tensor()
    assert torch.equal(got.reshape(2, -1)[:, pick], full.reshape(2, -1)[:, pick])
    half = drr.density.to(dtype)
    drr.density = half.float()
    up = drr.render_polyrigid(rot, xyz, motions=X, **kw)
    drr.density = half
    assert relerr(drr.render_polyrigid(rot, xyz, motions=X, **kw).cpu().numpy(), up.cpu().numpy()) <= 1e-6


def test_cuda_graph_replays_one_step():
    _, drr, W = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=11))
    xi0 = _twists(3, seed=12)
    w = torch.rand(2, 1, 40, 40, device=DEV)

    def step(r, x, t):
        img = drr.render_polyrigid(r, x, motions=se3_exp(t), weights=W, n_points=100, blend="log_euclidean", **KW)
        (img * w).sum().backward()
        return img.detach()

    r_e, x_e, t_e = (t.clone().requires_grad_(True) for t in (rot0, xyz0, xi0))
    img_e = step(r_e, x_e, t_e)
    r_d, x_d, t_d = (t.clone().requires_grad_(True) for t in (rot0, xyz0, xi0))
    step(r_d, x_d, t_d)

    def body():
        for t in (r_d, x_d, t_d):
            t.grad.zero_()
        return step(r_d, x_d, t_d)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        img_g = body()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(img_g, img_e)
    for a, b in ((r_d, r_e), (x_d, x_e), (t_d, t_e)):
        assert relerr(a.grad.cpu().numpy(), b.grad.cpu().numpy()) < 1e-5


def test_unsupported_combinations_raise_before_any_launch():
    vol, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=13))
    X = torch.eye(4, device=DEV).expand(3, 4, 4).contiguous()
    call = lambda d=drr, **kw: d.render_polyrigid(rot, xyz, motions=X, weights=W, **KW, **kw)   # noqa: E731
    with pytest.raises(ValueError, match="blend must be"):
        call(blend="dual_quaternion")
    for bad in (0, 17, 2.5, True):
        with pytest.raises(ValueError, match="steps must be"):
            call(blend="log_euclidean", steps=bad)
    siddon = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40)).to(DEV)
    with pytest.raises(NotImplementedError, match="Trilinear renderer"):
        call(siddon, blend="log_euclidean")
    with pytest.raises(ValueError, match="sum to at most 1"):
        drr.render_polyrigid(rot, xyz, motions=X, weights=torch.full_like(W, 0.5), blend="log_euclidean", **KW)
    with pytest.raises(NotImplementedError, match="blend weights"):
        drr.render_polyrigid(rot, xyz, motions=X, weights=W.clone().requires_grad_(True), blend="log_euclidean", **KW)
    v = torch.zeros(3, 6, 6, 6, device=DEV)
    with pytest.raises(ValueError, match="velocity must be"):
        exp_velocity(drr, v.double())
    with pytest.raises(ValueError, match="velocity must be"):
        exp_velocity(drr, v[0])
    with pytest.raises(ValueError, match="velocity must be"):
        exp_velocity(drr, torch.zeros(2, 6, 6, 6, device=DEV))
    with pytest.raises(_lib.B200DRRError, match="no CPU"):
        exp_velocity(drr, v.cpu())
    for bad in (0, 17):
        with pytest.raises(ValueError, match="steps must be"):
            exp_velocity(drr, v, steps=bad)


def test_registration_recovers_two_structures():
    """test_gpu_polyrigid.py's two-structure registration with the target rendered by the log-Euclidean blend and the same blend
    fitted: Adam on each block's rotation and translation from (almost) the identity reaches the same bounds."""
    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    rng = np.random.default_rng(3)
    lab = np.zeros((n, n, n), np.float32)
    lab[30:58, 40:70, 36:60] = 1
    lab[70:100, 60:86, 66:96] = 2
    vol = (vol + (lab > 0) * (1.0 + 0.5 * rng.random((n, n, n)))).astype(np.float32)
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(96), renderer="trilinear").to(DEV)
    aff = torch.as_tensor(synthetic.make_affine(n), dtype=torch.float32)
    W = polyrigid_weights(drr.mask, (1, 2), grid=(32, 32, 32), sigma=6.0, spacing=tuple(float(aff[a, a]) for a in range(3)))
    centre = torch.stack([torch.as_tensor(np.argwhere(lab == k).mean(0), dtype=torch.float32) for k in (1, 2)])
    centre = (centre @ aff[:3, :3].T + aff[:3, 3]).to(DEV)
    rot = torch.tensor([[0.0, 0.0, 0.0], [math.pi / 2, 0.0, 0.0], [0.0, math.pi / 2, 0.0]], device=DEV)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(3, 3).contiguous()
    w_true = torch.tensor([[0.05, -0.03, 0.04], [-0.04, 0.05, 0.03]], device=DEV)
    t_true = torch.tensor([[8.0, -6.0, 5.0], [-7.0, 9.0, -4.0]], device=DEV)
    kw = dict(weights=W, n_points=250, blend="log_euclidean", **KW)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=_about(w_true, t_true, centre), **kw)
    w = torch.full((2, 3), 1e-4, device=DEV, requires_grad=True)
    t = torch.zeros(2, 3, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[w], lr=5e-3), dict(params=[t], lr=0.5)])
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.994)
    ncc = NormalizedCrossCorrelation2d()
    steps = 500
    for _ in range(steps):
        opt.zero_grad()
        loss = -ncc(drr.render_polyrigid(rot, xyz, motions=_about(w, t, centre), **kw), target).mean()
        loss.backward()
        opt.step()
        sched.step()
    err_w = float((w.detach() - w_true).abs().max())
    err_t = float((t.detach() - t_true).abs().max())
    print(f"log-Euclidean polyrigid registration after {steps} steps: rotation error {err_w:.4f} rad, translation error "
          f"{err_t:.3f} mm, loss {float(loss):.5f}")
    assert err_w < 0.02 and err_t < 2.0, (err_w, err_t, float(loss))


def test_diffeomorphic_registration_lowers_ncc_and_stays_invertible():
    """test_gpu_deform.py's deformable scene (128^3 phantom, four views at 96^2, a target from a smooth 8^3 world-mm field), fitted
    through a stationary velocity: Adam on an 8^3 velocity from zero through render_deformed(field=exp_velocity(drr, V)).  The
    objective falls and the recovered map keeps det grad phi > 0 at every interior node."""
    import deform_cases as dc

    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(96), renderer="trilinear").to(DEV)
    rot = torch.tensor([[0.0, 0.0, 0.0], [torch.pi / 2, 0.0, 0.0], [0.0, torch.pi / 2, 0.0], [torch.pi / 4, torch.pi / 4, 0.0]],
                       device=DEV)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(4, 3).contiguous()
    grid = (8, 8, 8)
    U_true = _t(dc.smooth_field(np.random.default_rng(21), 1, grid, 6.0)[0])
    kw = dict(n_points=250, **KW)
    with torch.no_grad():
        target = drr.render_deformed(rot, xyz, field=U_true, **kw)
    ncc = NormalizedCrossCorrelation2d()
    V = torch.zeros_like(U_true, requires_grad=True)
    opt = torch.optim.Adam([V], lr=0.3)

    def objective():
        return (1 - ncc(drr.render_deformed(rot, xyz, field=exp_velocity(drr, V), **kw), target)).mean()

    with torch.no_grad():
        loss0 = float(objective())
    steps = 200
    for _ in range(steps):
        opt.zero_grad()
        loss = objective()
        (loss + 1e-3 * sum((V.diff(dim=a) ** 2).mean() for a in (1, 2, 3))).backward()
        opt.step()
    with torch.no_grad():
        loss1 = float(objective())
        u = exp_velocity(drr, V)
    lin = drr._affine_inverse.reshape(4, 4)[:3, :3].double()
    vox = torch.einsum("ij,jxyz->xyzi", lin, u.double())[None].cpu()
    det = so.jacobian_det(vox, (n, n, n))
    print(f"diffeomorphic registration after {steps} steps: mean 1 - NCC {loss0:.3e} -> {loss1:.3e} ({loss0 / loss1:.1f}x), "
          f"det grad phi in [{float(det.min()):.3f}, {float(det.max()):.3f}]")
    assert loss0 / loss1 >= 2.0, (loss0, loss1)
    assert float(det.min()) > 0
