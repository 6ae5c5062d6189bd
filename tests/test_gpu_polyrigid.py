"""Blended-rigid (skinned) renders on the GPU (DRR.render_polyrigid; DESIGN.md 6h): the kernels on the seeded cases of
polyrigid_cases.py against the fp64 reference of polyrigid_oracle.py, plain / packed / 16-bit routes, the identities that tie the
march to the Trilinear renderer, autograd to the camera pose and the motions against the reference chained through torch in
float64, reproducible bits, CUDA-graph capture, the refusals, and a two-structure registration."""
import math

import numpy as np
import pytest
import torch

import polyrigid_cases as pc
import polyrigid_oracle as po
import trilinear_cases as tc
from conftest import relerr
from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, Trilinear, polyrigid_weights, synthetic
from diffdrr_b200 import polyrigid as pr
from diffdrr_b200.pose import RigidTransform, convert
from diffdrr_b200.structures import _rigid_inverse, se3_exp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
FLOOR = 1e-4
DIMS = (48, 56, 40)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _kernels(c, packed=False, dtype=torch.float32, grads=True, M=None, weights=None, vol=None):
    """The case through b200drr_polyrigid_fwd / _bwd (the autograd function is their only caller) -> numpy dict as the reference's."""
    vol = _t(c["vol"] if vol is None else vol).to(dtype)
    pk = Trilinear()._packed_volume(vol) if packed else None
    assert (pk is not None) == packed
    src, tgt, raylen, Mt = (_t(a).requires_grad_(grads) for a in (c["src"][:, None], c["tgt"], c["raylen"][:, None],
                                                                  c["M"] if M is None else M))
    w = _t(c["weights"] if weights is None else weights)
    K, g0, g1, g2 = w.shape
    lib = pr._lib.load()
    wp = torch.empty(int(lib.b200drr_polyrigid_weight_floats(K, g0, g1, g2)), device=DEV)
    pr._lib.check(lib.b200drr_polyrigid_pack_weights(pr._ptr(w), K, g0, g1, g2, pr._ptr(wp), pr._stream()), "pack_weights")
    arange = torch.tensor([c["amin"], c["amax"]], device=DEV, requires_grad=grads)
    grid = (c["H"], c["W"]) if c["H"] else None
    out = pr._PolyrigidFunction.apply(vol, pk, src, tgt, raylen, Mt, arange, wp, (g0, g1, g2), 0.5, 1e-8, c["n_points"], grid)
    res = dict(out=out.detach().cpu().numpy()[:, 0])
    if grads:
        out.backward(_t(c["gout"])[:, None])
        res.update(g_src=src.grad.cpu().numpy()[:, 0], g_tgt=tgt.grad.cpu().numpy(), g_raylen=raylen.grad.cpu().numpy()[:, 0],
                   g_M=Mt.grad.cpu().numpy(), g_alphamin=float(arange.grad[0]), g_alphamax=float(arange.grad[1]))
    return res


@pytest.fixture(scope="module", params=sorted(pc.CASES))
def case(request):
    c = pc.CASES[request.param]()
    c["ref"] = po.fwd(*pc.args(c))
    c["gref"] = po.bwd(*pc.args(c)[:6], c["gout"], *pc.args(c)[6:])
    c["g32"] = po.bwd(*pc.args(c)[:6], c["gout"], *pc.args(c)[6:], dtype=np.float32)
    return c


def test_kernels_match_fp64_reference(case):
    c = case
    got = _kernels(c)
    assert relerr(got["out"], c["ref"]) <= 1e-4
    ref, r32 = c["gref"], c["g32"]
    assert relerr(got["g_raylen"], ref["g_raylen"]) <= tc.tol(r32["g_raylen"], ref["g_raylen"], FLOOR)
    smooth = slice(None) if c["kinks"] is None else ~c["kinks"]   # a ray on an integer plane has a one-sided derivative
    assert relerr(got["g_tgt"][:, smooth], ref["g_tgt"][:, smooth]) <= tc.tol(r32["g_tgt"][:, smooth], ref["g_tgt"][:, smooth], FLOOR)
    if c["kinks"] is not None:
        return
    for key in ("g_src", "g_M"):
        assert relerr(got[key], ref[key]) <= tc.tol(r32[key], ref[key], FLOOR), key
    scale = tc.alpha_scale(ref["g_raylen"], c["raylen"], c["amin"], c["amax"])
    for key in ("g_alphamin", "g_alphamax"):
        assert abs(got[key] - ref[key]) / scale <= tc.tol(r32[key], ref[key], FLOOR, scale=scale), key


def test_packed_equals_plain_and_repeats_bitwise(case):
    a, b, again = _kernels(case), _kernels(case, packed=True), _kernels(case)
    for key in a:
        assert np.array_equal(a[key], again[key]), key     # no atomics: g_M, g_src and the range partials repeat bit for bit
    for key in ("out", "g_tgt", "g_raylen", "g_M", "g_src", "g_alphamin", "g_alphamax"):
        assert np.array_equal(a[key], b[key]), key


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("packed", [False, True])
def test_16bit_density_equals_fp32_on_the_upcast_volume(dtype, packed):
    c = pc.CASES["k3_per_pose"]()
    up = _t(c["vol"]).to(dtype).float().cpu().numpy()
    a, b = _kernels(c, packed=packed, dtype=dtype), _kernels(c, vol=up)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_identities_in_the_kernels(case):
    c = case
    plain = DRR_free_trilinear(c)
    eye = np.broadcast_to(np.eye(3, 4, dtype=np.float32), c["M"].shape)
    assert np.array_equal(_kernels(c, grads=False, M=eye)["out"], plain)
    assert np.array_equal(_kernels(c, grads=False, weights=np.zeros_like(c["weights"]))["out"], plain)


def DRR_free_trilinear(c):
    """The Trilinear renderer on the case's rays with the case's explicit range."""
    r = Trilinear()
    out = r(_t(c["vol"]), _t(c["src"][:, None]), _t(c["tgt"]), _t(c["raylen"][:, None]), n_points=c["n_points"], alphamin=c["amin"],
            alphamax=c["amax"])
    return out.cpu().numpy()[:, 0]


# ---- through DRR.render_polyrigid -----------------------------------------------------------------------------------------------
def _scene(K=3, H=40, seed=0, **kw):
    vol = tc.volume(DIMS)
    lab = np.zeros(DIMS, np.float32)
    lab[8:20, 10:26, 6:18], lab[26:40, 30:48, 20:34], lab[10:22, 34:50, 22:36] = 3, 7, 12
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(H), renderer="trilinear",
              **kw).to(DEV)
    W = polyrigid_weights(drr.mask, (3, 7, 12)[:K], grid=(12, 14, 10), sigma=12.0, spacing=(4.0, 4.0, 4.0))
    return vol, drr, W


def _twists(K, B=None, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    shape = (K, 6) if B is None else (B, K, 6)
    xi = (torch.rand(*shape, generator=g) * 2 - 1) * torch.tensor([0.08, 0.08, 0.08, 10.0, 10.0, 10.0]) * scale
    return xi.to(DEV)


def _rays(drr, rot, xyz):
    """(src (B, 3), tgt (B, N, 3), raylen (B, N)) in voxel-index space, as the module builds them, and the range it would use."""
    with torch.no_grad():
        source, target = drr.detector(convert(rot, xyz, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = drr.affine_inverse(source), drr.affine_inverse(target)
    src, tgt, raylen = (t.cpu().numpy() for t in (src[:, 0], tgt, raylen))
    return src, tgt, raylen, tc.range_of(DIMS, src, tgt)


@pytest.mark.parametrize("per_pose", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_module_matches_fp64_reference(per_pose, dtype):
    vol, drr, W = _scene()
    assert float(W.max()) > 0.5
    if dtype != torch.float32:
        drr.density = drr.density.to(dtype)
        vol = drr.density.float().cpu().numpy()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=1))
    X = se3_exp(_twists(3, 2 if per_pose else None, seed=2))
    img = drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=150, **KW)
    assert img.shape == (2, 1, 40, 40)
    src, tgt, raylen, (amin, amax) = _rays(drr, rot, xyz)
    M = pr.voxel_maps(drr, X).cpu().numpy().reshape(-1, 3, 3, 4)
    ref = po.fwd(vol, src, tgt, raylen, M, W.cpu().numpy(), 150, amin, amax)
    assert relerr(img.cpu().numpy().reshape(ref.shape), ref) <= 1e-4
    plain = drr(rot, xyz, n_points=150, **KW)
    assert relerr(img.cpu().numpy(), plain.cpu().numpy()) > 1e-2          # the motions do move the image


def test_identities_against_forward():
    vol, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=3))
    plain = drr(rot, xyz, n_points=150, **KW)
    eye = torch.eye(4, device=DEV).expand(3, 4, 4).contiguous()
    assert torch.equal(pr.voxel_maps(drr, eye)[..., :3], torch.eye(3, device=DEV).expand(3, 3, 3))
    # the map's translation column is A^-1 t - A^-1 t evaluated in float64: zero to ~1e-16 voxel, not to the bit
    err_eye = relerr(drr.render_polyrigid(rot, xyz, motions=eye, weights=W, n_points=150, **KW).cpu().numpy(), plain.cpu().numpy())
    assert err_eye <= 1e-6, err_eye
    X = se3_exp(_twists(3, seed=4))
    assert torch.equal(drr.render_polyrigid(rot, xyz, motions=X, weights=torch.zeros_like(W), n_points=150, **KW), plain)
    # K = 1, w = 1: the camera X^-1 P sees the unmoved volume.  A lattice of ones falls to 0 within half a cell of the faces, so the
    # density is cut to a core no sample with w < 1 can reach; one explicit range for both renders.
    core = np.zeros_like(vol)
    core[12:-12, 12:-12, 12:-12] = vol[12:-12, 12:-12, 12:-12]
    drr1 = DRR(synthetic.make_subject(core), **synthetic.detector_kwargs(40), renderer="trilinear").to(DEV)
    X1 = se3_exp(_twists(1, seed=5, scale=0.5))
    P = convert(rot, xyz, **KW).matrix
    amin, amax = _rays(drr1, rot, xyz)[3]
    kw = dict(n_points=150, alphamin=0.9 * amin, alphamax=min(1.0, 1.1 * amax))
    got = drr1.render_polyrigid(rot, xyz, motions=X1, weights=torch.ones(1, 6, 7, 5, device=DEV), **KW, **kw)
    want = drr1(RigidTransform(_rigid_inverse(X1[0]) @ P), **kw)
    err_one = relerr(got.cpu().numpy(), want.cpu().numpy())
    assert float(want.max()) > 0 and err_one <= 1e-4, err_one


def test_autograd_to_pose_and_motions_matches_fp64_reference():
    """rot, xyz and the twists of the motions: the module's autograd against the fp64 reference's gradients chained through the same
    host algebra in float64 (rays, maps and the batch-global range are torch ops in both)."""
    vol, drr, W = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=6))
    xi0 = _twists(3, 2, seed=7)
    g = torch.Generator().manual_seed(8)
    gout = torch.randn(2, 1, 40, 40, generator=g).to(DEV)
    rot, xyz, xi = (t.clone().requires_grad_(True) for t in (rot0, xyz0, xi0))
    img = drr.render_polyrigid(rot, xyz, motions=se3_exp(xi).float(), weights=W, n_points=150, **KW)
    (img * gout).sum().backward()

    def chain(dtype):
        """d loss / d (rot, xyz, xi) with the kernels' part replaced by the reference evaluated in `dtype`."""
        host = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(torch.float64)
        r, x, t = (v.detach().cpu().double().requires_grad_(True) for v in (rot0, xyz0, xi0))
        source, target = host.detector(convert(r, x, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = host.affine_inverse(source)[:, 0], host.affine_inverse(target)
        A, Ainv = host._affine.reshape(4, 4), host._affine_inverse.reshape(4, 4)
        M = (Ainv @ _rigid_inverse(se3_exp(t)) @ A)[..., :3, :]
        dims = torch.tensor(DIMS, dtype=torch.float64)
        from diffdrr_b200.renderers import _get_alpha_minmax
        amin, amax = _get_alpha_minmax(src[:, None], tgt, dims, 0.5, 1e-8)
        amin, amax = amin.min(), amax.max()
        q = po.bwd(vol, src.detach().numpy(), tgt.detach().numpy(), raylen.detach().numpy(), M.detach().numpy(), W.cpu().numpy(),
                   gout.cpu().numpy().reshape(2, -1), 150, float(amin), float(amax), dtype=dtype)
        lin = sum((torch.from_numpy(np.asarray(q[k], np.float64)) * v).sum() for k, v in
                  (("g_src", src), ("g_tgt", tgt), ("g_raylen", raylen), ("g_M", M)))
        (lin + q["g_alphamin"] * amin + q["g_alphamax"] * amax).backward()
        return [v.grad.numpy() for v in (r, x, t)]

    ref, r32 = chain(np.float64), chain(np.float32)
    for got, want, w32, name in zip((rot.grad, xyz.grad, xi.grad), ref, r32, ("rot", "xyz", "twists")):
        assert np.abs(want).max() > 0
        assert relerr(got.cpu().numpy(), want) <= tc.tol(w32, want, 1e-3), name


def test_subsampled_and_patched_detectors_render_the_same_pixels():
    _, drr, W = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=9))
    amin, amax = _rays(drr, rot, xyz)[3]       # one explicit range: Trilinear's own is that of the rays in the call
    kw = dict(n_points=120, alphamin=amin, alphamax=amax)
    X = se3_exp(_twists(3, seed=10))
    full = drr.render_polyrigid(rot, xyz, motions=X, weights=W, **KW, **kw)
    _, patched, _ = _scene(patch_size=10)
    assert torch.equal(patched.render_polyrigid(rot, xyz, motions=X, weights=W, **KW, **kw), full)
    _, sub, _ = _scene(p_subsample=0.3)
    got = sub.render_polyrigid(rot, xyz, motions=X, weights=W, **KW, **kw)
    pick = sub.detector.pick_tensor()
    assert torch.equal(got.reshape(2, -1)[:, pick], full.reshape(2, -1)[:, pick])
    assert float(got.reshape(2, -1).count_nonzero()) <= 2 * len(pick)


def test_cuda_graph_replays_one_step():
    _, drr, W = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=11))
    xi0 = _twists(3, seed=12)
    w = torch.rand(2, 1, 40, 40, device=DEV)

    def step(r, x, t):
        img = drr.render_polyrigid(r, x, motions=se3_exp(t), weights=W, n_points=100, **KW)
        (img * w).sum().backward()
        return img.detach()

    r_e, x_e, t_e = (t.clone().requires_grad_(True) for t in (rot0, xyz0, xi0))
    img_e = step(r_e, x_e, t_e)
    r_d, x_d, t_d = (t.clone().requires_grad_(True) for t in (rot0, xyz0, xi0))
    step(r_d, x_d, t_d)   # creates the .grad tensors and the cached packed lattice outside the capture

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
    call = lambda d=drr, X=X, W=W, **kw: d.render_polyrigid(rot, xyz, motions=X, weights=W, **KW, **kw)   # noqa: E731
    siddon = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40)).to(DEV)
    with pytest.raises(NotImplementedError, match="Trilinear renderer"):
        call(siddon)
    with pytest.raises(NotImplementedError, match="default options"):
        call(DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear", reducefn="max").to(DEV))
    for bad in (dict(mask_to_channels=True), dict(align_corners=True), dict(stop_gradients=True)):
        with pytest.raises(NotImplementedError, match="no renderer options"):
            call(**bad)
    with pytest.raises(NotImplementedError, match="fp32 / fp16 / bf16"):
        call(DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(DEV).to(torch.float64))
    grad_vol = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(DEV)
    grad_vol.density.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="no volume gradient"):
        call(grad_vol)
    with pytest.raises(NotImplementedError, match="at most 8"):
        call(X=torch.eye(4, device=DEV).expand(9, 4, 4).contiguous(), W=torch.zeros(9, 4, 4, 4, device=DEV))
    with pytest.raises(ValueError, match="motions must be"):
        call(X=X[:2])
    with pytest.raises(ValueError, match="fp32 lattice"):
        call(W=W.double())
    with pytest.raises(ValueError, match=r"in \[0, 1\]"):
        call(W=W - 0.5)
    with pytest.raises(ValueError, match="sum to at most 1"):
        call(W=torch.full_like(W, 0.5))
    with pytest.raises(NotImplementedError, match="blend weights"):
        call(W=W.clone().requires_grad_(True))


def _axis_angle(w):
    th = w.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    k = w / th
    Kx = torch.zeros(*w.shape[:-1], 3, 3, device=w.device, dtype=w.dtype)
    Kx[..., 0, 1], Kx[..., 0, 2], Kx[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    Kx = Kx - Kx.mT
    s, c = th.sin()[..., None], th.cos()[..., None]
    return torch.eye(3, device=w.device, dtype=w.dtype) + s * Kx + (1 - c) * (Kx @ Kx)


def _about(w, t, centre):
    """Rigid motion rotating by w about `centre` (K, 3), then translating by t: x -> R (x - c) + c + t."""
    R = _axis_angle(w)
    top = torch.cat([R, (centre + t - (R @ centre[..., None])[..., 0])[..., None]], dim=-1)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], device=w.device).expand(*w.shape[:-1], 1, 4)
    return torch.cat([top, bottom], dim=-2)


def test_registration_recovers_two_structures():
    """The scene of test_gpu_structures.py's registration (128^3, two labelled blocks, three orthogonal views, 96^2), rendered
    blended: the target by render_polyrigid itself with known motions, then Adam on each block's rotation (about its centroid) and
    translation from the identity, on the NCC."""
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
    kw = dict(weights=W, n_points=250, **KW)
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
    print(f"polyrigid registration after {steps} steps: rotation error {err_w:.4f} rad, translation error {err_t:.3f} mm, "
          f"loss {float(loss):.5f}")
    assert err_w < 0.02 and err_t < 2.0, (err_w, err_t, float(loss))
