"""Deformable renders on the GPU (DRR.render_deformed; DESIGN.md 6i): the kernels on the seeded cases of deform_cases.py against
the fp64 reference of deform_oracle.py, plain / packed / 16-bit routes, the zero-field identity with the Trilinear renderer, the
cross-check with render_polyrigid, autograd to the camera pose and the field against the reference chained through torch in
float64, repeatable bits, CUDA-graph capture, the refusals, and a small deformable registration."""
import numpy as np
import pytest
import torch

import deform_cases as dc
import deform_oracle as do
import trilinear_cases as tc
from conftest import relerr
from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, Trilinear, polyrigid_weights, synthetic
from diffdrr_b200 import deform as dm
from diffdrr_b200.pose import convert

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KW = dict(parameterization="euler_angles", convention="ZXY")
FLOOR = 1e-4
DIMS = (48, 56, 40)
REORDER = 1e-5   # the field gradient is summed with atomics: two calls agree to fp32 reordering


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _kernels(c, packed=False, dtype=torch.float32, grads=True, U=None, vol=None):
    """The case through b200drr_deform_fwd / _bwd (the autograd function is their only caller) -> numpy dict as the reference's."""
    vol = _t(c["vol"] if vol is None else vol).to(dtype)
    pk = Trilinear()._packed_volume(vol) if packed else None
    assert (pk is not None) == packed
    field = _t(dc.pack(c["U"] if U is None else U))
    src, tgt, raylen, field = (x.requires_grad_(grads) for x in (_t(c["src"][:, None]), _t(c["tgt"]), _t(c["raylen"][:, None]), field))
    arange = torch.tensor([c["amin"], c["amax"]], device=DEV, requires_grad=grads)
    grid = (c["H"], c["W"]) if c["H"] else None
    out = dm._DeformFunction.apply(vol, pk, src, tgt, raylen, field, arange, 0.5, 1e-8, c["n_points"], grid)
    res = dict(out=out.detach().cpu().numpy()[:, 0])
    if grads:
        out.backward(_t(c["gout"])[:, None])
        gf = field.grad.cpu().numpy()
        assert np.all(gf[..., 3] == 0)
        res.update(g_src=src.grad.cpu().numpy()[:, 0], g_tgt=tgt.grad.cpu().numpy(), g_raylen=raylen.grad.cpu().numpy()[:, 0],
                   g_U=np.ascontiguousarray(np.moveaxis(gf[..., :3], -1, 1)), g_alphamin=float(arange.grad[0]),
                   g_alphamax=float(arange.grad[1]))
    return res


@pytest.fixture(scope="module", params=sorted(dc.CASES))
def case(request):
    c = dc.CASES[request.param]()
    c["ref"] = do.fwd(*dc.args(c))
    c["gref"] = do.bwd(*dc.args(c)[:5], c["gout"], *dc.args(c)[5:])
    c["g32"] = do.bwd(*dc.args(c)[:5], c["gout"], *dc.args(c)[5:], dtype=np.float32)
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
    for key in ("g_src", "g_U"):
        assert relerr(got[key], ref[key]) <= tc.tol(r32[key], ref[key], FLOOR), key
    scale = tc.alpha_scale(ref["g_raylen"], c["raylen"], c["amin"], c["amax"])
    for key in ("g_alphamin", "g_alphamax"):
        assert abs(got[key] - ref[key]) / scale <= tc.tol(r32[key], ref[key], FLOOR, scale=scale), key


def test_packed_equals_plain_and_repeats(case):
    a, b, again = _kernels(case), _kernels(case, packed=True), _kernels(case)
    for other in (again, b):
        for key in ("out", "g_tgt", "g_raylen", "g_src", "g_alphamin", "g_alphamax"):
            assert np.array_equal(a[key], other[key]), key   # per-ray values and fixed-order sums: bit for bit
        assert relerr(other["g_U"], a["g_U"]) <= REORDER     # atomics: fp32 reordering only


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("packed", [False, True])
def test_16bit_density_equals_fp32_on_the_upcast_volume(dtype, packed):
    c = dc.CASES["per_pose"]()
    up = _t(c["vol"]).to(dtype).float().cpu().numpy()
    a, b = _kernels(c, packed=packed, dtype=dtype), _kernels(c, vol=up)
    for key in a:
        if key == "g_U":
            assert relerr(a[key], b[key]) <= REORDER
        else:
            assert np.array_equal(a[key], b[key]), key


def test_zero_field_in_the_kernels_is_the_trilinear_march(case):
    c = case
    r = Trilinear()
    plain = r(_t(c["vol"]), _t(c["src"][:, None]), _t(c["tgt"]), _t(c["raylen"][:, None]), n_points=c["n_points"],
              alphamin=c["amin"], alphamax=c["amax"]).cpu().numpy()[:, 0]
    assert np.array_equal(_kernels(c, grads=False, U=np.zeros_like(c["U"]))["out"], plain)


# ---- through DRR.render_deformed ------------------------------------------------------------------------------------------------
def _scene(H=40, **kw):
    vol = tc.volume(DIMS)
    lab = np.zeros(DIMS, np.float32)
    lab[8:20, 10:26, 6:18], lab[26:40, 30:48, 20:34], lab[10:22, 34:50, 22:36] = 3, 7, 12
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(H), renderer="trilinear",
              **kw).to(DEV)
    return vol, drr


def _field(B=None, grid=(10, 12, 9), seed=0, amp=10.0):
    """A smooth world-mm field (3, *grid) or (B, 3, *grid) of about `amp` mm."""
    U = dc.smooth_field(np.random.default_rng(seed), 1 if B is None else B, grid, amp)
    return _t(U[0] if B is None else U)


def _rays(drr, rot, xyz):
    """(src (B, 3), tgt (B, N, 3), raylen (B, N)) in voxel-index space, as the module builds them, and the range it would use."""
    with torch.no_grad():
        source, target = drr.detector(convert(rot, xyz, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = drr.affine_inverse(source), drr.affine_inverse(target)
    src, tgt, raylen = (t.cpu().numpy() for t in (src[:, 0], tgt, raylen))
    return src, tgt, raylen, tc.range_of(DIMS, src, tgt)


def _voxel_np(drr, U):
    lin = drr._affine_inverse.reshape(4, 4)[:3, :3].double().cpu().numpy()
    U = U.double().cpu().numpy()
    U = U if U.ndim == 5 else U[None]
    return np.einsum("ij,bjxyz->bixyz", lin, U)


@pytest.mark.parametrize("per_pose", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_module_matches_fp64_reference(per_pose, dtype):
    vol, drr = _scene()
    if dtype != torch.float32:
        drr.density = drr.density.to(dtype)
        vol = drr.density.float().cpu().numpy()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=1))
    U = _field(2 if per_pose else None, seed=2)
    img = drr.render_deformed(rot, xyz, field=U, n_points=150, **KW)
    assert img.shape == (2, 1, 40, 40)
    src, tgt, raylen, (amin, amax) = _rays(drr, rot, xyz)
    ref = do.fwd(vol, src, tgt, raylen, _voxel_np(drr, U), 150, amin, amax)
    assert relerr(img.cpu().numpy().reshape(ref.shape), ref) <= 1e-4
    plain = drr(rot, xyz, n_points=150, **KW)
    assert relerr(img.cpu().numpy(), plain.cpu().numpy()) > 1e-2          # the field does move the image


def test_zero_field_is_forward_bitwise():
    _, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=3))
    plain = drr(rot, xyz, n_points=150, **KW)
    assert torch.equal(drr.render_deformed(rot, xyz, field=torch.zeros(3, 6, 7, 5, device=DEV), n_points=150, **KW), plain)
    assert torch.equal(drr.render_deformed(rot, xyz, field=torch.zeros(2, 3, 6, 7, 5, device=DEV), n_points=150, **KW), plain)


def test_translations_match_render_polyrigid():
    """K purely translational world motions c_k blended by a weight lattice W: render_polyrigid pulls x back to
    x + sum_k w_k(x) A^-1 (-c_k), and so does the node-wise field sum_k W_k (x) (-c_k) (trilinear interpolation is linear).  Images
    and dI/dc_k through both paths agree to round-off; the deformed path's dI/dc_k goes through the field scatter."""
    _, drr = _scene()
    W = polyrigid_weights(drr.mask, (3, 7, 12), grid=(12, 14, 10), sigma=12.0, spacing=(4.0, 4.0, 4.0))
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=4))
    c0 = torch.tensor([[6.0, -4.0, 3.0], [-5.0, 7.0, 2.0], [3.0, 3.0, -8.0]], device=DEV)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(5)).to(DEV)

    def poly(c):
        X = torch.eye(4, device=DEV).repeat(3, 1, 1)
        X[:, :3, 3] = c
        return drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=150, **KW)

    def deformed(c):
        return drr.render_deformed(rot, xyz, field=torch.einsum("kxyz,ki->ixyz", W, -c), n_points=150, **KW)

    grads, imgs = [], []
    for fn in (poly, deformed):
        c = c0.clone().requires_grad_(True)
        img = fn(c)
        (img * gout).sum().backward()
        imgs.append(img.detach().cpu().numpy())
        grads.append(c.grad.cpu().numpy())
    assert relerr(imgs[1], imgs[0]) <= 1e-4
    assert np.abs(grads[0]).max() > 0 and relerr(grads[1], grads[0]) <= 1e-3, (grads[0], grads[1])


@pytest.mark.parametrize("per_pose", [False, True])
def test_autograd_to_pose_and_field_matches_fp64_reference(per_pose):
    """rot, xyz and the world-mm field: the module's autograd against the fp64 reference's gradients chained through the same
    host algebra in float64 (rays, the field conversion and the batch-global range are torch ops in both)."""
    vol, drr = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=6))
    U0 = _field(2 if per_pose else None, seed=7)
    gout = torch.randn(2, 1, 40, 40, generator=torch.Generator().manual_seed(8)).to(DEV)
    rot, xyz, U = (t.clone().requires_grad_(True) for t in (rot0, xyz0, U0))
    img = drr.render_deformed(rot, xyz, field=U, n_points=150, **KW)
    (img * gout).sum().backward()

    def chain(dtype):
        """d loss / d (rot, xyz, field) with the kernels' part replaced by the reference evaluated in `dtype`."""
        host = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40), renderer="trilinear").to(torch.float64)
        r, x, u = (v.detach().cpu().double().requires_grad_(True) for v in (rot0, xyz0, U0))
        source, target = host.detector(convert(r, x, **KW), None)
        raylen = (target - source).norm(dim=-1)
        src, tgt = host.affine_inverse(source)[:, 0], host.affine_inverse(target)
        lin = host._affine_inverse.reshape(4, 4)[:3, :3]
        Uv = torch.einsum("ij,bjxyz->bixyz", lin, u if u.dim() == 5 else u[None])
        dims = torch.tensor(DIMS, dtype=torch.float64)
        from diffdrr_b200.renderers import _get_alpha_minmax
        amin, amax = _get_alpha_minmax(src[:, None], tgt, dims, 0.5, 1e-8)
        amin, amax = amin.min(), amax.max()
        q = do.bwd(vol, src.detach().numpy(), tgt.detach().numpy(), raylen.detach().numpy(), Uv.detach().numpy(),
                   gout.cpu().numpy().reshape(2, -1), 150, float(amin), float(amax), dtype=dtype)
        total = sum((torch.from_numpy(np.asarray(q[k], np.float64)) * v).sum() for k, v in
                    (("g_src", src), ("g_tgt", tgt), ("g_raylen", raylen), ("g_U", Uv)))
        (total + q["g_alphamin"] * amin + q["g_alphamax"] * amax).backward()
        return [v.grad.numpy() for v in (r, x, u)]

    ref, r32 = chain(np.float64), chain(np.float32)
    for got, want, w32, name in zip((rot.grad, xyz.grad, U.grad), ref, r32, ("rot", "xyz", "field")):
        assert np.abs(want).max() > 0
        assert relerr(got.cpu().numpy(), want) <= tc.tol(w32, want, 1e-3), name


def test_subsampled_and_patched_detectors_render_the_same_pixels():
    _, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=9))
    amin, amax = _rays(drr, rot, xyz)[3]       # one explicit range: Trilinear's own is that of the rays in the call
    kw = dict(n_points=120, alphamin=amin, alphamax=amax)
    U = _field(2, seed=10)
    full = drr.render_deformed(rot, xyz, field=U, **KW, **kw)
    _, patched = _scene(patch_size=10)
    assert torch.equal(patched.render_deformed(rot, xyz, field=U, **KW, **kw), full)
    _, sub = _scene(p_subsample=0.3)
    got = sub.render_deformed(rot, xyz, field=U, **KW, **kw)
    pick = sub.detector.pick_tensor()
    assert torch.equal(got.reshape(2, -1)[:, pick], full.reshape(2, -1)[:, pick])
    assert float(got.reshape(2, -1).count_nonzero()) <= 2 * len(pick)


def test_cuda_graph_replays_one_step():
    _, drr = _scene()
    rot0, xyz0 = (t.to(DEV) for t in synthetic.make_poses(2, seed=11))
    U0 = _field(seed=12)
    w = torch.rand(2, 1, 40, 40, device=DEV)

    def step(r, x, u):
        img = drr.render_deformed(r, x, field=u, n_points=100, **KW)
        (img * w).sum().backward()
        return img.detach()

    r_e, x_e, u_e = (t.clone().requires_grad_(True) for t in (rot0, xyz0, U0))
    img_e = step(r_e, x_e, u_e)
    r_d, x_d, u_d = (t.clone().requires_grad_(True) for t in (rot0, xyz0, U0))
    step(r_d, x_d, u_d)   # creates the .grad tensors outside the capture

    def body():
        for t in (r_d, x_d, u_d):
            t.grad.zero_()
        return step(r_d, x_d, u_d)

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
    for a, b in ((r_d, r_e), (x_d, x_e), (u_d, u_e)):
        assert relerr(a.grad.cpu().numpy(), b.grad.cpu().numpy()) < 1e-5


def test_unsupported_combinations_raise_before_any_launch():
    vol, drr = _scene()
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(2, seed=13))
    U = _field()
    call = lambda d=drr, U=U, **kw: d.render_deformed(rot, xyz, field=U, **KW, **kw)   # noqa: E731
    siddon = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(40)).to(DEV)
    torch.cuda.synchronize()
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
    for bad in (U.double(), U[:2], U[None].expand(3, -1, -1, -1, -1), U[0], torch.zeros(2, 3, 4, 0, 4, device=DEV)):
        with pytest.raises(ValueError, match="displacement lattice"):
            call(U=bad)
    with pytest.raises(ValueError, match="density's device"):
        call(U=U.cpu())
    with pytest.raises(NotImplementedError, match="2\\^31"):
        call(U=torch.empty(3, 1024, 1024, 512, device="meta"))
    torch.cuda.synchronize()


def test_registration_lowers_ncc_and_field_error():
    """128^3 phantom, four views at 96^2, a target rendered from a smooth 8^3 world-mm field; Adam on an 8^3 field from zero with
    the test's own smoothness term (squared differences of neighbouring nodes).  One run on an NVIDIA H100 80GB HBM3 (700 W) took
    mean 1 - NCC from 1.80e-3 to 2.76e-4 (6.5x) and the field's RMS error over the nodes inside the body from 4.84 to 3.95 mm
    (1.23x; four views leave much of the field unobserved); the bounds below keep a margin for the field gradient's atomics."""
    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(96), renderer="trilinear").to(DEV)
    rot = torch.tensor([[0.0, 0.0, 0.0], [torch.pi / 2, 0.0, 0.0], [0.0, torch.pi / 2, 0.0], [torch.pi / 4, torch.pi / 4, 0.0]],
                       device=DEV)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=DEV).expand(4, 3).contiguous()
    grid = (8, 8, 8)
    U_true = _field(grid=grid, seed=21, amp=6.0)
    kw = dict(n_points=250, **KW)
    with torch.no_grad():
        target = drr.render_deformed(rot, xyz, field=U_true, **kw)
    # the lattice nodes inside the body: density at the node's voxel above a tenth of the maximum
    idx = [((np.arange(g) + 0.5) * n / g - 0.5).round().astype(int) for g in grid]
    body = torch.from_numpy(vol[np.ix_(*idx)] > 0.1 * vol.max()).to(DEV)
    assert int(body.sum()) >= 20

    def rms(U):
        return float(((U - U_true) ** 2).sum(0)[body].mean().sqrt())

    def smooth(U):
        return sum(((U.diff(dim=a)) ** 2).mean() for a in (1, 2, 3))

    ncc = NormalizedCrossCorrelation2d()
    U = torch.zeros_like(U_true, requires_grad=True)
    opt = torch.optim.Adam([U], lr=0.3)
    steps = 300
    with torch.no_grad():
        loss0 = float((1 - ncc(drr.render_deformed(rot, xyz, field=U, **kw), target)).mean())
    rms0 = rms(U.detach())
    for _ in range(steps):
        opt.zero_grad()
        loss = (1 - ncc(drr.render_deformed(rot, xyz, field=U, **kw), target)).mean()
        (loss + 1e-3 * smooth(U)).backward()
        opt.step()
    with torch.no_grad():
        loss1 = float((1 - ncc(drr.render_deformed(rot, xyz, field=U, **kw), target)).mean())
    rms1 = rms(U.detach())
    print(f"deformable registration after {steps} steps: mean 1 - NCC {loss0:.3e} -> {loss1:.3e} ({loss0 / loss1:.1f}x), field RMS "
          f"error inside the body {rms0:.3f} -> {rms1:.3f} mm ({rms0 / rms1:.2f}x)")
    assert loss0 / loss1 >= 4.0 and rms0 / rms1 >= 1.1, (loss0, loss1, rms0, rms1)
