"""16-bit volumes on the GPU (DESIGN.md 4.5): a density stored as fp16 / bf16 renders the same images and ray / pose gradients as the
fp32 path on its up-cast, through each of the seventeen _v16 entry points (Siddon and Trilinear); against the reference goldens it
stays within the storage error measured on the CPU (test_volume16_cpu.py); every option outside the contract raises; the
registration loop converges from an fp16 density under a CUDA graph; and the density and the packed trilinear copy take half the
bytes, with no up-cast copy."""
import numpy as np
import pytest
import torch

from conftest import load_golden, relerr
from gpu_common import DEV

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
IMG_TOL, GRAD_TOL = 1e-6, 1e-5


@pytest.fixture
def calls(monkeypatch):
    """Names of the _v16 entry points the renderers call."""
    from diffdrr_b200 import _lib
    lib = _lib.load()
    seen = []
    for name in _lib.exported_symbols():
        if name.endswith("_v16"):
            fn = getattr(lib, name)

            def wrap(*a, _fn=fn, _name=name):
                seen.append(_name)
                return _fn(*a)
            monkeypatch.setattr(lib, name, wrap)
    return seen


def _pair(vol_np, dtype, **kw):
    """(DRR on the 16-bit density, DRR on its fp32 up-cast)."""
    from diffdrr_b200 import DRR, synthetic
    v16 = torch.from_numpy(vol_np).to(dtype)
    torch.manual_seed(0)   # the same detector sub-sample on both
    d16 = DRR(synthetic.make_subject(v16), **kw).to(DEV)
    torch.manual_seed(0)
    d32 = DRR(synthetic.make_subject(v16.float()), **kw).to(DEV)
    assert d16.density.dtype == dtype and d16.dtype == torch.float32 and d32.density.dtype == torch.float32
    return d16, d32


def _render(drr, rot, xyz, train):
    rot, xyz = rot.clone().to(DEV), xyz.clone().to(DEV)
    if not train:
        with torch.no_grad():
            return drr(rot, xyz, parameterization="euler_angles", convention="ZXY"), None
    rot.requires_grad_(True)
    xyz.requires_grad_(True)
    img = drr(rot, xyz, parameterization="euler_angles", convention="ZXY")
    w = torch.linspace(0.5, 1.5, img.numel(), device=DEV).view_as(img)
    (img * w).sum().backward()
    return img.detach(), (rot.grad, xyz.grad)


def _check(d16, d32, B, train, seed=3, img_tol=IMG_TOL, grad_tol=GRAD_TOL):
    from diffdrr_b200 import synthetic
    rot, xyz = synthetic.make_poses(B, seed=seed)
    if B == 1:
        rot = rot + torch.tensor([[0.1, -0.05, 0.08]])
    a, ga = _render(d16, rot, xyz, train)
    b, gb = _render(d32, rot, xyz, train)
    assert float(b.abs().max()) > 0
    assert relerr(a.cpu().numpy(), b.cpu().numpy()) <= img_tol
    if train:
        # The brick kernel's sensitivities are summed over bricks with atomics in the order the CTAs claim the bricks, so the pose
        # gradient (a sum over all rays, with cancellation) moves between two fp32 runs as well: allow 3x that run-to-run spread.
        reruns = [_render(d32, rot, xyz, train)[1] for _ in range(3)]
        for i, (x, y) in enumerate(zip(ga, gb)):
            noise = max(relerr(g[i].cpu().numpy(), y.cpu().numpy()) for g in reruns)
            err = relerr(x.cpu().numpy(), y.cpu().numpy())
            print(f"pose gradient {i}: 16-bit vs fp32 {err:.2e}, fp32 run-to-run {noise:.2e}")
            assert err <= max(grad_tol, 3.0 * noise), (err, noise)


# ---- exactness against the fp32 path, one case per route --------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("train", [False, True])
def test_full_grid_one_pose_pieces(dtype, train, calls):
    from diffdrr_b200 import synthetic
    d16, d32 = _pair(synthetic.make_volume(192, "phantom", seed=1), dtype, **synthetic.detector_kwargs(96))
    _check(d16, d32, 1, train)
    assert calls[-1] == ("b200drr_siddon_fwd_sens_pose_v16" if train else "b200drr_siddon_fwd_pose_v16")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("train", [False, True])
def test_full_grid_four_poses_brick(dtype, train, calls):
    """384^3 -> 160^2: 2304 bricks, sparse rays, 4 poses -- the brick kernel in pose-in mode (inference) and sensitivities mode."""
    from diffdrr_b200 import synthetic
    d16, d32 = _pair(synthetic.make_volume(384, "phantom", seed=2), dtype, **synthetic.detector_kwargs(160))
    # training: the brick kernel's atomics make the fp32 pose gradient itself vary between runs (see _check)
    _check(d16, d32, 4, train)
    assert calls[-1] == ("b200drr_siddon_fwd_sens_pose_v16" if train else "b200drr_siddon_fwd_brick_v16")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,train,entry", [(1, False, "b200drr_siddon_fwd_grid_v16"), (4, False, "b200drr_siddon_fwd_brick_v16"),
                                           (2, True, "b200drr_siddon_fwd_sens_grid_v16")])
def test_render_with_ray_tensors(dtype, B, train, entry, calls, monkeypatch):
    """DRR.render on the full grid's ray tensors: the tiled grid kernels and the brick kernel in ray-tensor mode."""
    from diffdrr_b200 import renderers, synthetic
    from diffdrr_b200.pose import convert
    monkeypatch.setattr(renderers, "_BRICK_MIN_BRICKS", 1)
    d16, d32 = _pair(synthetic.make_volume(256, "phantom", seed=4), dtype, **synthetic.detector_kwargs(160))
    rot, xyz = synthetic.make_poses(B, seed=5)
    out = []
    for drr in (d16, d32):
        src, tgt = drr.detector(convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        tgt = tgt.detach().requires_grad_(train)
        img = drr.render(drr.density, src, tgt)
        g = None
        if train:
            img.sum().backward()
            g = tgt.grad.cpu().numpy()
        out.append((img.detach().cpu().numpy(), g))
    assert entry in calls
    assert relerr(out[0][0], out[1][0]) <= IMG_TOL
    if train:
        assert relerr(out[0][1], out[1][1]) <= GRAD_TOL


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,train,entry", [(4, False, "b200drr_siddon_fwd_brick_subset_v16"),
                                           (1, False, "b200drr_siddon_fwd_sorted_v16"),
                                           (2, True, "b200drr_siddon_fwd_sens_sorted_v16")])
def test_subsampled_detector(dtype, B, train, entry, calls, monkeypatch):
    from diffdrr_b200 import renderers, synthetic
    monkeypatch.setattr(renderers, "_BRICK_MIN_BRICKS", 1)
    vol = synthetic.make_volume(128, "phantom", seed=6)
    d16, d32 = _pair(vol, dtype, **synthetic.detector_kwargs(96), p_subsample=0.3)
    _check(d16, d32, B, train)
    assert entry in calls


@pytest.mark.parametrize("dtype", DTYPES)
def test_patches(dtype, calls):
    from diffdrr_b200 import synthetic
    d16, d32 = _pair(synthetic.make_volume(96, "phantom", seed=7), dtype, **synthetic.detector_kwargs(48), patch_size=12)
    _check(d16, d32, 2, False)
    _check(d16, d32, 2, True)
    assert "b200drr_siddon_fwd_v16" in calls and "b200drr_siddon_fwd_sens_v16" in calls   # 144-ray patches


@pytest.mark.parametrize("dtype", DTYPES)
def test_user_rays_under_1024(dtype, calls):
    from diffdrr_b200 import Siddon
    rng = np.random.default_rng(8)
    vol = torch.from_numpy(rng.random((40, 48, 56), dtype=np.float32)).to(dtype).to(DEV)
    src = torch.tensor([[[-30.0, 20.0, 25.0]], [[70.0, 10.0, 30.0]]], device=DEV)
    tgt = torch.from_numpy(rng.uniform(-5, 60, (2, 300, 3)).astype(np.float32)).to(DEV)
    raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
    res = []
    for v in (vol, vol.float()):
        t = tgt.clone().requires_grad_(True)
        with torch.no_grad():
            inf = Siddon()(v, src, tgt, raylen)
        img = Siddon()(v, src, t, raylen)
        img.sum().backward()
        res.append((inf.cpu().numpy(), img.detach().cpu().numpy(), t.grad.cpu().numpy()))
    assert "b200drr_siddon_fwd_v16" in calls and "b200drr_siddon_fwd_sens_v16" in calls
    for a, b in zip(res[0][:2], res[1][:2]):
        assert relerr(a, b) <= IMG_TOL
    assert relerr(res[0][2], res[1][2]) <= GRAD_TOL


@pytest.mark.parametrize("dtype", DTYPES)
def test_d2_not_a_multiple_of_8_takes_the_slab_path(dtype, calls):
    """384 x 384 x 388: the fp32 volume's rows are 16-byte multiples (brick kernel), the 16-bit volume's are not (776 bytes): it
    takes the slab-major / pieces kernels and agrees with the fp32 brick path to the summation-order rounding."""
    from diffdrr_b200 import renderers, synthetic
    vol = synthetic.make_volume((384, 384, 388), "phantom", seed=9)
    d16, d32 = _pair(vol, dtype, **synthetic.detector_kwargs(128))
    assert renderers._brick_ok(d32.density, 4, 128, 128) and not renderers._brick_ok(d16.density, 4, 128, 128)
    _check(d16, d32, 4, False, img_tol=1e-5)
    _check(d16, d32, 4, True, img_tol=1e-5, grad_tol=1e-4)
    assert "b200drr_siddon_fwd_brick_v16" not in calls and "b200drr_siddon_fwd_pose_v16" in calls


def test_assigning_a_16bit_density_to_an_existing_module():
    from diffdrr_b200 import DRR, synthetic
    vol = synthetic.make_volume(64, "phantom", seed=10)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(32)).to(DEV)
    drr.density = drr.density.to(torch.bfloat16)
    assert drr.dtype == torch.float32
    drr.set_intrinsics_(height=40, width=40)
    assert drr.detector.target.dtype == torch.float32 and drr.detector.target.is_cuda
    ref = DRR(synthetic.make_subject(torch.from_numpy(vol).to(torch.bfloat16).float()), **synthetic.detector_kwargs(32)).to(DEV)
    ref.set_intrinsics_(height=40, width=40)
    _check(drr, ref, 2, True)


# ---- against the reference goldens ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["siddon_nc_b4", "siddon_nc_b4_ragged", "siddon_nc_inside", "siddon_c1", "siddon_nc_axis"])
def test_goldens_within_the_storage_error(name, dtype):
    """The bar is the C oracle's error on the same rounded volume (the storage error measured in test_volume16_cpu.py) plus 2e-5."""
    from diffdrr_b200 import Siddon
    from oracle import oracle
    g = load_golden(name)
    v16 = torch.from_numpy(g["volume"]).to(dtype)
    storage = relerr(oracle.siddon_fwd(v16.float().numpy(), g["source"], g["target"], g["raylen"]), g["img_f32"])
    src, tgt, raylen = (torch.from_numpy(g[k]).to(DEV) for k in ("source", "target", "raylen"))
    img = Siddon()(v16.to(DEV), src, tgt, raylen)
    assert relerr(img.cpu().numpy(), g["img_f32"]) < storage + 2e-5


# ---- what raises ------------------------------------------------------------------------------------------------------------------
def test_everything_outside_the_contract_raises():
    from diffdrr_b200 import DRR, Siddon, Trilinear, synthetic
    vol = torch.from_numpy(synthetic.make_volume(24, "phantom")).to(torch.float16).to(DEV)
    src = torch.tensor([[[-20.0, 12.0, 12.0]]], device=DEV)
    tgt = torch.rand(1, 20, 3, device=DEV) * 20 + torch.tensor([40.0, 2.0, 2.0], device=DEV)
    raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
    with pytest.raises(NotImplementedError, match="cannot require grad"):
        Siddon()(vol.clone().requires_grad_(True), src, tgt, raylen)
    for kw in (dict(mode="bilinear"), dict(reducefn="max"), dict(reducefn=lambda x: x.sum(-1))):
        with pytest.raises(NotImplementedError, match="default Siddon options"):
            Siddon(**kw)(vol, src, tgt, raylen)
    with pytest.raises(NotImplementedError, match="default Siddon options"):
        Siddon()(vol, src, tgt, raylen, align_corners=True)
    with pytest.raises(NotImplementedError, match="default Siddon options"):
        Siddon()(vol, src, tgt, raylen, mask=torch.zeros_like(vol, dtype=torch.float32))
    with pytest.raises(NotImplementedError, match="fp32 rays"):
        Siddon()(vol, src.half(), tgt.half(), raylen.half())
    with pytest.raises(NotImplementedError, match="cannot require grad"):
        Trilinear()(vol.clone().requires_grad_(True), src, tgt, raylen)
    for kw in (dict(reducefn="max"), dict(reducefn=lambda x: x.sum(-1))):
        with pytest.raises(NotImplementedError, match="default Trilinear options"):
            Trilinear(**kw)(vol, src, tgt, raylen)
    with pytest.raises(NotImplementedError, match="default Trilinear options"):
        Trilinear()(vol, src, tgt, raylen, align_corners=True)
    with pytest.raises(NotImplementedError, match="default Trilinear options"):
        Trilinear()(vol, src, tgt, raylen, mask=torch.zeros_like(vol, dtype=torch.float32))
    with pytest.raises(NotImplementedError, match="fp32 rays"):
        Trilinear()(vol, src.half(), tgt.half(), raylen.half(), alphamin=0.0, alphamax=1.0)
    drr = DRR(synthetic.make_subject(vol.cpu()), **synthetic.detector_kwargs(16)).to(DEV)
    rot, xyz = synthetic.make_poses(1)
    drr.half()   # the whole module in 16 bits: 16-bit rays and poses
    with pytest.raises(NotImplementedError, match="fp32 rays"):
        drr(rot.to(DEV).half(), xyz.to(DEV).half(), parameterization="euler_angles", convention="ZXY")
    drr = DRR(synthetic.make_subject(vol.cpu()), **synthetic.detector_kwargs(16)).to(DEV).to(torch.bfloat16)
    with pytest.raises(NotImplementedError, match="fp32 rays"):
        drr(rot.to(DEV).bfloat16(), xyz.to(DEV).bfloat16(), parameterization="euler_angles", convention="ZXY")


# ---- the registration loop from an fp16 density ------------------------------------------------------------------------------------
def test_registration_loop_converges_from_an_fp16_density_under_a_cuda_graph():
    """test_gpu_registration.test_registration_loop_converges (graph=True) with the density stored in fp16: same start, bounds."""
    from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, Registration, synthetic
    vol = torch.from_numpy(synthetic.make_volume(128, "smooth", seed=1)).to(torch.float16)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(96), renderer="siddon",
              stop_gradients_through_grid_sample=True).to(DEV)
    true_rot, true_xyz = torch.tensor([[0.0, 0.0, 0.0]], device=DEV), torch.tensor([[0.0, 850.0, 0.0]], device=DEV)
    with torch.no_grad():
        target = drr(true_rot, true_xyz, parameterization="euler_angles", convention="ZXY")
    reg = Registration(drr, (true_rot + torch.tensor([[0.12, -0.08, 0.06]], device=DEV)).clone(),
                       (true_xyz + torch.tensor([[10.0, -20.0, 8.0]], device=DEV)).clone(), "euler_angles", "ZXY").to(DEV)
    ncc = NormalizedCrossCorrelation2d()
    opt = torch.optim.Adam([{"params": [reg.rotation], "lr": 5e-3}, {"params": [reg.translation], "lr": 5e-1}], capturable=True)

    def step():
        opt.zero_grad(set_to_none=False)
        loss = 1.0 - ncc(target, reg()).mean()
        loss.backward()
        opt.step()
        return loss

    with torch.no_grad():
        start = float(1.0 - ncc(target, reg()).mean())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(400):
        g.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        final = float(1.0 - ncc(target, reg()).mean())
    assert drr.density.dtype == torch.float16
    assert start > 0.02 and final < 1e-3 and final < 0.05 * start
    assert float((reg.rotation.detach() - true_rot).abs().max()) < 0.02
    assert float((reg.translation.detach() - true_xyz).abs().max()) < 2.0


# ---- memory ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_512_cubed_density_takes_half_the_bytes_and_is_never_upcast(dtype):
    from diffdrr_b200 import DRR, synthetic
    D, H, B = 512, 256, 16
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H)).to(DEV)
    base = torch.cuda.memory_allocated()
    drr.density = torch.rand(D, D, D, device=DEV, dtype=torch.float32).to(dtype)
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated() - base
    assert resident < 0.52 * 4 * D ** 3          # half of the fp32 volume's 512 MiB (+ detector buffers)
    rot, xyz = synthetic.make_poses(B, seed=1)
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    _render(drr, rot, xyz, True)
    with torch.no_grad():
        drr(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - before
    assert peak < D ** 3                           # images, sensitivities, gradients: nothing near the 16-bit volume's 2 D^3 bytes


# ---- Trilinear -------------------------------------------------------------------------------------------------------------------
def _tri_pair(dtype, D=96, H=48, pack=True):
    from diffdrr_b200 import synthetic
    d16, d32 = _pair(synthetic.make_volume(D, "phantom", seed=11), dtype, **synthetic.detector_kwargs(H), renderer="trilinear")
    d16.renderer.pack_corners = d32.renderer.pack_corners = pack
    return d16, d32


def _tri_check(d16, d32, B, train, n_points=200):
    from diffdrr_b200 import synthetic
    rot, xyz = synthetic.make_poses(B, seed=12)
    out = []
    for drr in (d16, d32):
        r, x = rot.clone().to(DEV), xyz.clone().to(DEV)
        if train:
            r.requires_grad_(True)
            x.requires_grad_(True)
            img = drr(r, x, parameterization="euler_angles", convention="ZXY", n_points=n_points)
            (img * torch.linspace(0.5, 1.5, img.numel(), device=DEV).view_as(img)).sum().backward()
            out.append((img.detach(), r.grad, x.grad))
        else:
            with torch.no_grad():
                out.append((drr(r, x, parameterization="euler_angles", convention="ZXY", n_points=n_points),))
    assert float(out[1][0].abs().max()) > 0
    assert relerr(out[0][0].cpu().numpy(), out[1][0].cpu().numpy()) <= IMG_TOL
    for a, b in zip(out[0][1:], out[1][1:]):
        assert relerr(a.cpu().numpy(), b.cpu().numpy()) <= GRAD_TOL


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", [1, 2])
def test_trilinear_packed_grid_inference(dtype, B, calls):
    d16, d32 = _tri_pair(dtype)
    _tri_check(d16, d32, B, False)
    assert calls == ["b200drr_pack_corners_v16", "b200drr_trilinear_fwd_packed_v16"]
    packed = d16.renderer._packed
    assert packed.numel() * 4 == 97 ** 3 * 8 * 2  # 16 B per base voxel


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", [1, 3])
def test_trilinear_training_through_drr_forward(dtype, B, calls):
    """The fused pose-in march over the 16-bit packed copy (b200drr_trilinear_fwd_sens_pose_v16)."""
    d16, d32 = _tri_pair(dtype)
    _tri_check(d16, d32, B, True)
    assert "b200drr_trilinear_fwd_sens_pose_v16" in calls


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("train", [False, True])
def test_trilinear_without_packed_copy(dtype, train, calls):
    d16, d32 = _tri_pair(dtype, pack=False)
    _tri_check(d16, d32, 2, train)
    assert calls[-1] == ("b200drr_trilinear_fwd_sens_v16" if train else "b200drr_trilinear_fwd_grid_v16")
    assert "b200drr_pack_corners_v16" not in calls


@pytest.mark.parametrize("dtype", DTYPES)
def test_trilinear_render_with_ray_gradients_from_the_packed_copy(dtype, calls):
    from diffdrr_b200 import synthetic
    from diffdrr_b200.pose import convert
    d16, d32 = _tri_pair(dtype)
    rot, xyz = synthetic.make_poses(2, seed=13)
    out = []
    for drr in (d16, d32):
        src, tgt = drr.detector(convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        tgt = tgt.detach().requires_grad_(True)
        img = drr.render(drr.density, src, tgt, n_points=150)
        img.sum().backward()
        out.append((img.detach().cpu().numpy(), tgt.grad.cpu().numpy()))
    assert "b200drr_trilinear_fwd_sens_packed_v16" in calls
    assert relerr(out[0][0], out[1][0]) <= IMG_TOL and relerr(out[0][1], out[1][1]) <= GRAD_TOL


@pytest.mark.parametrize("dtype", DTYPES)
def test_trilinear_arbitrary_rays(dtype, calls):
    from diffdrr_b200 import Trilinear
    rng = np.random.default_rng(14)
    vol = torch.from_numpy(rng.random((40, 48, 56), dtype=np.float32)).to(dtype).to(DEV)
    src = torch.tensor([[[-30.0, 20.0, 25.0]], [[70.0, 10.0, 30.0]]], device=DEV)
    tgt = torch.from_numpy(rng.uniform(-5, 60, (2, 300, 3)).astype(np.float32)).to(DEV)
    raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
    res = []
    for v in (vol, vol.float()):
        with torch.no_grad():
            inf = Trilinear()(v, src, tgt, raylen, n_points=120)
        t = tgt.clone().requires_grad_(True)
        img = Trilinear()(v, src, t, raylen, n_points=120)
        img.sum().backward()
        res.append((inf.cpu().numpy(), img.detach().cpu().numpy(), t.grad.cpu().numpy()))
    assert "b200drr_trilinear_fwd_v16" in calls and "b200drr_trilinear_fwd_sens_v16" in calls
    assert relerr(res[0][0], res[1][0]) <= IMG_TOL and relerr(res[0][1], res[1][1]) <= IMG_TOL
    assert relerr(res[0][2], res[1][2]) <= GRAD_TOL


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name,n_points", [("trilinear_nc_b4", 160), ("trilinear_nc_b4_ragged", 77), ("trilinear_nc_inside", 150),
                                           ("trilinear_c1", 500), ("trilinear_nc_axis", 200)])
def test_trilinear_goldens_within_the_storage_error(name, n_points, dtype):
    """The bar is the C oracle's error on the same rounded volume (test_volume16_cpu.py) plus 2e-5."""
    from diffdrr_b200 import Trilinear
    from oracle import oracle
    g = load_golden(name)
    v16 = torch.from_numpy(g["volume"]).to(dtype)
    ref = oracle.trilinear_fwd(v16.float().numpy(), g["source"], g["target"], g["raylen"], n_points=n_points)
    storage = relerr(ref, g["img_f32"])
    src, tgt, raylen = (torch.from_numpy(g[k]).to(DEV) for k in ("source", "target", "raylen"))
    img = Trilinear()(v16.to(DEV), src, tgt, raylen, n_points=n_points)
    assert relerr(img.cpu().numpy(), g["img_f32"]) < storage + 2e-5


@pytest.mark.parametrize("dtype", DTYPES)
def test_512_cubed_packed_trilinear_copy_takes_half_the_bytes(dtype):
    from diffdrr_b200 import DRR, _lib, synthetic
    D = 512
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(64), renderer="trilinear").to(DEV)
    drr.density = torch.rand(D, D, D, device=DEV, dtype=torch.float32).to(dtype)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    packed = drr.renderer._packed_volume(drr.density)
    torch.cuda.synchronize()
    fp32_bytes = int(_lib.load().b200drr_packed_volume_floats(D, D, D)) * 4
    assert packed.numel() * packed.element_size() == fp32_bytes // 2
    assert torch.cuda.max_memory_allocated() - before <= fp32_bytes // 2 + (1 << 21)   # the copy only, no fp32 staging
