"""Direct oracle parity for the PRODUCTION kernels at the BASELINE.json configurations (VERDICT r1 item 2).

Every test calls the C ABI entry point the product uses at that size -- the slab-major / brick-major Siddon kernels with
more than one slab / many bricks, the packed-corner trilinear kernels -- and compares full images (and gradients) with the
fp64 oracle on the same rays.  The oracle needs ~0.1-0.3 s per 512^3 -> 256^2 DRR on the GPU box's host cores."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import relerr
from gpu_common import DEV

pytestmark = pytest.mark.gpu

IMG_TOL = 1e-4  # north_star: <= 1e-4 relative error


def _setup(D, H, B, seed=0, kind="rand"):
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import convert
    vol_np = synthetic.make_volume(D, kind, seed=seed)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H)).to(DEV)
    rot, xyz = synthetic.make_poses(max(B, 2), seed=seed)
    rot, xyz = rot[:B], xyz[:B]
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
        src = drr.affine_inverse(src).reshape(B, 3).contiguous()
        tgt = drr.affine_inverse(tgt).contiguous()
    vol = torch.as_tensor(vol_np).to(DEV)
    return vol_np, vol, src, tgt, raylen


def _np(*ts):
    return [x.detach().cpu().numpy() for x in ts]


def _p(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from diffdrr_b200 import _lib as L
    return L, L.load()


@pytest.mark.parametrize("D,H,B", [(512, 256, 8), (256, 256, 16)])
def test_siddon_forward_grid_kernels_vs_oracle(D, H, B):
    """b200drr_siddon_fwd_grid -- the library's default for the batch (512^3 x 8: rays cut into 16 pieces along their major axis;
    256^3 x 16: slab-major) AND the slab-major kernel explicitly (variant 15: 16 slabs of 32 planes at 512^3) -- and
    b200drr_siddon_fwd_brick (TMA bricks: 22x16x16 of them), full images of rotated poses, against the fp64 oracle: the metric's
    configuration and BASELINE config 2 (256^3, B=16)."""
    from oracle import oracle
    L, lib = _lib()
    vol_np, vol, src, tgt, raylen = _setup(D, H, B)
    ref = oracle.siddon_fwd(vol_np, *_np(src, tgt, raylen), dtype=np.float64).reshape(B, -1)
    out = torch.full((B, H * H), float("nan"), device=DEV)
    for variant in (0, 15):
        out.fill_(float("nan"))
        L.check(lib.b200drr_siddon_fwd_grid(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out), B, H, H, 0.5, 1e-8, variant,
                                            _stream()), "fwd_grid")
        assert relerr(out.cpu().numpy(), ref) < IMG_TOL, variant
    ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(B, H, H), dtype=torch.uint8, device=DEV)
    out.fill_(float("nan"))
    L.check(lib.b200drr_siddon_fwd_brick(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), None, None, None, None, _p(out),
                                         ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, H, H, 0.5, 1e-8, 0, _stream()),
            "fwd_brick")
    assert relerr(out.cpu().numpy(), ref) < IMG_TOL


def test_brick_forward_pose_in_and_module_routing(monkeypatch):
    """The brick kernel with rays generated in-kernel from the pose matrices (the DRR module's inference path for batches):
    same images as the slab-major pose-in kernel on the same matrices (fp32 round-off), and both within the north star's
    1e-4 of the oracle on all but the handful of rays that run almost inside a voxel-boundary plane -- there the line
    integral jumps with the ray's position, and the in-kernel rays differ from the torch-chain rays by ~1e-4 voxel."""
    from diffdrr_b200 import DRR, renderers, synthetic
    from diffdrr_b200.pose import convert
    from oracle import oracle
    monkeypatch.setattr(renderers, "_BRICK_MIN_BRICKS", 1)   # 256^3 is below the production threshold: force the brick path
    monkeypatch.setattr(renderers, "_BRICK_FULL_GRID_MIN_LOAD", 0.0)   # ... and 5 poses are below the brick kernel's batch range
    D, H, B = 256, 192, 5
    vol_np = synthetic.make_volume(D, "rand", seed=2)
    drr = DRR(synthetic.make_subject(vol_np), **synthetic.detector_kwargs(H)).to(DEV)
    rot, xyz = synthetic.make_poses(B, seed=4)
    with torch.no_grad():
        img = drr(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
        monkeypatch.setattr(renderers, "_BRICK_MIN_BATCH", 10 ** 9)   # same call through the library's own pose-in kernel
        img_slab = drr(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
        src, tgt = drr.detector(convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
    assert relerr(img.cpu().numpy(), img_slab.cpu().numpy()) < 5e-5   # two decompositions of the same fp32 sums
    ref = oracle.siddon_fwd(vol_np, *_np(src, tgt, raylen), dtype=np.float64)
    got = img.cpu().numpy().reshape(ref.shape)
    err = np.abs(got - ref) / np.abs(ref).max()
    assert (err > IMG_TOL).sum() <= 5 and err.max() < 1e-3 and float(np.sqrt((err ** 2).mean())) < 1e-5


# 0: the default for 2 poses (rays cut into 16 major-axis pieces); 41: 16-plane slabs, the default of the 16-pose training step;
# 38: 48-plane slabs
@pytest.mark.parametrize("variant", [0, 41, 38])
def test_siddon_sensitivities_and_volume_gradient_vs_oracle(variant):
    """b200drr_siddon_fwd_sens_grid + _bwd_sens (the training step's dominant kernel) and b200drr_siddon_bwd_grid
    WITH g_vol (reconstruction) at 512^3 -> 256^2, rotated poses, against the fp64 closed form.  Smooth volume for the
    end-point gradients (SURVEY 8c: on noise the reference's own fp32 is 1e-2 off), noise for image / volume gradient."""
    from oracle import oracle
    L, lib = _lib()
    D, H, B = 512, 256, 2
    N = H * H
    vol_np, vol, src, tgt, raylen = _setup(D, H, B, kind="smooth")
    gout = torch.rand(B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    ref = oracle.siddon_bwd(vol_np, *_np(src, tgt, raylen, gout), dtype=np.float64, want_vol=True)
    ref_img = oracle.siddon_fwd(vol_np, *_np(src, tgt, raylen), dtype=np.float64).reshape(B, N)
    out = torch.empty(B, N, device=DEV)
    sens = torch.empty(B, N, 8, device=DEV)
    L.check(lib.b200drr_siddon_fwd_sens_grid(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out), _p(sens), B, H, H, 0.5,
                                             1e-8, variant, _stream()), "fwd_sens_grid")
    g_src, g_tgt, g_len = torch.empty(B, 3, device=DEV), torch.empty(B, N, 3, device=DEV), torch.empty(B, N, device=DEV)
    L.check(lib.b200drr_siddon_bwd_sens(_p(sens), _p(gout), _p(g_src), _p(g_tgt), _p(g_len), B, N, 0, _stream()), "bwd_sens")
    assert relerr(out.cpu().numpy(), ref_img) < IMG_TOL
    assert relerr(g_tgt.cpu().numpy(), ref["g_target"]) < 2e-3
    assert relerr(g_src.cpu().numpy(), ref["g_source"].reshape(B, 3)) < 2e-3
    assert relerr(g_len.cpu().numpy(), ref["g_raylen"].reshape(B, N)) < IMG_TOL
    if variant != 0:
        return
    # two-walk backward with the volume gradient
    g_vol = torch.zeros_like(vol)
    g_src2, g_tgt2, g_len2 = torch.empty_like(g_src), torch.empty_like(g_tgt), torch.empty_like(g_len)
    L.check(lib.b200drr_siddon_bwd_grid(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), _p(gout), _p(g_src2), _p(g_tgt2),
                                        _p(g_len2), _p(g_vol), B, H, H, 0.5, 1e-8, 0, 0, _stream()), "bwd_grid")
    # per-voxel gradients: which of two neighbouring voxels receives a segment that ends within position round-off of their
    # common plane is decided differently by ANY fp32 evaluation (the rays start ~1700 voxels away: ~1e-4 voxel of round-off),
    # so the bar is the reference algorithm's own fp32-vs-fp64 disagreement (SURVEY 8c rule), not a fixed 1e-4
    ref32 = oracle.siddon_bwd(vol_np, *_np(src, tgt, raylen, gout), dtype=np.float32, want_vol=True)
    tol = max(IMG_TOL, 2.0 * relerr(ref32["g_volume"], ref["g_volume"]))
    assert relerr(g_vol.cpu().numpy(), ref["g_volume"]) < tol
    assert abs(float(g_vol.double().sum()) - float(ref["g_volume"].sum())) < 1e-5 * abs(float(ref["g_volume"].sum()))
    assert relerr(g_tgt2.cpu().numpy(), ref["g_target"]) < 2e-3
    assert relerr(g_src2.cpu().numpy(), ref["g_source"].reshape(B, 3)) < 2e-3
    assert relerr(g_len2.cpu().numpy(), ref["g_raylen"].reshape(B, N)) < IMG_TOL


def test_trilinear_packed_kernels_vs_oracle_config3_shape():
    """BASELINE config 3's shape (512^3 -> 512^2, n_points = 500) on 8 poses: the slab-major packed forward and the packed
    forward-with-sensitivities + elementwise backward, against the fp64 oracle (image) and its closed-form gradients."""
    from oracle import oracle
    L, lib = _lib()
    D, H, B, P = 512, 512, 8, 500
    N = H * H
    vol_np, vol, src, tgt, raylen = _setup(D, H, B, kind="smooth")
    amin, amax = oracle.alpha_minmax(vol_np.shape, *_np(src, tgt), 0.5, 1e-8, np.float32)
    arange = torch.tensor([amin, amax], dtype=torch.float32, device=DEV)
    packed = torch.empty(int(lib.b200drr_packed_volume_floats(D, D, D)), device=DEV)
    L.check(lib.b200drr_pack_corners(_p(vol), D, D, D, _p(packed), _stream()), "pack")
    sub = slice(0, N, 61)  # oracle on ~4300 rays per pose spread over the detector (500 samples each)
    args = (vol_np, src.cpu().numpy(), tgt[:, sub].cpu().numpy(), raylen[:, sub].cpu().numpy())
    ref = oracle.trilinear_fwd(*args, n_points=P, alphamin=amin, alphamax=amax, dtype=np.float64).reshape(B, -1)
    out = torch.full((B, N), float("nan"), device=DEV)
    L.check(lib.b200drr_trilinear_fwd_packed(_p(packed), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out), B, H, H, 0.5, 1e-8, P,
                                             _p(arange), 16, _stream()), "fwd_packed slab")
    assert relerr(out[:, sub].cpu().numpy(), ref) < IMG_TOL
    sens = torch.empty(B, N, 12, device=DEV)
    out2 = torch.full((B, N), float("nan"), device=DEV)
    L.check(lib.b200drr_trilinear_fwd_sens_packed(_p(packed), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out2), _p(sens), B, H, H,
                                                  0.5, 1e-8, P, _p(arange), 0, _stream()), "fwd_sens_packed")
    assert relerr(out2[:, sub].cpu().numpy(), ref) < IMG_TOL
    gout = torch.zeros(B, N, device=DEV)
    gout[:, sub] = torch.rand(B, ref.shape[1], device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    g_src, g_tgt, g_len = torch.empty(B, 3, device=DEV), torch.empty(B, N, 3, device=DEV), torch.empty(B, N, device=DEV)
    g_ar = torch.zeros(2, device=DEV)
    L.check(lib.b200drr_trilinear_bwd_sens(_p(sens), _p(gout), _p(g_src), _p(g_tgt), _p(g_len), _p(g_ar), B, N, _stream()),
            "tri bwd_sens")
    gref = oracle.trilinear_bwd(*args, gout[:, sub].cpu().numpy(), n_points=P, alphamin=amin, alphamax=amax, dtype=np.float64,
                                want_vol=False)
    assert relerr(g_tgt[:, sub].cpu().numpy(), gref["g_target"]) < 2e-3
    assert relerr(g_src.cpu().numpy(), gref["g_source"].reshape(B, 3)) < 2e-3
    assert relerr(g_len[:, sub].cpu().numpy(), gref["g_raylen"].reshape(B, -1)) < IMG_TOL


def test_sorted_arbitrary_ray_sets_match_plain_kernels_and_goldens(monkeypatch):
    """Arbitrary ray sets (sub-sampled detector, ragged user rays) go through the locality-ordered slab-major kernels
    (b200drr_siddon_fwd_sorted / _fwd_sens_sorted): same images and gradients as the one-thread-per-ray kernels, on the
    ragged golden recorded from the reference and on a 25 % random sub-sample of the metric's detector at 512^3."""
    from conftest import load_golden
    from diffdrr_b200 import Siddon, renderers
    from gpu_common import t
    # (1) the ragged golden through the sorted kernels (forced: it has fewer rays than the production threshold)
    g = load_golden("siddon_nc_b4_ragged")
    monkeypatch.setattr(renderers, "_SORT_MIN_RAYS", 1)
    vol, src, tgt, img = t(g["volume"]), t(g["source"], True), t(g["target"], True), t(g["raylen"], True)
    out = Siddon()(vol, src, tgt, img)
    assert relerr(out.detach().cpu().numpy(), g["img_f64"]) < IMG_TOL
    out.sum().backward()
    monkeypatch.setattr(renderers, "_SORT_MIN_RAYS", 10 ** 9)
    src2, tgt2, img2 = t(g["source"], True), t(g["target"], True), t(g["raylen"], True)
    out2 = Siddon()(vol, src2, tgt2, img2)
    out2.sum().backward()
    assert relerr(out.detach().cpu().numpy(), out2.detach().cpu().numpy()) < 2e-5
    assert relerr(tgt.grad.cpu().numpy(), tgt2.grad.cpu().numpy()) < 1e-4
    assert relerr(src.grad.cpu().numpy(), src2.grad.cpu().numpy()) < 1e-4
    # (2) 25 % of the metric's detector, 4 poses, 512^3: sorted vs plain (forward and the sensitivities path)
    D, H, B = 512, 256, 4
    vol_np, volb, srcb, tgtb, lenb = _setup(D, H, B)
    sel = torch.randperm(H * H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(0))[: H * H // 4].sort().values
    tg, ln = tgtb[:, sel].contiguous(), lenb[:, sel].contiguous()
    res = {}
    for name, thr in (("sorted", 1), ("plain", 10 ** 9)):
        monkeypatch.setattr(renderers, "_SORT_MIN_RAYS", thr)
        with torch.no_grad():
            img_ = Siddon()(volb, srcb.reshape(B, 1, 3), tg, ln.reshape(B, 1, -1))
        s_, t_ = srcb.reshape(B, 1, 3).clone().requires_grad_(True), tg.clone().requires_grad_(True)
        o = Siddon()(volb, s_, t_, ln.reshape(B, 1, -1))
        (o * o).sum().backward()
        res[name] = (img_, o.detach(), t_.grad, s_.grad)
    for a, b in zip(res["sorted"], res["plain"]):
        assert relerr(a.cpu().numpy(), b.cpu().numpy()) < 1e-4


def test_subsampled_detector_inference_takes_the_brick_kernel(monkeypatch):
    """DRR(p_subsample=0.25) under no_grad on a batch: the brick-major kernel with a pixel -> ray map (b200drr_siddon_fwd_brick_subset)
    gives the same sub-sampled image as the ray-by-ray kernels and the fp64 oracle on the same rays."""
    from diffdrr_b200 import DRR, renderers, synthetic
    from diffdrr_b200.pose import convert
    from oracle import oracle
    D, H, B = 256, 128, 4
    monkeypatch.setattr(renderers, "_BRICK_MIN_BRICKS", 1)
    vol_np = synthetic.make_volume(D, "rand", seed=7)
    torch.manual_seed(0)
    drr = DRR(synthetic.make_subject(vol_np), **synthetic.detector_kwargs(H), p_subsample=0.25).to(DEV)
    rot, xyz = synthetic.make_poses(B, seed=9)
    calls = []
    orig = renderers._lib.load().b200drr_siddon_fwd_brick_subset
    with torch.no_grad():
        img = drr(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")       # scattered to (B,1,H,W)
        monkeypatch.setattr(renderers, "_BRICK_MIN_BATCH", 10 ** 9)
        img_ref = drr(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
        src, tgt = drr.detector(convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
    assert img.shape == (B, 1, H, H) and int((img != 0).sum()) > 0.2 * B * H * H * 0.5
    assert relerr(img.cpu().numpy(), img_ref.cpu().numpy()) < 3e-5
    ref = oracle.siddon_fwd(vol_np, *_np(src, tgt, raylen), dtype=np.float64)            # (B, 1, n_sub) in sub-sample order
    pick = torch.as_tensor(drr.detector.subsamples[-1])
    got = img.reshape(B, -1)[:, pick].cpu().numpy()
    assert relerr(got, ref.reshape(B, -1)) < IMG_TOL


@pytest.mark.parametrize("dims,H,W,B", [((56, 72, 44), 40, 36, 3), ((96, 96, 96), 64, 64, 2), ((256, 256, 256), 128, 128, 4),
                                        ((100, 96, 64), 48, 40, 9)])   # B >= 8: the 22-plane-brick / 8-tile-round instantiation
def test_brick_volume_gradient_vs_oracle_and_slab_kernel(dims, H, W, B):
    """b200drr_siddon_bwd_vol_brick (the brick kernel as a scatter: shared-memory accumulation, one TMA store per brick) against
    the fp64 oracle's g_volume and the slab-major kernel with global atomics; partial bricks on every axis in the first case."""
    import ctypes

    from diffdrr_b200 import DRR, _lib, synthetic
    from diffdrr_b200.pose import convert
    from diffdrr_b200.renderers import _ptr, _stream
    from oracle import oracle
    vol = torch.as_tensor(synthetic.make_volume(dims, "rand", seed=3)).to(DEV)
    drr = DRR(synthetic.make_subject(vol.cpu().numpy()), **synthetic.detector_kwargs(H, W)).to(DEV)
    rot, xyz = synthetic.make_poses(max(B, 2), seed=6)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot[:B].to(DEV), xyz[:B].to(DEV), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
        s, t = drr.affine_inverse(src).reshape(B, 3).contiguous(), drr.affine_inverse(tgt).contiguous()
    gout = torch.rand(B, H * W, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    lib = _lib.load()
    g_brick = torch.full_like(vol, float("nan"))
    ws = torch.empty(int(lib.b200drr_siddon_brick_workspace_bytes(B, H, W)), dtype=torch.uint8, device=DEV)
    _lib.check(lib.b200drr_siddon_bwd_vol_brick(_ptr(gout), *dims, _ptr(s), _ptr(t), _ptr(raylen), None, None, None, None, _ptr(g_brick),
                                                ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, H, W, 0.5, 1e-8, _stream()), "bwd_vol_brick")
    g_slab = torch.zeros_like(vol)
    _lib.check(lib.b200drr_siddon_bwd_grid(_ptr(vol), *dims, _ptr(s), _ptr(t), _ptr(raylen), _ptr(gout), None, None, None, _ptr(g_slab),
                                           B, H, W, 0.5, 1e-8, 0, 0, _stream()), "bwd_grid")
    torch.cuda.synchronize()
    assert torch.isfinite(g_brick).all()                      # every voxel written exactly once
    assert relerr(g_brick.cpu().numpy(), g_slab.cpu().numpy()) < 1e-4
    args = [x.cpu().numpy() for x in (s.reshape(B, 1, 3), t, raylen.reshape(B, 1, -1), gout.reshape(B, 1, -1))]
    ref64 = oracle.siddon_bwd(np.zeros(dims, np.float32), *args, dtype=np.float64)["g_volume"]
    ref32 = oracle.siddon_bwd(np.zeros(dims, np.float32), *args, dtype=np.float32)["g_volume"]
    tol = max(1e-4, 2 * relerr(ref32, ref64))                 # SURVEY 8c rule: fp32 chord lengths are differences of alphas
    assert relerr(g_brick.cpu().numpy(), ref64) < tol


def test_module_volume_gradient_takes_the_brick_scatter_and_matches_the_slab_path():
    """DRR with a density that requires grad (reconstruction): pose-in backward routes g_vol through the brick scatter
    (sparse ray sets only: 64^2 rays over a 96 x 128 x 128 volume)."""
    import diffdrr_b200.renderers as R
    from diffdrr_b200 import DRR, synthetic
    vol = synthetic.make_volume((96, 128, 128), "rand", seed=2)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(64)).to(DEV)
    rot, xyz = synthetic.make_poses(3, seed=1)
    w = torch.rand(3, 1, 64, 64, device=DEV, generator=torch.Generator(DEV).manual_seed(0))
    keep = R._BRICK_BWD, R._BRICK_MIN_BRICKS
    grads = []
    try:
        R._BRICK_MIN_BRICKS = 1
        for flag in (True, False):
            R._BRICK_BWD = flag
            dens = drr.density.detach().clone().requires_grad_(True)
            drr.density = dens
            assert R._brick_bwd_ok(dens, 3, 64, 64) == flag
            img = drr(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
            (img * w).sum().backward()
            grads.append(dens.grad.detach().clone())
    finally:
        R._BRICK_BWD, R._BRICK_MIN_BRICKS = keep
    assert relerr(grads[0].cpu().numpy(), grads[1].cpu().numpy()) < 1e-4


@pytest.mark.parametrize("D,H,B", [(512, 256, 1), (256, 200, 1), (256, 200, 2), (100, 40, 1)])
def test_small_batch_major_axis_pieces_vs_oracle(D, H, B):
    """Batches of one or two poses (the registration loop; single-DRR inference): b200drr_siddon_fwd_grid,
    b200drr_siddon_fwd_sens_grid + _bwd_sens and the pose-in module path cut every ray into pieces along its OWN major axis
    (siddon.cu small_batch_pieces: 12 pieces at 512^3, 10 at 256^3, 4 at 100^3).  Full images and end-point gradients
    against the fp64 oracle; detector sizes that are not a multiple of the 16 x 16 / 8 x 16 tiles."""
    from oracle import oracle
    L, lib = _lib()
    N = H * H
    vol_np, vol, src, tgt, raylen = _setup(D, H, B, seed=3, kind="smooth")
    ref_img = oracle.siddon_fwd(vol_np, *_np(src, tgt, raylen), dtype=np.float64).reshape(B, N)
    out = torch.full((B, N), float("nan"), device=DEV)
    L.check(lib.b200drr_siddon_fwd_grid(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out), B, H, H, 0.5, 1e-8, 0,
                                        _stream()), "fwd_grid")
    assert relerr(out.cpu().numpy(), ref_img) < IMG_TOL
    gout = torch.rand(B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    ref = oracle.siddon_bwd(vol_np, *_np(src, tgt, raylen, gout), dtype=np.float64, want_vol=False)
    out2 = torch.full((B, N), float("nan"), device=DEV)
    sens = torch.full((B, N, 8), float("nan"), device=DEV)
    L.check(lib.b200drr_siddon_fwd_sens_grid(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out2), _p(sens), B, H, H, 0.5,
                                             1e-8, 0, _stream()), "fwd_sens_grid")
    g_src, g_tgt, g_len = torch.empty(B, 3, device=DEV), torch.empty(B, N, 3, device=DEV), torch.empty(B, N, device=DEV)
    L.check(lib.b200drr_siddon_bwd_sens(_p(sens), _p(gout), _p(g_src), _p(g_tgt), _p(g_len), B, N, 0, _stream()), "bwd_sens")
    assert relerr(out2.cpu().numpy(), ref_img) < IMG_TOL
    assert relerr(g_tgt.cpu().numpy(), ref["g_target"]) < 2e-3
    assert relerr(g_src.cpu().numpy(), ref["g_source"].reshape(B, 3)) < 2e-3
    assert relerr(g_len.cpu().numpy(), ref["g_raylen"].reshape(B, N)) < IMG_TOL
    # the un-cut kernel (one thread per ray: variant 34 = a single 512-plane slab) agrees to fp32 summation order
    if D <= 512:
        out3, sens3 = torch.empty(B, N, device=DEV), torch.empty(B, N, 8, device=DEV)
        L.check(lib.b200drr_siddon_fwd_sens_grid(_p(vol), D, D, D, _p(src), _p(tgt), _p(raylen), _p(out3), _p(sens3), B, H, H,
                                                 0.5, 1e-8, 34, _stream()), "fwd_sens_grid uncut")
        assert relerr(out2.cpu().numpy(), out3.cpu().numpy()) < 1e-5
        # ... and so do the per-ray sensitivities: the cut keeps every crossing coefficient on its axis, also where a ray runs
        # through a voxel edge exactly on a cut (start_walk_frame<CUT>; 2e-3 apart before that rule, 1e-6 in CPU emulation now)
        assert relerr(sens.cpu().numpy(), sens3.cpu().numpy()) < 1e-4


def test_small_batch_module_path_matches_the_oracle_image_and_two_walk_gradients():
    """DRR(rot, xyz) for ONE pose (pose-in kernels with major-axis pieces, forward-only AND forward-with-sensitivities): image
    against the fp64 oracle on the module's own rays, pose gradients against the same module run with four copies of the pose
    (batch of 4: the slab-major kernels)."""
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import convert
    from oracle import oracle
    D, H = 128, 72
    vol_np = synthetic.make_volume(D, "smooth", seed=5)
    drr = DRR(synthetic.make_subject(vol_np), **synthetic.detector_kwargs(H), stop_gradients_through_grid_sample=True).to(DEV)
    rot, xyz = synthetic.make_poses(2, seed=6)
    rot, xyz = rot[:1].to(DEV), xyz[:1].to(DEV)
    w = torch.rand(1, 1, H, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    with torch.no_grad():
        img_inf = drr(rot, xyz, parameterization="euler_angles", convention="ZXY")
        src, tgt = drr.detector(convert(rot, xyz, parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
    ref = oracle.siddon_fwd(vol_np, *_np(src, tgt, raylen), dtype=np.float64).reshape(1, 1, H, H)
    assert relerr(img_inf.cpu().numpy(), ref) < IMG_TOL
    r1, t1 = rot.clone().requires_grad_(True), xyz.clone().requires_grad_(True)
    img = drr(r1, t1, parameterization="euler_angles", convention="ZXY")
    (img * w).sum().backward()
    assert relerr(img.detach().cpu().numpy(), ref) < IMG_TOL
    r4, t4 = rot.repeat(4, 1).requires_grad_(True), xyz.repeat(4, 1).requires_grad_(True)
    img4 = drr(r4, t4, parameterization="euler_angles", convention="ZXY")
    (img4 * w).sum().backward()
    assert relerr(img4[:1].detach().cpu().numpy(), img.detach().cpu().numpy()) < 1e-5
    assert relerr(r1.grad.cpu().numpy(), r4.grad[:1].cpu().numpy()) < 1e-3
    assert relerr(t1.grad.cpu().numpy(), t4.grad[:1].cpu().numpy()) < 1e-3
