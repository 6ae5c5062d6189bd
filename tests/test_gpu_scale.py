"""GPU parity beyond the goldens: seeded mid-size cases against the oracle and size-independent properties at the
BASELINE.json sizes (512^3 volume, 256^2 detector) where the oracle would take too long."""
import numpy as np
import pytest
import torch

from conftest import relerr
from gpu_common import DEV, t

pytestmark = pytest.mark.gpu


def _rays(drr, rot, xyz):
    from diffdrr_b200.pose import convert
    with torch.no_grad():
        pose = convert(rot.to(DEV), xyz.to(DEV), parameterization="euler_angles", convention="ZXY")
        src, tgt = drr.detector(pose, None)
        raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
        return drr.affine_inverse(src).contiguous(), drr.affine_inverse(tgt).contiguous(), raylen.contiguous()


@pytest.mark.parametrize("D,H,B", [(96, 80, 3), (256, 256, 2)])
def test_mid_size_vs_oracle(D, H, B):
    """BASELINE config[1] shape (256^3 -> 256^2) on a reduced batch, checked ray by ray against the fp64 oracle."""
    from diffdrr_b200 import DRR, synthetic
    from oracle import oracle
    vol = synthetic.make_volume(D, "rand", seed=5)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H)).to(DEV)
    rot, xyz = synthetic.make_poses(B, seed=3)
    src, tgt, raylen = _rays(drr, rot, xyz)
    args = (vol, src.cpu().numpy(), tgt.cpu().numpy(), raylen.cpu().numpy())
    from diffdrr_b200 import Siddon, Trilinear
    out = Siddon()(drr.density, src, tgt, raylen).cpu().numpy()
    assert relerr(out, oracle.siddon_fwd(*args, dtype=np.float64)) < 1e-4
    out = Trilinear()(drr.density, src, tgt, raylen, n_points=300).cpu().numpy()
    amin, amax = oracle.alpha_minmax(vol.shape, args[1], args[2], 0.5, 1e-8, np.float32)
    assert relerr(out, oracle.trilinear_fwd(*args, n_points=300, alphamin=amin, alphamax=amax, dtype=np.float64)) < 1e-4
    # gradients of a random linear functional vs the fp64 oracle on a subset of rays (keeps the oracle fast), on the
    # SMOOTH volume: on white noise every crossing contributes (v_before - v_after)*alpha with random sign and the fp32
    # sums are ill-conditioned (the reference's own fp32 run is 2e-4..1e-2 off there, SURVEY 8c), and a hard edge
    # makes the gradient of a grazing ray an O(1) coin toss between fp32 and fp64
    phantom = synthetic.make_volume(D, "smooth", seed=4)
    pv = t(phantom)
    sub = slice(0, 4096)
    w = torch.rand(B, 1, 4096, device=DEV, generator=torch.Generator(device=DEV).manual_seed(0))
    s, tg, l = src.clone().requires_grad_(True), tgt[:, sub].clone().requires_grad_(True), raylen[:, :, sub].clone().requires_grad_(True)
    v = pv.clone().requires_grad_(True)
    (Siddon()(v, s, tg, l) * w).sum().backward()
    ref = oracle.siddon_bwd(phantom, args[1], args[2][:, sub], args[3][:, :, sub], w.cpu().numpy(), dtype=np.float64)
    assert relerr(tg.grad.cpu().numpy(), ref["g_target"]) < 2e-3
    assert relerr(s.grad.cpu().numpy(), ref["g_source"]) < 2e-3
    assert relerr(l.grad.cpu().numpy(), ref["g_raylen"]) < 1e-4
    assert relerr(v.grad.cpu().numpy(), ref["g_volume"]) < 1e-4


@pytest.fixture(scope="module")
def big():
    from diffdrr_b200 import DRR, synthetic
    g = torch.Generator(device=DEV).manual_seed(0)
    vol = torch.rand(512, 512, 512, device=DEV, generator=g)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))  # placeholder; the real volume is passed to render()
    subj.volume.affine = synthetic.make_affine(512)
    drr = DRR(subj, **synthetic.detector_kwargs(256)).to(DEV)
    rot, xyz = synthetic.make_poses(4, seed=0)
    return drr, vol, _rays(drr, rot, xyz)


def test_full_size_properties(big):
    """512^3 -> 256^2 (the metric's configuration): properties that pin the result without an oracle run."""
    from diffdrr_b200 import Siddon, Trilinear
    from diffdrr_b200.renderers import siddon_visits
    drr, vol, (src, tgt, raylen) = big
    sid = Siddon()
    out = sid(vol, src, tgt, raylen)
    assert torch.isfinite(out).all() and out.shape == (4, 1, 256 * 256)
    # (1) a constant volume integrates to (chord length through the box) = L * (alpha_out - alpha_in)
    ones = torch.ones_like(vol)
    d = tgt - src + 1e-8
    a0, a1 = (-0.5 - src) / d, (511.5 - src) / d
    chord = (torch.maximum(a0, a1).amin(-1) - torch.minimum(a0, a1).amax(-1)).clamp_min(0) * raylen[:, 0]
    got = sid(ones, src, tgt, raylen)[:, 0]
    assert relerr(got.cpu().numpy(), chord.cpu().numpy()) < 1e-5
    # (2) linearity in the volume
    vol2 = torch.rand(vol.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    lin = sid(0.25 * vol + 2.0 * vol2, src, tgt, raylen)
    assert relerr(lin.cpu().numpy(), (0.25 * out + 2.0 * sid(vol2, src, tgt, raylen)).cpu().numpy()) < 1e-5
    del vol2, ones
    # (3) batch / patch invariance of Siddon (every ray is independent)
    one = sid(vol, src[1:2], tgt[1:2, 1000:3000].contiguous(), raylen[1:2, :, 1000:3000].contiguous())
    # (not bitwise: the 4-pose call takes the locality-sorted SLAB-major kernels -- per-slab partial sums combined by
    # red.global.add in run-dependent order -- while a 2000-ray call of one pose may take another decomposition; kernels agree
    # to fp32 round-off of the partial sums, DESIGN.md 4.1).  Each fp32 decomposition sums ~670 visits per ray and lands
    # ~1.5e-5 from the fp64 oracle at this size, so both are pinned to the oracle and to each other at 2e-5.
    from oracle import oracle
    ref = oracle.siddon_fwd(vol.cpu().numpy(), src[1:2].cpu().numpy(), tgt[1:2, 1000:3000].cpu().numpy(),
                            raylen[1:2, :, 1000:3000].cpu().numpy(), dtype=np.float64)[0, 0]
    assert relerr(one[0, 0].cpu().numpy(), ref) < 2e-5
    assert relerr(out[1, 0, 1000:3000].cpu().numpy(), ref) < 2e-5
    assert relerr(one[0, 0].cpu().numpy(), out[1, 0, 1000:3000].cpu().numpy()) < 2e-5
    # (4) the general (plane-by-plane, reference-literal) kernel: max over segments is in [0, sum] for a density >= 0
    mx = Siddon(reducefn="max")(vol, src[:1], tgt[:1, :4096].contiguous(), raylen[:1, :, :4096].contiguous())
    assert (mx >= 0).all() and (mx <= out[:1, :, :4096] + 1e-6).all()
    # (5) visit counts: every hit ray crosses between 1 and D0+D1+D2 voxels; mean matches SURVEY 8d (~666)
    visits = siddon_visits((512, 512, 512), src, tgt)
    assert int(visits.max()) <= 3 * 512 and ((visits > 0) == (chord > 0).reshape(visits.shape)).float().mean() > 0.999
    assert 550 < float(visits.float().mean()) < 750
    # (6) trilinear with a fine step converges to Siddon's exact integral on a smooth volume
    x = torch.linspace(-1, 1, 512, device=DEV)
    smooth = torch.exp(-(x[:, None, None] ** 2 + x[None, :, None] ** 2 + x[None, None, :] ** 2) / 0.3)
    a = sid(smooth, src[:1], tgt[:1], raylen[:1])
    b = Trilinear()(smooth, src[:1], tgt[:1], raylen[:1], n_points=2000)
    assert relerr(b.cpu().numpy(), a.cpu().numpy()) < 5e-3


def test_full_size_grid_kernels_match_plain_kernels(big):
    """The tiled kernels (used when the rays are a full detector grid; 4 poses: every ray cut into 12 major-axis pieces)
    against the one-thread-per-ray kernels on the metric's configuration; gradients too.  Partial sums are combined with red.global.add, so the
    comparison is to fp32 round-off, not bitwise."""
    from diffdrr_b200 import Siddon
    drr, vol, (src, tgt, raylen) = big
    plain, tiled = Siddon(), Siddon()
    tiled.detector_shape = (256, 256)
    w = torch.rand(4, 1, 256 * 256, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    x = torch.linspace(-1, 1, 512, device=DEV)
    smooth = torch.exp(-(x[:, None, None] ** 2 + x[None, :, None] ** 2 + x[None, None, :] ** 2) / 0.3)
    # images on the white-noise volume; end-point gradients on a smooth one (on white noise they are fp32-ill-conditioned)
    for volume, tols in ((vol, (3e-5, None, None, 3e-5)), (smooth, (3e-5, 1e-3, 1e-3, 3e-5))):
        outs = []
        for mod in (plain, tiled):
            s, t_, l = src.clone().requires_grad_(True), tgt.clone().requires_grad_(True), raylen.clone().requires_grad_(True)
            out = mod(volume, s, t_, l)
            (out * w).sum().backward()
            outs.append((out.detach(), s.grad, t_.grad, l.grad))
        for a, b, tol in zip(outs[0], outs[1], tols):
            if tol is not None:
                assert relerr(b.cpu().numpy(), a.cpu().numpy()) < tol
    del smooth
    # volume gradient through the tiled kernel: adjoint identity
    v = vol.clone().requires_grad_(True)
    (tiled(v, src[:2], tgt[:2], raylen[:2]) * w[:2]).sum().backward()
    vol2 = torch.rand(vol.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(6))
    lhs = (tiled(vol2, src[:2], tgt[:2], raylen[:2]) * w[:2]).sum().double()
    rhs = (vol2.double() * v.grad.double()).sum()
    assert abs(float(lhs - rhs)) / abs(float(lhs)) < 1e-4


def test_full_size_gradients(big):
    """fwd+bwd at 512^3 -> 256^2: the adjoint identity <J v, w> = <v, J^T w> ties backward to forward."""
    from diffdrr_b200 import Siddon
    drr, vol, (src, tgt, raylen) = big
    sid = Siddon()
    v = vol.clone().requires_grad_(True)
    w = torch.rand(1, 1, tgt.shape[1], device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    out = sid(v, src[:1], tgt[:1], raylen[:1])
    (out * w).sum().backward()
    # the map volume -> image is linear: <A vol2, w> == <vol2, A^T w>
    vol2 = torch.rand(vol.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    lhs = (sid(vol2, src[:1], tgt[:1], raylen[:1]) * w).sum().double()
    rhs = (vol2.double() * v.grad.double()).sum()
    assert abs(float(lhs - rhs)) / abs(float(lhs)) < 1e-4
    # d/d raylen is the un-scaled line integral
    l = raylen[:1].clone().requires_grad_(True)
    sid(vol, src[:1], tgt[:1], l).sum().backward()
    assert relerr((l.grad * raylen[:1]).cpu().numpy(), out.detach().cpu().numpy()) < 1e-5
    # pose gradient by central finite differences on a smooth volume (source shifted along each axis)
    x = torch.linspace(-1, 1, 512, device=DEV)
    smooth = torch.exp(-(x[:, None, None] ** 2 + x[None, :, None] ** 2 + x[None, None, :] ** 2) / 0.3)
    s = src[:1].clone().requires_grad_(True)
    sub = slice(20000, 24096)
    tg, ln, ww = tgt[:1, sub].contiguous(), raylen[:1, :, sub].contiguous(), w[:, :, sub].contiguous()
    (sid(smooth, s, tg, ln) * ww).sum().backward()
    for a in range(3):
        h = 0.25
        e = torch.zeros_like(src[:1]); e[..., a] = h
        fd = ((sid(smooth, src[:1] + e, tg, ln) * ww).sum() - (sid(smooth, src[:1] - e, tg, ln) * ww).sum()) / (2 * h)
        assert abs(float(fd - s.grad[0, 0, a])) < 2e-2 * max(1.0, abs(float(fd)))


def test_pose_in_path_matches_ray_tensor_path():
    """DRR.forward's fused pose-in kernels (rays generated in-kernel from 3x4 matrices) against the generic path that
    materialises source/target tensors (detector -> render), images and pose gradients, incl. a non-zero principal point."""
    from diffdrr_b200 import DRR, synthetic
    vol = synthetic.make_volume(128, "smooth", seed=9)
    drr = DRR(synthetic.make_subject(vol), sdd=1020.0, height=96, width=80, delx=2.5, dely=3.0, x0=7.0, y0=-4.0).to(DEV)
    rot0, xyz0 = synthetic.make_poses(3, seed=5)
    w = torch.rand(3, 1, 96, 80, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    res = []
    for fused in (True, False):
        rot, xyz = rot0.to(DEV).requires_grad_(True), xyz0.to(DEV).requires_grad_(True)
        if fused:
            assert drr._pose_in_ok(False, {})
            img = drr(rot, xyz, parameterization="euler_angles", convention="ZXY")
        else:
            from diffdrr_b200.pose import convert
            src, tgt = drr.detector(convert(rot, xyz, parameterization="euler_angles", convention="ZXY"), None)
            img = drr.reshape_transform(drr.render(drr.density, src, tgt), batch_size=3)
        (img * w).sum().backward()
        res.append((img.detach(), rot.grad, xyz.grad))
    assert relerr(res[0][0].cpu().numpy(), res[1][0].cpu().numpy()) < 2e-5
    assert relerr(res[0][1].cpu().numpy(), res[1][1].cpu().numpy()) < 1e-3
    assert relerr(res[0][2].cpu().numpy(), res[1][2].cpu().numpy()) < 1e-3


def test_trilinear_packed_corner_path():
    """Packed-corner kernels (one 32-byte read per sample) == scalar-gather kernels; a volume that requires grad takes
    the gather path and gets its gradient; an in-place volume update invalidates the packed copy."""
    from diffdrr_b200 import DRR, Trilinear, synthetic
    vol = synthetic.make_volume((72, 96, 80), "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), sdd=1020.0, height=64, width=72, delx=3.0, renderer="trilinear").to(DEV)
    rot0, xyz0 = synthetic.make_poses(3, seed=8)
    w = torch.rand(3, 1, 64, 72, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    import diffdrr_b200.drr as drr_mod
    res = []
    keep = drr_mod._TRILINEAR_POSE_IN
    drr_mod._TRILINEAR_POSE_IN = False   # this test compares KERNELS on identical ray tensors (pose-in: test_gpu_trilinear_pose.py)
    try:
        for packed in (True, False):
            drr.renderer.pack_corners = packed
            rot, xyz = rot0.to(DEV).requires_grad_(True), xyz0.to(DEV).requires_grad_(True)
            img = drr(rot, xyz, parameterization="euler_angles", convention="ZXY", n_points=180)
            (img * w).sum().backward()
            res.append((img.detach(), rot.grad, xyz.grad))
            assert (drr.renderer._packed is not None) == packed or not packed
    finally:
        drr_mod._TRILINEAR_POSE_IN = keep
    assert torch.equal(res[0][0], res[1][0])
    assert relerr(res[0][1].cpu().numpy(), res[1][1].cpu().numpy()) < 1e-5
    assert relerr(res[0][2].cpu().numpy(), res[1][2].cpu().numpy()) < 1e-5
    drr.renderer.pack_corners = True
    # batch >= 8 switches the forward to slab-major scheduling (partial sums combined with red.global.add)
    rot8, xyz8 = synthetic.make_poses(9, seed=12)
    with torch.no_grad():
        slabbed = drr(rot8.to(DEV), xyz8.to(DEV), parameterization="euler_angles", convention="ZXY", n_points=180)
        drr.renderer.pack_corners = False
        plain = drr(rot8.to(DEV), xyz8.to(DEV), parameterization="euler_angles", convention="ZXY", n_points=180)
        drr.renderer.pack_corners = True
    assert relerr(slabbed.cpu().numpy(), plain.cpu().numpy()) < 5e-6
    with torch.no_grad():
        before = drr(rot0.to(DEV), xyz0.to(DEV), parameterization="euler_angles", convention="ZXY", n_points=180)
        drr.density.mul_(2.0)  # in-place update bumps the tensor version -> the packed copy is rebuilt
        after = drr(rot0.to(DEV), xyz0.to(DEV), parameterization="euler_angles", convention="ZXY", n_points=180)
    assert relerr(after.cpu().numpy(), 2.0 * before.cpu().numpy()) < 1e-6
    # reconstruction mode: the volume is a parameter -> gather path, volume gradient present
    from diffdrr_b200.pose import convert
    dens = drr.density.clone().requires_grad_(True)
    src, tgt = drr.detector(convert(rot0.to(DEV), xyz0.to(DEV), parameterization="euler_angles", convention="ZXY"), None)
    out = drr.render(dens, src, tgt, n_points=60)
    out.sum().backward()
    assert dens.grad is not None and float(dens.grad.abs().sum()) > 0


def test_fused_sensitivities_match_two_walk_backward():
    """Training-step fast path (one walk: image + per-ray sensitivities, elementwise backward) against the two-walk
    path (forward kernel + backward walk) it replaces: images, pose gradients, ray-tensor gradients, stop-gradient flag;
    and a volume that requires grad must still get its gradient (two-walk path)."""
    from diffdrr_b200 import DRR, Siddon, renderers, synthetic
    from diffdrr_b200.pose import convert
    vol = synthetic.make_volume((112, 128, 96), "smooth", seed=13)
    rot0, xyz0 = synthetic.make_poses(3, seed=8)
    w = torch.rand(3, 1, 88, 72, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    for stop in (False, True):
        drr = DRR(synthetic.make_subject(vol), sdd=1020.0, height=88, width=72, delx=2.5, dely=3.0, x0=5.0,
                  stop_gradients_through_grid_sample=stop).to(DEV)
        res = []
        for fused in (True, False):
            renderers._FUSED_SENSITIVITIES = fused
            try:
                rot, xyz = rot0.to(DEV).requires_grad_(True), xyz0.to(DEV).requires_grad_(True)
                img = drr(rot, xyz, parameterization="euler_angles", convention="ZXY")     # pose-in kernels
                (img * w).sum().backward()
                src, tgt = drr.detector(convert(rot0.to(DEV), xyz0.to(DEV), parameterization="euler_angles",
                                                convention="ZXY"), None)
                s, t_ = src.clone().requires_grad_(True), tgt.clone().requires_grad_(True)
                img2 = drr.render(drr.density, s, t_)                                           # detector-grid kernels
                (img2.view(3, 1, 88, 72) * w).sum().backward()
                res.append((img.detach(), rot.grad, xyz.grad, img2.detach(), s.grad, t_.grad))
            finally:
                renderers._FUSED_SENSITIVITIES = True
        # partial sums are combined with red.global.add in a run-dependent order: fp32 round-off level, with head-room.  (The
        # fused walk cuts every ray into pieces along its major axis here -- 3 poses -- and the backward walk into slabs along
        # axis 0; both keep every crossing coefficient on its axis, tests/test_hostemu.py::test_major_axis_pieces_keep_...:
        # CPU emulation of this very case 6e-8 on the ray-tensor gradients, 1e-6 on the images.)
        for a, b, tol in zip(res[0], res[1], (1e-5, 5e-5, 5e-5, 1e-5, 5e-5, 5e-5)):
            assert relerr(a.cpu().numpy(), b.cpu().numpy()) < tol
    # volume gradient requested -> backward walk; pose gradients identical to the fused ones
    sid = Siddon()
    sid.detector_shape = (88, 72)
    aff = drr.affine_inverse
    raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
    sv, tv = aff(src).detach(), aff(tgt).detach()
    outs = []
    for need_vol in (False, True):
        v = drr.density.clone().requires_grad_(need_vol)
        t_ = tv.clone().requires_grad_(True)
        (sid(v, sv, t_, raylen).view(3, 1, 88, 72) * w).sum().backward()
        outs.append(t_.grad)
        assert (v.grad is not None) == need_vol
    assert relerr(outs[0].cpu().numpy(), outs[1].cpu().numpy()) < 5e-5


@pytest.mark.parametrize("B", [3, 8])
def test_trilinear_fused_sensitivities_match_two_march_backward(B):
    """Trilinear twin of the test above: one march from the packed-corner copy (image + per-ray sensitivities, incl. the
    batch-global alphamin/alphamax partials) + elementwise backward == forward march + backward march (B = 8: the
    two-march forward is slab-major there)."""
    from diffdrr_b200 import DRR, renderers, synthetic
    vol = synthetic.make_volume((80, 96, 72), "smooth", seed=17)
    drr = DRR(synthetic.make_subject(vol), sdd=1020.0, height=64, width=56, delx=3.5, renderer="trilinear").to(DEV)
    rot0, xyz0 = synthetic.make_poses(B, seed=6)
    w = torch.rand(B, 1, 64, 56, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    res = []
    for fused, slab in ((True, 0), (False, 0), (True, 16)):   # slab 16: the slab-major form of the fused march (opt-in)
        renderers._FUSED_SENSITIVITIES, renderers._PACKED_SLAB_SENS = fused, slab
        try:
            rot, xyz = rot0.to(DEV).requires_grad_(True), xyz0.to(DEV).requires_grad_(True)
            img = drr(rot, xyz, parameterization="euler_angles", convention="ZXY", n_points=150)
            (img * w).sum().backward()
            res.append((img.detach(), rot.grad, xyz.grad))
        finally:
            renderers._FUSED_SENSITIVITIES, renderers._PACKED_SLAB_SENS = True, 0
    for other, tols in ((res[0], (2e-6, 1e-4, 1e-4)), (res[2], (5e-6, 3e-4, 3e-4))):
        for a, b, tol in zip(other, res[1], tols):
            assert relerr(a.cpu().numpy(), b.cpu().numpy()) < tol
