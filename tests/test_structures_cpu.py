"""Piecewise-rigid renders (csrc/structures.cu, DRR.render_structures) on the CPU: the gated box walk and the footprint culling
compiled for the host against the C oracle on density * (label == k), the label boxes against numpy, and every refusal of
render_structures raised before any launch."""
import math

import numpy as np
import pytest
import torch

from conftest import relerr
from diffdrr_b200 import DRR, _lib, synthetic
from diffdrr_b200.drr import pose_in_matrices
from diffdrr_b200.pose import convert
from diffdrr_b200.structures import _rigid_inverse
from hostemu import emu_structures
from oracle import oracle

SHAPE = (24, 20, 28)
LABELS = (3, 7, 12)


def _label_volume():
    lab = np.zeros(SHAPE, np.uint8)
    lab[3:9, 4:12, 5:15] = 3
    lab[12:20, 8:16, 14:24] = 7
    lab[14:18, 2:6, 2:8] = 12
    lab[20:23, 15:19, 20:26] = 9     # a label no slot asks for: background
    return lab


def _drr(H=24, **kw):
    vol = synthetic.make_volume(SHAPE, "phantom", seed=2)
    lab = _label_volume()
    return DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab.astype(np.float32))), **synthetic.detector_kwargs(H), **kw), vol, lab


def _motion(rx, rz, t):
    """Rigid world motion (float64): rotation about x then z, then translation t (mm)."""
    cx, sx, cz, sz = math.cos(rx), math.sin(rx), math.cos(rz), math.sin(rz)
    Rx = torch.tensor([[1, 0, 0], [0, cx, -sx], [0, sx, cx]], dtype=torch.float64)
    Rz = torch.tensor([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]], dtype=torch.float64)
    X = torch.eye(4, dtype=torch.float64)
    X[:3, :3] = Rz @ Rx
    X[:3, 3] = torch.tensor(t, dtype=torch.float64)
    return X


def _slot_inputs(drr, P, X, background=True):
    """float64 (src, G, Wd) of the B * S (pose, slot) pairs: structure k seen by X_k^-1 P, then the background with P."""
    B, K = P.shape[0], X.shape[-3]
    Ps = _rigid_inverse(X.expand(B, K, 4, 4)) @ P[:, None]
    if background:
        Ps = torch.cat([Ps, P[:, None]], dim=1)
    S = Ps.shape[1]
    det = drr.detector
    src, G, Wd = pose_in_matrices(Ps.reshape(B * S, 4, 4), det._reorient.double(), det._calibration.double(),
                                  drr._affine_inverse.double())
    grid = det.target.view(det.height, det.width, 3)
    return src, G, Wd, grid[:, 0, 1].double(), grid[0, :, 0].double(), S


def _slot_tables(lab, labels, background):
    boxes = emu_structures.label_boxes(lab)
    slot = np.full(256, len(labels) if background else -1, np.int32)
    slot[list(labels)] = np.arange(len(labels))
    box = boxes[list(labels)]
    if background:
        box = np.concatenate([box, np.array([[0, 0, 0, *SHAPE]], np.int32)])
    return slot, box


def _rays(src, G, Wd, rows, cols):
    """Per-pixel float64 rays of every (pose, slot): src (BS, 1, 3), tgt (BS, H*W, 3), raylen (BS, 1, H*W)."""
    H, W = rows.numel(), cols.numel()
    p = torch.stack([cols.expand(H, W), rows[:, None].expand(H, W), torch.ones(H, W, dtype=torch.float64),
                     torch.ones(H, W, dtype=torch.float64)], dim=-1).reshape(H * W, 4)
    tgt = torch.einsum("bij,nj->bni", G, p)
    raylen = torch.einsum("bij,nj->bni", Wd, p).norm(dim=-1)
    return src[:, None, :].numpy(), tgt.numpy(), raylen[:, None, :].numpy()


def _camera(B, seed=0):
    """B seeded oblique poses (never the canonical AP view: its source sits on voxel planes of this volume, and fp32 and fp64
    walks may then attribute a tied crossing to different axes)."""
    rot, xyz = synthetic.make_poses(max(B, 2), seed=seed, rot_range=0.3, xyz_range=10.0)
    return convert(rot[:B].double(), xyz[:B].double(), parameterization="euler_angles", convention="ZXY").matrix


def _f32(*ts):
    return [t.float().numpy() for t in ts]


@pytest.mark.parametrize("B", [1, 2])
def test_slots_match_the_oracle_on_masked_densities(B):
    drr, vol, lab = _drr()
    P = _camera(B, seed=B)
    X = torch.stack([_motion(0.05, -0.08, [6.0, -4.0, 3.0]), _motion(-0.1, 0.04, [-8.0, 2.0, 10.0]),
                     _motion(0.0, 0.12, [3.0, 9.0, -5.0])])
    src, G, Wd, rows, cols, S = _slot_inputs(drr, P, X)
    slot, box = _slot_tables(lab, LABELS, True)
    got = emu_structures.structures(vol, lab, *_f32(src, G, Wd, rows, cols), slot, box, S)
    s_, t_, l_ = _rays(src, G, Wd, rows, cols)
    in_slot = [lab == k for k in LABELS] + [~np.isin(lab, LABELS)]
    N = rows.numel() * cols.numel()
    for bs in range(B * S):
        v = vol * in_slot[bs % S]
        ref = oracle.siddon_fwd(v, s_[bs:bs + 1], t_[bs:bs + 1], l_[bs:bs + 1], dtype=np.float64)
        assert np.abs(ref).max() > 0
        assert relerr(got["out"][bs], ref.reshape(N)) < 1e-5, bs
        # sensitivities: every ray as its own pose, unit upstream gradient
        g = oracle.siddon_bwd(v, np.repeat(s_[bs], N, 0)[:, None, :], t_[bs][:, None, :], l_[bs].reshape(N, 1, 1),
                              np.ones((N, 1, 1)), want_vol=False)
        assert relerr(got["sens"][bs, :, 0:3], g["g_target"].reshape(N, 3)) < 1e-4, bs
        assert relerr(got["sens"][bs, :, 4:7], g["g_source"].reshape(N, 3)) < 1e-4, bs
        assert relerr(got["sens"][bs, :, 3] * l_[bs].reshape(N), ref.reshape(N)) < 1e-5, bs


def test_identity_motions_match_mask_channels_and_sum_to_the_ungated_walk():
    drr, vol, lab = _drr()
    B = 2
    P = _camera(B, seed=5)
    X = torch.eye(4, dtype=torch.float64).expand(len(LABELS), 4, 4)
    src, G, Wd, rows, cols, S = _slot_inputs(drr, P, X)
    slot, box = _slot_tables(lab, LABELS, True)
    got = emu_structures.structures(vol, lab, *_f32(src, G, Wd, rows, cols), slot, box, S)
    img = got["out"].reshape(B, S, -1)
    s_, t_, l_ = _rays(src.view(B, S, 3)[:, -1], G.view(B, S, 3, 4)[:, -1], Wd.view(B, S, 3, 4)[:, -1], rows, cols)
    chans = oracle.siddon_fwd_mask(vol, lab.astype(np.float64), s_, t_, l_, 13, dtype=np.float64)
    for k, label in enumerate(LABELS):
        assert relerr(img[:, k], chans[:, label]) < 1e-5, label
    whole = oracle.siddon_fwd(vol, s_, t_, l_, dtype=np.float64)
    assert relerr(img.sum(1), whole[:, 0]) < 1e-5
    # the image-only walk (no sensitivities) renders the same channels
    fwd = emu_structures.structures(vol, lab, *_f32(src, G, Wd, rows, cols), slot, box, S, sens=False)
    assert relerr(fwd["out"], got["out"]) < 1e-5   # a different walk set-up: fp32 round-off


def test_culling_changes_no_bit():
    """Every pixel a box's walk can reach lies in its footprint rectangle, so culled and unculled renders are bitwise equal --
    including a structure moved onto the source (its box straddles the source plane: the whole detector) and one moved off the
    detector (an empty rectangle)."""
    drr, vol, lab = _drr(H=32)
    P = _camera(2, seed=3)
    X = torch.stack([_motion(0.2, 0.1, [5.0, -3.0, 2.0]),
                     _motion(0.0, 0.0, [0.0, 850.0, 0.0]),       # label 7 around the source
                     _motion(0.0, 0.0, [420.0, 0.0, 0.0])])      # label 12 far to the side
    src, G, Wd, rows, cols, S = _slot_inputs(drr, P, X)
    slot, box = _slot_tables(lab, LABELS, True)
    args = (vol, lab, *_f32(src, G, Wd, rows, cols), slot, box, S)
    culled, full = emu_structures.structures(*args), emu_structures.structures(*args, cull=False)
    assert np.array_equal(culled["out"], full["out"]) and np.array_equal(culled["sens"], full["sens"])
    rect = culled["rect"].reshape(2, S, 4)
    H, W = rows.numel(), cols.numel()
    assert (rect[:, 1] == [0, W - 1, 0, H - 1]).all()                               # straddles the source plane
    assert ((rect[:, 2, 0] > rect[:, 2, 1]) | (rect[:, 2, 2] > rect[:, 2, 3])).all()  # off the detector
    assert (full["out"].reshape(2, S, -1)[:, 2] == 0).all()
    small = (rect[:, 0, 1] - rect[:, 0, 0] + 1) * (rect[:, 0, 3] - rect[:, 0, 2] + 1)
    assert (small < H * W).all()                                                    # the culling does cull
    nz = full["out"].reshape(2 * S, H, W) != 0
    for bs in range(2 * S):
        ys, xs = np.nonzero(nz[bs])
        r = culled["rect"][bs]
        assert ((xs >= r[0]) & (xs <= r[1]) & (ys >= r[2]) & (ys <= r[3])).all()


def test_label_boxes_match_numpy():
    rng = np.random.default_rng(0)
    lab = _label_volume()
    lab[rng.random(SHAPE) < 0.002] = 200     # scattered voxels of one more label
    boxes = emu_structures.label_boxes(lab)
    for l in range(256):
        idx = np.argwhere(lab == l)
        if idx.size == 0:
            assert (boxes[l, :3] > boxes[l, 3:]).any(), l
        else:
            assert boxes[l].tolist() == [*idx.min(0), *(idx.max(0) + 1)], l


def _call(drr, **kw):
    args = dict(motions=torch.eye(4).expand(len(LABELS), 4, 4), labels=LABELS)
    args.update(kw)
    rot, xyz = synthetic.make_poses(2)
    return drr.render_structures(rot, xyz, parameterization="euler_angles", convention="ZXY", **args)


def test_refusals_raise_before_any_launch():
    drr, vol, lab = _drr(H=8)
    with pytest.raises(_lib.B200DRRError, match="CUDA"):                 # CPU density: the last check, everything else passed
        _call(drr)
    with pytest.raises(NotImplementedError, match="Siddon"):
        _call(DRR(drr.subject, **synthetic.detector_kwargs(8), renderer="trilinear"))
    for kw in (dict(mode="bilinear"), dict(reducefn="max")):
        with pytest.raises(NotImplementedError, match="default options"):
            _call(DRR(drr.subject, **synthetic.detector_kwargs(8), **kw))
    with pytest.raises(NotImplementedError, match="renderer options"):
        _call(drr, align_corners=True)
    with pytest.raises(NotImplementedError, match="p_subsample"):
        _call(DRR(drr.subject, **synthetic.detector_kwargs(8), p_subsample=0.5))
    with pytest.raises(NotImplementedError, match="patch_size"):
        _call(DRR(drr.subject, **synthetic.detector_kwargs(8), patch_size=4))
    with pytest.raises(ValueError, match="no mask"):
        _call(DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(8)))
    with pytest.raises(ValueError, match="integers"):
        _call(drr, labels=(3, 7.5, 12))
    with pytest.raises(ValueError, match="0..255"):
        _call(drr, labels=(3, 7, 300))
    with pytest.raises(ValueError, match="do not occur"):
        _call(drr, labels=(3, 7, 5))
    with pytest.raises(ValueError, match="distinct"):
        _call(drr, labels=(3, 7, 3))
    for m in (torch.eye(4), torch.eye(4).expand(2, 4, 4), torch.eye(4).expand(3, 3, 4, 4), torch.eye(4, dtype=torch.float64).expand(3, 4, 4)):
        with pytest.raises(ValueError, match="motions"):
            _call(drr, motions=m)
    drr.density.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="require grad"):
        _call(drr)


def test_pose_batch_size_and_motion_shapes_from_every_pose_form():
    """The number of camera poses comes from the pose matrix's leading dimension ('matrix', RigidTransform) or the rotation
    parameters' -- never from the trailing (4, 4) -- and (B, K, 4, 4) motions may arrive wrapped in a RigidTransform."""
    from diffdrr_b200.pose import RigidTransform
    from diffdrr_b200.structures import _batch_size, _motion_matrices
    eye = torch.eye(4)
    assert _batch_size((eye,), "matrix") == 1
    assert _batch_size((eye[None],), "matrix") == 1
    assert _batch_size((eye.expand(3, 4, 4),), "matrix") == 3
    assert _batch_size((RigidTransform(eye.expand(3, 4, 4)),), None) == 3
    assert _batch_size((torch.zeros(2, 3), torch.zeros(2, 3)), "euler_angles") == 2
    assert _batch_size((torch.zeros(5, 4), torch.zeros(5, 3)), "quaternion") == 5
    X = eye.expand(2, 3, 4, 4)
    assert _motion_matrices(RigidTransform(X), 3, 2).shape == (2, 3, 4, 4)
    assert _motion_matrices(RigidTransform(X[0]), 3, 2).shape == (3, 4, 4)
    with pytest.raises(ValueError, match="motions"):
        _motion_matrices(RigidTransform(X), 3, 1)
    drr, _, _ = _drr(H=8)
    with pytest.raises(ValueError, match="4, 4"):
        drr.render_structures(torch.zeros(2, 3, 4), motions=eye.expand(3, 4, 4), labels=LABELS, parameterization="matrix")
