"""Named piecewise-rigid scenes, their fp64 references and the per-ray comparison shared by the structures tests
(test_structures_cases_cpu.py on the host emulation, test_gpu_structures_oracle.py on the kernels).

A scene is a density and a uint8 label volume, the slot tables of b200drr_siddon_fwd_sens_structures (slot_of_label (256,),
box (S, 6)) and, per (pose b, slot s) at index b*S + s, the fp32 pose-in inputs src, G, Wd and the shared rows / cols.  A motion
of structure s is just another pose of slot s, so every (pose, slot) gets its own geometry here.  G and Wd are dyadic
(siddon_cases.pose_matrices), so G p is exact in fp32: the kernels walk exactly the fp32 rays `tgt` / `raylen` of the scene,
and the un-cut walk on those rays, over the slot's masked density, is the reference for their per-ray sensitivities at ties.

Bounds, per (pose, slot), relative to the reference's largest value on that slot:
  image          every ray but near-face ones, <= IMAGE_TOL of the fp64 oracle on density x (label in slot);
  sensitivities  well-conditioned rays against the fp64 oracle at siddon_cases.siddon_tol (both end points); near-tie rays and
                 every lattice ray against the un-cut walk at TIE_TOL; every ray satisfies sum jt_a d_a = -I and
                 sum (js_a + jt_a) d_a = 0."""
import functools

import numpy as np

import siddon_cases as sc
import trilinear_cases as tc

IMAGE_TOL = 1e-4
TIE_TOL = 1e-5
SENS_FLOOR = 5e-4
IDENTITY_TOL = 1e-5
# image-only walk against the sensitivities walk, per ray: the two set up their alphas differently (start_walk_box against the
# volume frame of start_walk_frame), so segment lengths differ by fp32 round-off -- up to 6.5e-6 of the slot's maximum on these
# scenes (the thin slab), as much as the oracle's own fp32 against fp64; bitwise equal on the lattices
LEAN_TOL = 1e-5


def label_boxes(lab):
    """numpy statement of b200drr_label_boxes: (256, 6) int32 [lo, hi) per label; an absent label keeps lo = D > hi = 0."""
    boxes = np.zeros((256, 6), np.int32)
    boxes[:, :3] = lab.shape
    for label in np.unique(lab):
        idx = np.argwhere(lab == label)
        boxes[label] = [*idx.min(0), *(idx.max(0) + 1)]
    return boxes


def slot_tables(lab, slots, background):
    """slots: one tuple of labels per structure slot.  -> slot_of_label (256,) int32 (-1 = no slot; the background slot takes
    every other label), box (S, 6) int32: the union of the slot's label boxes, the whole volume for the background."""
    boxes = label_boxes(lab)
    slot = np.full(256, len(slots) if background else -1, np.int32)
    box = []
    for s, labels in enumerate(slots):
        slot[list(labels)] = s
        b = boxes[list(labels)]
        box.append([*b[:, :3].min(0), *b[:, 3:].max(0)])
    if background:
        box.append([0, 0, 0, *lab.shape])
    return slot, np.asarray(box, np.int32)


def _view(D, rng, kind="rotated", src=None, shift_uv=(0.0, 0.0)):
    """(src, detector centre, u, v) of one cone view of a D-sided volume in a random direction: 'rotated' puts the source 1.6
    diagonals out with the volume filling most of the detector, 'inside' takes the given source (inside the volume) and a
    detector 1.5 diagonals beyond it.  shift_uv moves the detector centre by that many half-widths along u / v, so that what
    projects to detector coordinate c lands at c - shift."""
    diag, centre = float(np.linalg.norm(D)), (D - 1) / 2
    d, u, v = tc._frame(rng)
    if kind == "inside":
        s = np.asarray(src, np.float64)
        c, u, v = s + 1.5 * diag * d, 0.9 * diag * u, 0.7 * diag * v
    else:
        s = centre - 1.6 * diag * d
        c, u, v = centre + 0.6 * diag * d, 0.45 * diag * u, 0.4 * diag * v
    c = c + shift_uv[0] * u + shift_uv[1] * v
    return sc._q(s, 4), c, u, v


def _pose_in(views, H, W, flip=False, rows=None, cols=None):
    """Pose-in inputs of the (pose, slot) views -> src (BS, 3), G, Wd (BS, 3, 4), rows (H,), cols (W,) fp32, all exact."""
    s, c, u, v = (np.asarray(x) for x in zip(*views))
    src = s.astype(np.float32)
    assert (src == s).all()
    G, Wd, r, k = sc.pose_matrices(src, c, u, v, H, W)[:4]
    r = r if rows is None else np.asarray(rows, np.float32)
    k = k if cols is None else np.asarray(cols, np.float32)
    if flip:   # negative delx / dely: pixel coordinates decrease along rows and columns
        r, k = r[::-1].copy(), k[::-1].copy()
    return src, G, Wd, r, k


def _density(dims, rng):
    return (rng.random(dims) + 0.5).astype(np.float32)


def _scene(dims, H, W, B, slots, background, lab, views=None, kind=None, eps=1e-8, pose=None, seed=0, **view_kw):
    rng = np.random.default_rng(seed)
    vol = _density(dims, rng)
    D = np.asarray(dims, np.float64)
    S = len(slots) + int(background)
    if pose is None:
        vs = []
        for b in range(B):
            for s in range(S):
                kw = (views or {}).get((b, s), {})
                vs.append(_view(D, rng, **kw))
        pose = _pose_in(vs, H, W, **view_kw)
    slot, box = slot_tables(lab, slots, background)
    return dict(vol=vol, lab=lab, slots=slots, background=background, slot=slot, box=box, S=S, B=B, H=len(pose[3]),
                W=len(pose[4]), src=pose[0], G=pose[1], Wd=pose[2], rows=pose[3], cols=pose[4], shift=0.5, eps=eps,
                kind=kind)


def _blocks(dims, fill, blocks):
    lab = np.full(dims, fill, np.uint8)
    for label, sl in blocks:
        lab[sl] = label
    return lab


def _oblique():
    """A non-cubic volume, a 37 x 53 detector (partial 8 x 16 tiles both ways), three structures labelled 0, 255 and 7 over a
    tissue label 1, and the background slot."""
    dims = (40, 56, 36)
    lab = _blocks(dims, 1, [(0, np.s_[4:16, 6:26, 5:20]), (255, np.s_[20:34, 30:50, 12:30]), (7, np.s_[10:30, 8:20, 22:34])])
    return _scene(dims, 37, 53, 2, [(0,), (255,), (7,)], True, lab, seed=1)


def _source_straddle():
    """Slot 0's source lies inside its structure's box (the footprint falls back to the whole detector); slot 1 is an
    ordinary view."""
    dims = (32, 40, 28)
    lab = _blocks(dims, 1, [(3, np.s_[8:24, 10:30, 6:22]), (5, np.s_[24:30, 2:8, 20:27])])
    inside = dict(kind="inside", src=(15.3125, 19.6875, 13.4375))
    return _scene(dims, 24, 29, 2, [(3,), (5,)], True, lab, views={(0, 0): inside, (1, 0): inside}, kind="straddle", seed=2)


def _off_clipped():
    """Slot 0's detector is moved two half-widths aside (its box projects off the detector: an empty rectangle); slot 1's by
    one half-width along u in pose 0 and along v in pose 1 (its box straddles a detector edge: a clipped rectangle)."""
    dims = (36, 30, 44)
    lab = _blocks(dims, 1, [(2, np.s_[12:22, 10:20, 14:26]), (4, np.s_[14:24, 8:22, 16:30])])
    views = {(0, 0): dict(shift_uv=(2.5, 0.0)), (1, 0): dict(shift_uv=(0.0, -2.5)),
             (0, 1): dict(shift_uv=(1.0, 0.0)), (1, 1): dict(shift_uv=(0.0, 1.0))}
    return _scene(dims, 29, 41, 2, [(2,), (4,)], True, lab, views=views, kind="off_clipped", seed=3)


def _volume_face():
    """Boxes that reach the volume's faces: lo = 0 on axis 0 and hi = D on axis 1; hi = D on axes 0 and 2 and lo = 0 on
    axis 1."""
    dims = (24, 32, 20)
    lab = _blocks(dims, 1, [(2, np.s_[0:10, 4:32, 3:12]), (9, np.s_[14:24, 0:8, 10:20])])
    return _scene(dims, 33, 27, 2, [(2,), (9,)], True, lab, kind="volume_face", seed=4)


def _thin():
    """A one-voxel structure and a one-voxel-thick slab."""
    dims = (20, 24, 28)
    lab = _blocks(dims, 1, [(4, np.s_[9:10, 11:12, 13:14]), (8, np.s_[2:18, 15:16, 3:25])])
    return _scene(dims, 31, 35, 2, [(4,), (8,)], True, lab, kind="thin", seed=5)


def _flipped():
    """Decreasing rows and cols (negative delx / dely)."""
    dims = (28, 36, 24)
    lab = _blocks(dims, 1, [(6, np.s_[4:14, 6:20, 5:15]), (2, np.s_[16:26, 18:32, 10:22])])
    return _scene(dims, 26, 31, 2, [(6,), (2,)], True, lab, kind="flipped", seed=6, flip=True)


def _line(H, W):
    """A one-row or one-column detector through the detector's middle."""
    dims = (30, 26, 34)
    lab = _blocks(dims, 1, [(3, np.s_[6:20, 5:18, 8:26]), (7, np.s_[18:28, 14:24, 2:12])])
    kw = dict(rows=[0.0]) if H == 1 else dict(cols=[0.0])
    return _scene(dims, H, W, 2, [(3,), (7,)], True, lab, kind="line", seed=7, **kw)


def _multi_label():
    """Labels 3 and 11 share slot 0 (box = the union of theirs); label 6 lies inside that union and belongs to slot 1, so the
    gate, not the box, keeps it out of slot 0."""
    dims = (32, 28, 36)
    lab = _blocks(dims, 1, [(3, np.s_[2:12, 3:12, 4:14]), (11, np.s_[20:30, 16:26, 22:33]), (6, np.s_[13:19, 13:15, 15:21])])
    return _scene(dims, 30, 34, 2, [(3, 11), (6,)], True, lab, kind="multi_label", seed=8)


LATTICE_DIMS = (16, 32, 8)


def _lattice(S):
    """Exact ties (siddon_cases.lattice_ties, eps = 0): power-of-two dims, label-box faces on interior planes, every slot its
    own 2 x 2 pose-in detector.  S = 1: one structure, no background; S = 3: two structures and the background."""
    B = 512 if S == 1 else 192
    dims = LATTICE_DIMS
    lab = _blocks(dims, 1, [(5, np.s_[3:11, 5:20, 2:6]), (9, np.s_[8:16, 20:29, 4:8])])
    src, _, _, G, Wd, rows, cols = sc.lattice_ties(dims, B * S, seed=1 + S)
    slots = [(5,)] if S == 1 else [(5,), (9,)]
    return _scene(dims, 2, 2, B, slots, S == 3, lab, kind="lattice", eps=0.0, pose=(src, G, Wd, rows, cols), seed=9)


SCENES = {
    "oblique": _oblique, "source_straddle": _source_straddle, "off_clipped": _off_clipped, "volume_face": _volume_face,
    "thin": _thin, "flipped": _flipped, "line_h1": lambda: _line(1, 61), "line_w1": lambda: _line(45, 1),
    "multi_label": _multi_label, "lattice_s1": lambda: _lattice(1), "lattice_s3": lambda: _lattice(3),
}


@functools.lru_cache(maxsize=None)
def scene(name):
    """The scene with its fp64 rays (tgt (BS, N, 3), raylen (BS, N); tgt is exact in fp32), its masked densities (S, D0, D1,
    D2) and its ray classes (siddon_cases.classify of the same rays)."""
    c = SCENES[name]()
    tgt, raylen, p = sc.pose_rays(c["G"], c["Wd"], c["rows"], c["cols"])
    assert (tgt.astype(np.float32) == tgt).all(), name
    in_slot = c["slot"][c["lab"]]
    masked = np.stack([c["vol"] * (in_slot == s) for s in range(c["S"])])
    cls = sc.classify(c["vol"].shape, c["src"], tgt, c["shift"], c["eps"])
    return dict(c, name=name, tgt=tgt, raylen=raylen, p=p, masked=masked, cls=cls, N=tgt.shape[1])


def oracle_rays(c, dtype):
    """fp64 / fp32 oracle per (pose, slot) on its masked density: image (BS, N) and per-ray g_target, g_source (BS, N, 3) for a
    unit upstream gradient (each ray run as its own pose)."""
    from oracle import oracle
    BS, N = c["tgt"].shape[:2]
    img = np.empty((BS, N))
    gt = np.empty((BS, N, 3))
    gs = np.empty((BS, N, 3))
    kw = dict(voxel_shift=c["shift"], eps=c["eps"], dtype=dtype)
    for bs in range(BS):
        v = c["masked"][bs % c["S"]]
        s, t, l = c["src"][bs], c["tgt"][bs], c["raylen"][bs]
        img[bs] = oracle.siddon_fwd(v, s[None, None], t[None], l[None, None], **kw).reshape(N)
        r = oracle.siddon_bwd(v, np.repeat(s[None, None], N, 0), t[:, None], l.reshape(N, 1, 1), np.ones((N, 1, 1)),
                              want_vol=False, **kw)
        gt[bs], gs[bs] = r["g_target"].reshape(N, 3), r["g_source"].reshape(N, 3)
    return dict(image=img, g_target=gt, g_source=gs)


@functools.lru_cache(maxsize=None)
def references(name):
    """(fp64, fp32) oracle_rays of a scene."""
    c = scene(name)
    return oracle_rays(c, np.float64), oracle_rays(c, np.float32)


def uncut_emulated(c):
    """The host emulation of the un-cut walk (one walk over the whole ray, no box) on each slot's masked density, same fp32
    rays: (BS, N, 8) in the sensitivities layout [jt, -, js, -] (only 0:3 and 4:7 are filled)."""
    from hostemu import emu
    BS, N = c["tgt"].shape[:2]
    out = np.zeros((BS, N, 8))
    for bs in range(BS):
        r = emu.siddon_bwd(c["masked"][bs % c["S"]], np.repeat(c["src"][bs][None, None], N, 0),
                           c["tgt"][bs][:, None].astype(np.float32), c["raylen"][bs].reshape(N, 1).astype(np.float32),
                           np.ones((N, 1, 1)), voxel_shift=c["shift"], eps=c["eps"])
        out[bs, :, 0:3], out[bs, :, 4:7] = r["g_target"].reshape(N, 3), r["g_source"].reshape(N, 3)
    return out


def _per_slot(got, ref, keep):
    """Largest per-ray error over the kept rays of each (pose, slot), over that pair's reference maximum; the worst pair."""
    worst = 0.0
    for bs in range(ref.shape[0]):
        worst = max(worst, sc.per_ray_err(got[bs:bs + 1], ref[bs:bs + 1], None if keep is None else keep[bs:bs + 1]))
    return worst


def tie_rays(c):
    """Rays whose end-point sensitivities are pinned to the un-cut walk: near-tie rays, and every lattice ray but near-face ones."""
    cls = c["cls"]
    return cls["near_tie"] | ((c["kind"] == "lattice") & ~cls["near_face"])


def check_walk(c, out, sens, uncut, record, where):
    """The per-ray bounds of the module docstring for one structures walk: out (BS, N), sens (BS, N, 8); uncut (BS, N, 8) the
    un-cut walk's sensitivities on the same rays.  record(what, where, err, bound) asserts."""
    r64, r32 = references(c["name"])
    cls = c["cls"]
    out, sens = np.asarray(out, np.float64), np.asarray(sens, np.float64)
    BS, N = c["tgt"].shape[:2]
    out, sens = out.reshape(BS, N), sens.reshape(BS, N, 8)
    keep_img = ~cls["near_face"]
    lattice = c["kind"] == "lattice"
    record("image", where, _per_slot(out, r64["image"], keep_img), TIE_TOL if lattice else IMAGE_TOL)
    jt, js = sens[..., 0:3], sens[..., 4:7]
    if not lattice:
        keep = ~sc.excluded(cls, "sens")
        for what, got, key in (("sens target", jt, "g_target"), ("sens source", js, "g_source")):
            bound = sc.siddon_tol(_per_slot(r32[key], r64[key], keep), SENS_FLOOR)
            record(what, where, _per_slot(got, r64[key], keep), bound)
    tie = tie_rays(c)
    if tie.any():
        S = c["S"]
        for what, got, sl in (("ties target vs uncut", jt, np.s_[..., 0:3]), ("ties source vs uncut", js, np.s_[..., 4:7])):
            ref = uncut[sl]
            # over the slot's largest value in any pose: a lattice pose has 4 rays, and the un-cut walk is exactly 0 on a ray
            # that only touches the slot's box at an edge or corner
            scale = np.abs(ref).reshape(BS // S, S, -1).max(axis=(0, 2))
            worst = 0.0
            for bs in range(BS):
                if tie[bs].any():
                    err = np.abs(got[bs][tie[bs]] - ref[bs][tie[bs]]).max()
                    worst = max(worst, float(err / max(scale[bs % S], 1e-30)))
            record(what, where, worst, TIE_TOL)
    d = c["tgt"] - c["src"].astype(np.float64)[:, None, :] + c["eps"]
    scale = (np.abs(jt * d).sum(-1) + np.abs(js * d).sum(-1)).max(1) + np.abs(out).max(1)   # the terms' magnitude per slot
    scale = np.maximum(scale, 1e-30)[:, None]
    record("identity dt.d = -I", where, float((np.abs((jt * d).sum(-1) + out) / scale).max()), IDENTITY_TOL)
    record("identity (ds+dt).d = 0", where, float((np.abs(((jt + js) * d).sum(-1)) / scale).max()), IDENTITY_TOL)
    assert not sens[..., 7].any(), where


def excluded_fractions(c):
    """(near-face fraction, near-face or near-tie fraction) of the scene's rays."""
    cls = c["cls"]
    return float(cls["near_face"].mean()), float(sc.excluded(cls, "sens").mean())
