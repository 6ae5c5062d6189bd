"""The scenes of structures_cases.py on the CPU: each is what its name says, the ray classes cover every ray the oracle cannot
resolve in fp32 on the masked densities, and the host emulation of csrc/structures.cu (the same source as the kernel) meets
the bounds the GPU test holds the kernel to -- on the exact-tie lattices too, where the box walk must attribute every tied
crossing as the un-cut walk of density x (label in slot) does."""
import numpy as np
import pytest

import structures_cases as stc
from hostemu import emu_ncc_normal_structures, emu_structures

NAMES = list(stc.SCENES)


def _emulate(c, **kw):
    return emu_structures.structures(c["vol"], c["lab"], c["src"], c["G"], c["Wd"], c["rows"], c["cols"], c["slot"], c["box"],
                                     c["S"], voxel_shift=c["shift"], eps=c["eps"], **kw)


def _is_empty(r):
    return r[0] > r[1] or r[2] > r[3]


@pytest.mark.parametrize("name", NAMES)
def test_scene_is_what_it_says(name):
    c = stc.scene(name)
    dims, B, S, H, W = c["vol"].shape, c["B"], c["S"], c["H"], c["W"]
    in_slot = c["slot"][c["lab"]]
    for s in range(S):   # every voxel of a slot's labels lies in its box
        idx = np.argwhere(in_slot == s)
        assert len(idx), (name, s)
        assert (idx >= c["box"][s, :3]).all() and (idx < c["box"][s, 3:]).all(), (name, s)
    rect = _emulate(c)["rect"]
    # the footprint entry point's host build gives the render's rectangles
    assert np.array_equal(rect, emu_ncc_normal_structures.footprints(c["src"], c["G"], c["rows"], c["cols"], c["box"], S,
                                                                      c["shift"]))
    rect = rect.reshape(B, S, 4)
    whole = [0, W - 1, 0, H - 1]
    img = stc.references(name)[0]["image"].reshape(B, S, H, W)
    for b in range(B):   # the culling is sound: every pixel the oracle sees lies in its rectangle
        for s in range(S):
            ys, xs = np.nonzero(img[b, s])
            w0, w1, h0, h1 = rect[b, s]
            assert ((xs >= w0) & (xs <= w1) & (ys >= h0) & (ys <= h1)).all(), (name, b, s)
    lo, hi = c["box"][:, :3], c["box"][:, 3:]
    kind = c["kind"]
    if name == "oblique":
        assert len(set(dims)) == 3 and H % 16 and W % 8 and {0, 255} <= {lab for sl in c["slots"] for lab in sl}
    elif kind == "straddle":   # slot 0's source inside its box: a corner behind the source, the whole detector
        src = c["src"].reshape(B, S, 3)[:, 0]
        assert ((src >= lo[0] - c["shift"]) & (src <= hi[0] - c["shift"])).all()
        assert (rect[:, 0] == whole).all()
    elif kind == "off_clipped":
        assert all(_is_empty(r) for r in rect[:, 0])
        assert not (img[:, 0] != 0).any()
        # slot 1 is cut by the detector's left edge in pose 0 and its top edge in pose 1, with the oracle nonzero on that edge
        assert rect[0, 1, 0] == 0 and rect[0, 1, 1] < W - 1 and (img[0, 1, :, 0] != 0).any()
        assert rect[1, 1, 2] == 0 and rect[1, 1, 3] < H - 1 and (img[1, 1, 0, :] != 0).any()
    elif kind == "volume_face":
        ends = hi[:-1] == np.asarray(dims)
        assert (lo[:-1] == 0).any(axis=1).all() and ends.any(axis=1).all()
    elif kind == "thin":
        ext = hi[:-1] - lo[:-1]
        assert (ext[0] == 1).all() and sorted(ext[1].tolist())[0] == 1
    elif kind == "flipped":
        assert (np.diff(c["rows"]) < 0).all() and (np.diff(c["cols"]) < 0).all()
    elif kind == "line":
        assert min(H, W) == 1 and max(H, W) > 16
    elif kind == "multi_label":
        assert len(c["slots"][0]) == 2
        b = c["box"][0]
        inner = in_slot[b[0]:b[3], b[1]:b[4], b[2]:b[5]]
        assert (inner == 1).any()   # the gate, not the box, keeps slot 1's label out of slot 0
    elif kind == "lattice":
        assert c["eps"] == 0.0 and all(d & (d - 1) == 0 for d in dims)
        # label-box faces on interior planes of every axis
        assert ((lo[:len(c["slots"])] > 0) | (hi[:len(c["slots"])] < np.asarray(dims))).all()
        assert (lo[0] > 0).all() and (hi[0] < np.asarray(dims)).all()


@pytest.mark.parametrize("name", NAMES)
def test_classes_cover_every_ray_the_oracle_cannot_resolve(name):
    """Rays on which the oracle's own fp32 and fp64 differ by more than 1e-5 of the slot's maximum: near-face for the image,
    near-face or near-tie for the end-point sensitivities."""
    c = stc.scene(name)
    r64, r32 = stc.references(name)
    cls = c["cls"]
    for key, covered in (("image", cls["near_face"]), ("g_target", cls["near_face"] | cls["near_tie"]),
                         ("g_source", cls["near_face"] | cls["near_tie"])):
        e = np.abs(r32[key] - r64[key])
        scale = np.abs(r64[key]).reshape(e.shape[0], -1).max(1)
        if e.ndim == 3:
            e = e.max(-1)
        bad = e > 1e-5 * np.maximum(scale, 1e-30)[:, None]
        assert not (bad & ~covered).any(), (name, key, int((bad & ~covered).sum()))
    face, excl = stc.excluded_fractions(c)
    print(f"{name}: near-face {face:.2%}, excluded from the sensitivities' oracle comparison {excl:.2%}")
    assert face < 0.01
    if c["kind"] != "lattice":
        assert excl < 0.02


@pytest.mark.parametrize("name", NAMES)
def test_emulation_meets_the_bounds(name):
    """The host build of the structures walk against the oracle and the un-cut walk (per ray), culled and unculled bitwise
    equal.  On the lattices this fails if the box walk books a crossing that ties with an interior entry face on another
    axis than the un-cut walk does."""
    c = stc.scene(name)
    got = _emulate(c)
    full = _emulate(c, cull=False)
    assert np.array_equal(got["out"], full["out"]) and np.array_equal(got["sens"], full["sens"])

    def record(what, where, err, bound):
        print(f"{what:24s} {where:20s} err {err:.2e} bound {bound:.2e}")
        assert err <= bound, (what, where, err, bound)

    stc.check_walk(c, got["out"], got["sens"], stc.uncut_emulated(c), record, name)
    lean = _emulate(c, sens=False)["out"]   # the image-only walk over the same boxes
    keep = ~c["cls"]["near_face"]
    record("image-only vs sens", name, stc._per_slot(lean.astype(np.float64), got["out"].astype(np.float64), keep), stc.LEAN_TOL)
