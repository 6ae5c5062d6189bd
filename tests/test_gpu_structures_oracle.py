"""Every piecewise-rigid entry point against the fp64 oracle, ray by ray, on the scenes of structures_cases.py: a non-cubic
volume with partial tiles and labels 0 and 255, a source inside a structure's box, boxes projecting off and across the detector
edges, boxes on the volume's faces, one-voxel structures, decreasing pixel coordinates, one-row and one-column detectors, two
labels in one slot, and exact-tie lattices; then DRR.structures_jacobian and the block-sparse normal equations on the Jacobians
those renders produce.

Kernels are called through the C ABI; every overwritten output is NaN-filled first.  Bounds (structures_cases):
  image                per ray, <= 1e-4 of the slot's fp64 maximum (1e-5 on the lattices), near-face rays excluded;
  sensitivities        per ray: well-conditioned rays against the oracle at siddon_tol; near-tie rays and every lattice ray
                       against the un-cut walk (b200drr_siddon_fwd_sens on the masked density, same fp32 rays) at 1e-5; the two
                       telescoping identities on every ray;
  backward             b200drr_siddon_bwd_sens_pose at batch B*S against the fp64 contraction of the kernel's own per-ray values;
  culling              every pixel the oracle sees lies in the b200drr_structure_footprints rectangle, and outside it the image and
                       all 8 sensitivity channels are exactly 0;
  16-bit               fp16 / bf16 against the oracle on the upcast masked density, bitwise the fp32 kernel on the upcast volume;
  Jacobian             exactly 0 outside the returned rectangles; the six columns of a structure against an fp64 central
                       difference of the fp64 renderer on density x mask;
  normal equations     on those Jacobians against the host emulation (1e-11) and the dense float64 statement (1e-9)."""
import ctypes

import numpy as np
import pytest
import torch

import structures_cases as stc
import trilinear_cases as tc
from conftest import relerr
from gpu_common import DEV

pytestmark = pytest.mark.gpu

ENTRIES = ("b200drr_label_boxes", "b200drr_siddon_fwd_sens_structures", "b200drr_siddon_fwd_sens_structures_v16",
           "b200drr_structure_footprints", "b200drr_ncc_normal_structures")
SEEN = set()
WORST = {}   # quantity -> (largest observed error / its bound, error, bound, where)
VOL16 = {torch.float16: 1, torch.bfloat16: 2}


@pytest.fixture(autouse=True)
def _entry_points(monkeypatch):
    from diffdrr_b200 import _lib
    lib = _lib.load()
    for name in _lib.exported_symbols():
        if name.startswith(ENTRIES):
            fn = getattr(lib, name)

            def wrap(*a, _fn=fn, _name=name):
                SEEN.add(_name)
                return _fn(*a)
            wrap.__name__ = name
            monkeypatch.setattr(lib, name, wrap)


def _call(name, *args):
    from diffdrr_b200 import _lib as L
    lib = L.load()
    L.check(getattr(lib, name)(*args, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), name)


def _p(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def _t(a, dtype=np.float32):
    return torch.as_tensor(np.ascontiguousarray(a, dtype)).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _np(x):
    out = x.cpu().numpy()
    assert np.isfinite(out).all()
    return out


def _record(what, where, err, bound):
    print(f"{what:26s} {where:40s} err {err:.2e} bound {bound:.2e}")
    if what not in WORST or err / bound > WORST[what][0]:
        WORST[what] = (err / bound, err, bound, where)
    assert err <= bound, (what, where, err, bound)


def _inputs(c, vol=None):
    vol = _t(c["vol"]) if vol is None else vol
    return dict(vol=vol, lab=torch.as_tensor(c["lab"]).to(DEV), src=_t(c["src"]), G=_t(c["G"]), Wd=_t(c["Wd"]),
                rows=_t(c["rows"]), cols=_t(c["cols"]), slot=_t(c["slot"], np.int32), box=_t(c["box"], np.int32))


def _structures(c, d, sens=True, vol16=None):
    """One launch of b200drr_siddon_fwd_sens_structures (or its _v16 twin on the 16-bit volume vol16) -> out, sens."""
    BS, N = c["G"].shape[0], c["H"] * c["W"]
    out, sn = _nan(BS, N), (_nan(BS, N, 8) if sens else None)
    tail = (_p(d["lab"]), *c["vol"].shape, _p(d["src"]), _p(d["G"]), _p(d["Wd"]), _p(d["rows"]), _p(d["cols"]), _p(d["slot"]),
            _p(d["box"]), _p(out), _p(sn), c["B"], c["S"], c["H"], c["W"], c["shift"], c["eps"])
    if vol16 is None:
        _call("b200drr_siddon_fwd_sens_structures", _p(d["vol"]), *tail)
    else:
        _call("b200drr_siddon_fwd_sens_structures_v16", _p(vol16), VOL16[vol16.dtype], *tail)
    return out, sn


def _uncut(c):
    """The un-cut walk (b200drr_siddon_fwd_sens) on each slot's masked density, over the scene's fp32 rays: (BS, N, 8)."""
    BS, N, S = c["G"].shape[0], c["H"] * c["W"], c["S"]
    res = np.empty((BS, N, 8))
    for s in range(S):
        vol = _t(c["masked"][s])
        src, tgt, raylen = _t(c["src"][s::S]), _t(c["tgt"][s::S]), _t(c["raylen"][s::S])
        n = src.shape[0]
        out, sens = _nan(n, N), _nan(n, N, 8)
        _call("b200drr_siddon_fwd_sens", _p(vol), *c["vol"].shape, _p(src), _p(tgt), _p(raylen), _p(out), _p(sens), n, N, c["shift"],
              c["eps"])
        res[s::S] = _np(sens)
    return res


def _footprints(c, d):
    rects = torch.full((c["G"].shape[0], 4), -7, dtype=torch.int32, device=DEV)
    _call("b200drr_structure_footprints", _p(d["src"]), _p(d["G"]), _p(d["rows"]), _p(d["cols"]), _p(d["box"]), _p(rects), c["B"],
          c["S"], c["H"], c["W"], c["shift"])
    return rects.cpu().numpy()


def _oracle_image(c, masked):
    from oracle import oracle
    BS, N = c["tgt"].shape[:2]
    return np.stack([oracle.siddon_fwd(masked[bs % c["S"]], c["src"][bs][None, None], c["tgt"][bs][None], c["raylen"][bs][None, None],
                                       voxel_shift=c["shift"], eps=c["eps"], dtype=np.float64).reshape(N) for bs in range(BS)])


@pytest.mark.parametrize("name", list(stc.SCENES))
def test_structures_walk_vs_oracle(name):
    c = stc.scene(name)
    BS, N, S, H, W = c["G"].shape[0], c["H"] * c["W"], c["S"], c["H"], c["W"]
    d = _inputs(c)
    out, sens = _structures(c, d)
    o, s = _np(out), _np(sens)
    stc.check_walk(c, o, s, _uncut(c), _record, name)
    # the backward of the render: bwd_sens_pose at batch B*S against the fp64 contraction of the kernel's own per-ray values
    gout_np = (np.random.default_rng(3).random((BS, N)) + 0.25).astype(np.float32)
    gout = _t(gout_np)
    g64 = gout_np.astype(np.float64)[..., None]
    s64 = s.astype(np.float64)
    dl = np.einsum("bij,nj->bni", c["Wd"].astype(np.float64), c["p"])
    u = dl / np.linalg.norm(dl, axis=-1, keepdims=True)
    for stop in (0, 1):
        got = dict(g_source=_nan(BS, 3), g_G=_nan(BS, 3, 4), g_Wd=_nan(BS, 3, 4))
        _call("b200drr_siddon_bwd_sens_pose", _p(sens), _p(gout), _p(d["Wd"]), _p(d["rows"]), _p(d["cols"]), _p(got["g_source"]),
              _p(got["g_G"]), _p(got["g_Wd"]), BS, H, W, stop)
        g_len = np.zeros((BS, N, 1)) if stop else g64 * s64[..., 3:4]
        terms = dict(g_source=g64 * s64[..., 4:7], g_G=(g64 * s64[..., 0:3])[..., :, None] * c["p"][None, :, None, :],
                     g_Wd=(g_len * u)[..., :, None] * c["p"][None, :, None, :])
        for k, t in terms.items():
            ref, mag = t.sum(1), np.abs(t).sum(1).reshape(BS, -1).max(1)
            err = np.abs(_np(got[k]) - ref).reshape(BS, -1).max(1) / np.maximum(mag, 1e-30)
            _record(f"bwd_sens_pose {k}", f"{name}/stop{stop}", float(err.max()), 1e-5)
    # culling: the oracle's pixels inside the footprint rectangles, exact zeros outside them
    rects = _footprints(c, d)
    img64 = stc.references(name)[0]["image"].reshape(BS, H, W)
    hh, ww = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    o3, s3 = o.reshape(BS, H, W), s.reshape(BS, H, W, 8)
    for bs in range(BS):
        w0, w1, h0, h1 = rects[bs]
        outside = (ww < w0) | (ww > w1) | (hh < h0) | (hh > h1)
        assert not (img64[bs][outside] != 0).any(), (name, bs)
        assert not o3[bs][outside].any() and not s3[bs][outside].any(), (name, bs)
    rect = rects.reshape(c["B"], S, 4)
    if c["kind"] == "straddle":
        assert (rect[:, 0] == [0, W - 1, 0, H - 1]).all()
    if c["kind"] == "off_clipped":
        assert ((rect[:, 0, 0] > rect[:, 0, 1]) | (rect[:, 0, 2] > rect[:, 0, 3])).all()
        assert rect[0, 1, 0] == 0 and rect[1, 1, 2] == 0
    # the image-only launch (sens = NULL) and determinism
    lean, _ = _structures(c, d, sens=False)
    keep = ~c["cls"]["near_face"]
    _record("image-only vs sens", name, stc._per_slot(_np(lean).astype(np.float64), o.astype(np.float64), keep), stc.LEAN_TOL)
    out2, sens2 = _structures(c, d)
    assert torch.equal(out2, out) and torch.equal(sens2, sens)
    lean2, _ = _structures(c, d, sens=False)
    assert torch.equal(lean2, lean)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", ["oblique", "source_straddle", "off_clipped", "thin", "multi_label", "lattice_s3"])
def test_16bit_densities(name, dtype):
    """The _v16 twin against the oracle on the upcast masked density, and bitwise the fp32 kernel on the upcast volume."""
    c = stc.scene(name)
    v16 = torch.as_tensor(c["vol"]).to(dtype).to(DEV)
    up = v16.float()
    d = _inputs(c, vol=up)
    out16, sens16 = _structures(c, d, vol16=v16)
    out32, sens32 = _structures(c, d)
    assert torch.equal(out16, out32) and torch.equal(sens16, sens32)
    out16n, _ = _structures(c, d, sens=False, vol16=v16)
    out32n, _ = _structures(c, d, sens=False)
    assert torch.equal(out16n, out32n)
    up_np = up.cpu().numpy()
    in_slot = c["slot"][c["lab"]]
    masked = np.stack([up_np * (in_slot == s) for s in range(c["S"])])
    ref = _oracle_image(c, masked)
    tol = stc.TIE_TOL if c["kind"] == "lattice" else stc.IMAGE_TOL
    _record("image 16-bit", f"{name}/{str(dtype)[6:]}", stc._per_slot(_np(out16).astype(np.float64), ref, ~c["cls"]["near_face"]), tol)


def test_label_boxes_match_numpy():
    """A scattered-label volume with labels 0 and 255, and every scene's label volume."""
    rng = np.random.default_rng(0)
    dims = (37, 29, 45)
    lab = np.full(dims, 17, np.uint8)
    lab[rng.random(dims) < 0.01] = 0
    lab[rng.random(dims) < 0.003] = 255
    lab[3:9, 20:25, 40:45] = 200
    lab[36, 0, 0] = 1
    for where, L in [("scattered", lab)] + [(n, stc.scene(n)["lab"]) for n in stc.SCENES]:
        d = torch.as_tensor(np.ascontiguousarray(L)).to(DEV)
        boxes = torch.full((256, 6), -9, dtype=torch.int32, device=DEV)
        _call("b200drr_label_boxes", _p(d), *L.shape, _p(boxes))
        got, ref = boxes.cpu().numpy(), stc.label_boxes(L)
        present = np.isin(np.arange(256), np.unique(L))
        assert np.array_equal(got[present], ref[present]), where
        assert ((got[~present, :3] > got[~present, 3:]).any(axis=1)).all(), where


# ---- Jacobians and the block-sparse normal equations on them -----------------------------------------------------------------
KW = dict(parameterization="euler_angles", convention="ZXY")
JAC_B, JAC_H = 3, 40


def _jacobian_case(kind):
    """(drr, rot, xyz, motions (B, K, 4, 4), labels, scene) of the oblique scene's labels with a smooth density, in world
    coordinates: 'oblique' small motions of (0, 255, 7, 1) -- label 1 is the tissue around them, a whole-volume structure;
    'clipped' structure 0 moved across the detector's edge and structure 1 off the detector; 'straddle' structure 0 moved
    onto each pose's source."""
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import RigidTransform, convert
    from diffdrr_b200.structures import structure_pivots
    c = stc.scene("oblique")
    vol = tc.volume(c["vol"].shape) + 0.25
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(c["lab"].astype(np.float32))),
              **synthetic.detector_kwargs(JAC_H, JAC_H + 5)).to(DEV)
    rot, xyz = (t.to(DEV) for t in synthetic.make_poses(JAC_B, seed=4, rot_range=0.3, xyz_range=10.0))
    labels = (0, 255, 7, 1) if kind == "oblique" else (0, 255, 7)
    K = len(labels)
    g = torch.Generator().manual_seed(5)
    m = convert((torch.rand(JAC_B * K, 3, generator=g) * 2 - 1) * 0.05, (torch.rand(JAC_B * K, 3, generator=g) * 2 - 1) * 4.0,
                parameterization="euler_angles", convention="XYZ").matrix.reshape(JAC_B, K, 4, 4).to(DEV)
    if kind == "oblique":
        return drr, rot, xyz, m, labels
    P = convert(rot, xyz, **KW).matrix
    src_v = drr._pose_in_inputs(RigidTransform(P), None)[0].double()
    A = drr._affine.reshape(4, 4).double()
    s_w = src_v @ A[:3, :3].mT + A[:3, 3]
    c0 = structure_pivots(drr, labels)[0]
    X = torch.eye(4, dtype=torch.float64, device=DEV).repeat(JAC_B, K, 1, 1)
    X[:, 1:] = m[:, 1:].double()
    if kind == "straddle":   # the structure's box centre (plus a little) onto the source
        X[:, 0, :3, 3] = s_w - c0 - torch.tensor([0.3, -0.2, 0.1], dtype=torch.float64, device=DEV)
    else:
        # structure 1 far to the side (off the detector); structure 0 along world x to the middle of the translations at which
        # its footprint (host build of b200drr_structure_footprints) is cut by a detector edge
        from diffdrr_b200.structures import _mask_state, _slot_inputs, _slots
        from hostemu import emu_ncc_normal_structures as emu
        X[:, 1, :3, 3] = torch.tensor([420.0, 0.0, 0.0], dtype=torch.float64, device=DEV)
        box = _slots(_mask_state(drr), labels, True, tuple(drr.density.shape))[1].cpu().numpy()
        H, W = JAC_H, JAC_H + 5
        for b in range(JAC_B):
            cut = []
            for a in np.arange(0.0, 300.0, 4.0):
                X[b, 0, 0, 3] = a
                src, G, _, rows, cols = (t.cpu().numpy() for t in _slot_inputs(drr, P[b:b + 1], X[b:b + 1].float(), K, True, None))
                w0, w1, h0, h1 = emu.footprints(src, G, rows, cols, box, K + 1)[0]
                edge = w0 == 0 or w1 == W - 1 or h0 == 0 or h1 == H - 1
                if w0 <= w1 and h0 <= h1 and edge and (w1 - w0 + 1) * (h1 - h0 + 1) < H * W:
                    cut.append(a)
            assert cut, b
            X[b, 0, 0, 3] = float(np.median(cut))
    return drr, rot, xyz, X.float(), labels


@pytest.mark.parametrize("kind", ["oblique", "clipped", "straddle"])
def test_jacobian_footprints_and_central_differences(kind):
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import RigidTransform, convert
    from diffdrr_b200.structures import _translation, structure_pivots, structures_jacobian, twist_matrix
    drr, rot, xyz, X, labels = _jacobian_case(kind)
    img, J, rects = structures_jacobian(drr, rot, xyz, motions=X, labels=labels, return_footprints=True, **KW)
    B, K, H, W = J.shape[:4]
    r = rects.cpu().numpy()
    Jn = J.cpu().numpy()
    hh, ww = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    for b in range(B):
        for k in range(K):
            w0, w1, h0, h1 = r[b, k]
            outside = (ww < w0) | (ww > w1) | (hh < h0) | (hh > h1)
            assert not Jn[b, k][outside].any(), (kind, b, k)
    if kind == "straddle":
        assert (r[:, 0] == [0, W - 1, 0, H - 1]).all()
    if kind == "clipped":
        assert (r[:, 0, 0] == 0).any() or (r[:, 0, 1] == W - 1).any() or (r[:, 0, 2] == 0).any() or (r[:, 0, 3] == H - 1).any()
        assert ((r[:, 0, 1] - r[:, 0, 0] + 1) * (r[:, 0, 3] - r[:, 0, 2] + 1) < H * W).all()
        assert ((r[:, 1, 0] > r[:, 1, 1]) | (r[:, 1, 2] > r[:, 1, 3])).all()
    # the six columns of structure 0 against an fp64 central difference of the fp64 renderer on density * mask
    lab = drr.mask.cpu().numpy()
    dens = drr.density.cpu().numpy()
    ref = DRR(synthetic.make_subject(dens * (lab == labels[0])), **synthetic.detector_kwargs(JAC_H, JAC_H + 5)).to(DEV)
    ref = ref.to(torch.float64)
    wimg = 1.0 + torch.rand(B, H, W, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV, dtype=torch.float64)
    an = torch.einsum("bhw,bhwi->i", wimg, J[:, 0].double()).cpu().numpy()
    P = convert(rot.double(), xyz.double(), **KW).matrix
    c = structure_pivots(drr, labels)[0]
    h = 1e-6

    def f(i, s):
        xi = torch.zeros(6, dtype=torch.float64, device=DEV)
        xi[i] = s
        Xk = _translation(c) @ torch.linalg.matrix_exp(twist_matrix(xi)) @ _translation(-c) @ X[:, 0].double()
        with torch.no_grad():
            return float((wimg * ref(RigidTransform(torch.linalg.inv(Xk) @ P))[:, 0]).sum())

    fd = np.array([(f(i, h) - f(i, -h)) / (2 * h) for i in range(6)])
    _record("jacobian vs fp64 fd", kind, float(np.abs(an - fd).max() / np.abs(fd).max()), 1e-3)
    _normal_equations(kind, img, J, rects)


def _dense(x, t, J, eps):
    B, K = J.shape[:2]
    HW = x[0].numel()
    Jd = J.reshape(B, K, HW, 6).permute(0, 2, 1, 3).reshape(B, HW, 6 * K).double()
    x, t = x.double().flatten(1), t.double().flatten(1)

    def norm(a):
        mu = a.mean(-1, keepdim=True)
        s = (((a - mu) ** 2).mean(-1, keepdim=True) + eps).sqrt()
        return (a - mu) / s, s

    z, s = norm(x)
    zt, _ = norm(t)
    Jz = (Jd - Jd.mean(1, keepdim=True) - z[..., None] * (z[..., None] * Jd).mean(1, keepdim=True)) / s[..., None]
    return torch.einsum("bqk,bql->bkl", Jz, Jz), torch.einsum("bqk,bq->bk", Jz, z - zt)


def _normal_equations(kind, img, J, rects):
    """b200drr_ncc_normal_structures on the real Jacobians: K = 1 and every K (4 on the oblique case), t_batch 1 and B, the
    non-contiguous J[:, :K] view, against the emulation and the dense statement; two calls at weight 1 = one at weight 2."""
    from diffdrr_b200.registration import ncc_normal_structures_equations
    from hostemu import emu_ncc_normal_structures as emu
    B, Kall, H, W = J.shape[:4]
    S = rects.shape[1]
    x = img.sum(1).contiguous()
    gen = torch.Generator(device=DEV).manual_seed(6)
    tB = (0.7 * x + 0.1 * torch.rand(x.shape, generator=gen, device=DEV)).contiguous()
    storage = J.as_strided((J.untyped_storage().nbytes() // 4,), (1,), 0).cpu().numpy()
    eps = 1e-5
    for K in sorted({1, Kall}):
        Jk = J[:, :K]
        assert not Jk.is_contiguous()
        for t in (tB[:1].contiguous(), tB):
            A = torch.zeros(B, 6 * K, 6 * K, dtype=torch.float64, device=DEV)
            g = torch.zeros(B, 6 * K, dtype=torch.float64, device=DEV)
            ncc_normal_structures_equations(x, t, Jk, rects, eps, 1.0, A, g)
            An, gn = A.cpu().numpy(), g.cpu().numpy()
            where = f"{kind}/K{K}/t{t.shape[0]}"
            Ae, ge = emu.ncc_normal_structures(x.cpu().numpy(), t.cpu().numpy(), storage, (Jk.stride(0), Jk.stride(1), Jk.stride(-2),
                                               Jk.stride(-1)), rects.cpu().numpy(), K, S, eps=eps)
            _record("normal eq vs emulation", where, max(relerr(An, Ae), relerr(gn, ge)), 1e-11)
            Ar, gr = _dense(x, t.expand(B, H, W), Jk, eps)
            _record("normal eq vs dense", where, max(relerr(An, Ar.cpu().numpy()), relerr(gn, gr.cpu().numpy())), 1e-9)
            ncc_normal_structures_equations(x, t, Jk, rects, eps, 1.0, A, g)
            A2 = torch.zeros_like(A)
            g2 = torch.zeros_like(g)
            ncc_normal_structures_equations(x, t, Jk, rects, eps, 2.0, A2, g2)
            assert torch.equal(A, A2) and torch.equal(g, g2), where


def test_every_structures_entry_point_ran():
    missing = [e for e in ENTRIES if e not in SEEN]
    for what, (ratio, err, bound, where) in sorted(WORST.items()):
        print(f"WORST {what:26s} err {err:.2e} bound {bound:.2e} ({ratio:.2f} of it) at {where}")
    assert not missing, missing
