"""Every Siddon device path against the fp64 oracle, ray by ray, on the edge geometries of siddon_cases.py: ray-set, full-grid,
brick-major and pose-in launches, at shapes with partial tiles and bricks, thin volumes, sources inside the volume, misses, rays in
voxel faces, near-identical poses and exact ties.

Kernels are called through the C ABI with explicit variants; every overwritten output is NaN-filled first.  Bounds (siddon_cases):
  image                every ray but near-face ones, <= 1e-4 of the fp64 maximum (1e-5 on the lattice ties);
  g_raylen, g_volume   the SURVEY 8c rule, gout zeroed on near-face rays;
  end-point gradients  per ray: well-conditioned rays against the oracle at siddon_tol; near-tie rays and every lattice ray
                       against the un-cut walk (b200drr_siddon_bwd / fwd_sens_grid variant 34) at 1e-5 of the maximum, and that walk
                       against the host emulation of the same source on the lattice; the two telescoping identities on every ray;
  pose sums            against the fp64 contraction of the kernel's own per-ray gradients, at fp32 summation round-off."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import siddon_cases as sc
import trilinear_cases as tc
from conftest import relerr
from gpu_common import DEV

pytestmark = pytest.mark.gpu

FLOOR = dict(image=1e-4, g_raylen=1e-4, g_volume=1e-4, g_target=5e-4, g_source=1e-3)
TIE_TOL = 1e-5
ENTRIES = ("b200drr_siddon_fwd", "b200drr_siddon_fwd_general", "b200drr_siddon_bwd", "b200drr_siddon_bwd_general",
           "b200drr_siddon_fwd_sens", "b200drr_siddon_bwd_sens", "b200drr_siddon_fwd_sorted", "b200drr_siddon_fwd_sens_sorted",
           "b200drr_siddon_fwd_mask", "b200drr_siddon_bwd_mask", "b200drr_siddon_fwd_grid", "b200drr_siddon_bwd_grid",
           "b200drr_siddon_fwd_sens_grid", "b200drr_siddon_fwd_mask_grid", "b200drr_siddon_bwd_mask_grid", "b200drr_siddon_fwd_brick",
           "b200drr_siddon_fwd_brick_subset", "b200drr_siddon_bwd_vol_brick", "b200drr_siddon_fwd_pose", "b200drr_siddon_bwd_pose",
           "b200drr_siddon_fwd_sens_pose", "b200drr_siddon_bwd_sens_pose")
SEEN = set()
WORST = {}   # quantity -> (largest observed error / its bound, error, bound, where)


@pytest.fixture(autouse=True)
def _entry_points(monkeypatch):
    from diffdrr_b200 import _lib
    lib = _lib.load()
    for name in _lib.exported_symbols():
        if name.startswith("b200drr_siddon"):
            fn = getattr(lib, name)

            def wrap(*a, _fn=fn, _name=name):
                SEEN.add(_name)
                return _fn(*a)
            wrap.__name__ = name
            monkeypatch.setattr(lib, name, wrap)


def _lib():
    from diffdrr_b200 import _lib as L
    return L, L.load()


def _p(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def _call(name, *args):
    L, lib = _lib()
    L.check(getattr(lib, "b200drr_siddon_" + name)(*args, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), name)


def _t(a, dtype=np.float32):
    return torch.as_tensor(np.ascontiguousarray(a, dtype)).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _np(x):
    out = x.cpu().numpy()
    assert np.isfinite(out).all()
    return out


def _record(what, where, err, bound):
    print(f"{what:24s} {where:48s} err {err:.2e} bound {bound:.2e}")
    if what not in WORST or err / bound > WORST[what][0]:
        WORST[what] = (err / bound, err, bound, where)
    assert err <= bound, (what, where, err, bound)


# ---- cases --------------------------------------------------------------------------------------------------------------------
CASES = {  # name -> (geometry, shape)
    "A4/rotated": ("rotated", sc.SHAPE_A4), "A4/inside": ("inside", sc.SHAPE_A4), "A4/miss": ("miss", sc.SHAPE_A4),
    "thin/miss": ("miss", tc.SHAPE_THIN), "sliver/rotated": ("rotated", tc.SHAPE_SLIVER), "sliver/axis": ("axis", tc.SHAPE_SLIVER),
    "A/axis/s0": ("axis", tc.SHAPE_A), "near/16": ("near_identical", sc.SHAPE_NEAR),
    **{f"planar/A4/{f}": ("planar", sc.SHAPE_A4) for f in sc.planar_faces(sc.SHAPE_A4[0])},
    "planar/A4/15.5/s0": ("planar", sc.SHAPE_A4), "planar/thin/1.5": ("planar", tc.SHAPE_THIN),
    **{f"lattice/{i}": ("lattice", (d, 2, 2, 512)) for i, d in enumerate(sc.LATTICE_DIMS)},
    # exact ties on the pose-in walk's other two routes
    "lattice/pieces": ("lattice", ((128, 64, 64), 2, 2, 512)), "lattice/brick": ("lattice", ((512, 512, 256), 2, 2, 512)),
    "lattice_rays/0": ("lattice_rays", (sc.LATTICE_DIMS[0], 0, 0, 1000)),
    "brick_route/rotated": ("rotated", sc.SHAPE_BRICK_ROUTE),
}


@functools.lru_cache(maxsize=2)
def _case(name):
    """-> dict: vol, src, tgt, raylen (fp32 numpy), H, W (0 = no grid), shift, eps, pose (G, Wd, rows, cols) or None, cls."""
    geom, (dims, H, W, B) = CASES[name]
    shift = 0.0 if name.endswith("/s0") else 0.5
    eps, pose = 1e-8, None
    if geom in ("rotated", "inside"):
        src, G, Wd, rows, cols, t64, l64, _ = sc.cone_pose(geom, dims, H, W, B)
        tgt, raylen, pose = t64.astype(np.float32), l64.astype(np.float32), (G, Wd, rows, cols)
    elif geom in ("miss", "near_identical"):
        src, tgt, raylen = getattr(tc, geom)(dims, H, W, B, seed=2)
    elif geom == "axis":
        src, tgt, raylen = tc.axis(dims, H, W, shift)
    elif geom == "planar":
        src, tgt, raylen = sc.planar_axis(dims, H, W, float(name.split("/")[2]), shift)
        pose = sc.grid_matrices(src, tgt, H, W)
    elif geom == "lattice":
        src, tgt, raylen, *pose = sc.lattice_ties(dims, B, seed=1)
        pose = tuple(pose)
        eps = 0.0
    else:
        src, tgt, raylen = sc.lattice_rays(dims, B, seed=1)
        eps = 0.0
    return dict(vol=tc.volume(dims), src=src, tgt=tgt, raylen=raylen, H=H, W=W, shift=shift, eps=eps, pose=pose,
                cls=sc.classify(dims, src, tgt, shift, eps), lattice=geom.startswith("lattice"))


def _route(name):
    """The route b200drr_siddon_fwd_sens_pose takes on a case (siddon.cu: siddon_sens_brick_route, small_batch_pieces); the test
    asserts it from the launched kernel's name."""
    dims = CASES[name][1][0]
    return "brick" if name in ("brick_route/rotated", "lattice/brick") else "pieces" if max(dims) >= 96 else "slabs"


def _ref(c, gout, per_ray=False, **kw):
    """fp64 and fp32 oracle (image, per-ray g_target, g_raylen, g_volume, per-pose g_source and, with per_ray, the per-ray source
    gradients g_src_ray from every ray run as its own pose) for upstream gradient gout (B, N)."""
    from oracle import oracle
    B, N = c["tgt"].shape[:2]
    args = (c["vol"], c["src"][:, None], c["tgt"], c["raylen"][:, None])
    okw = dict(voxel_shift=c["shift"], eps=c["eps"])
    out = []
    bil = kw.pop("mode", 0) == 1
    for dt in (np.float64, np.float32):
        if bil:
            r = oracle.siddon_bilinear(*args, gout.reshape(B, 1, N), dtype=dt, **okw, **kw)
            img = r["img"]
        else:
            fkw = {k: v for k, v in kw.items() if k in ("reduce", "align_corners")}
            img = oracle.siddon_fwd(*args, dtype=dt, **okw, **fkw)
            r = oracle.siddon_bwd(*args, gout.reshape(B, 1, N), dtype=dt, **okw, **kw)
        out.append(dict(image=img.reshape(B, N), g_target=r["g_target"], g_raylen=r["g_raylen"].reshape(B, N),
                        g_volume=r["g_volume"], g_source=r["g_source"].reshape(B, 3)))
        if per_ray:
            rr = oracle.siddon_bwd(c["vol"], np.repeat(c["src"], N, axis=0)[:, None], np.asarray(c["tgt"]).reshape(B * N, 1, 3),
                                   np.asarray(c["raylen"]).reshape(B * N, 1, 1), gout.reshape(B * N, 1, 1), dtype=dt, want_vol=False,
                                   **okw)
            out[-1]["g_src_ray"] = rr["g_source"].reshape(B, N, 3)
    return out


def _gouts(c):
    B, N = c["tgt"].shape[:2]
    g = np.random.default_rng(7).random((B, N)) + 0.25
    ex = sc.excluded(c["cls"], "g_target")
    return (g * ~c["cls"]["near_face"]).astype(np.float32), (g * ~ex).astype(np.float32)


class Checker:
    """Compares one kernel's outputs with the oracle (r64, r32 for gout_all) and with the un-cut walk's per-ray end-point
    gradients uncut / uncut_src (B, N, 3) = gout x dI/dt, gout x dI/ds for the same gout."""

    def __init__(self, c, name, r64, r32, uncut, uncut_src=None, resolved=False):
        self.c, self.name, self.r64, self.r32, self.uncut, self.uncut_src = c, name, r64, r32, uncut, uncut_src
        cls = c["cls"]
        self.keep_img = ~cls["near_face"]
        self.keep_end = ~sc.excluded(cls, "g_target")
        self.resolved = resolved
        if resolved:   # options outside the classes' nearest-sum model: also leave out what the oracle cannot resolve itself
            self.keep_end = self.keep_end & _resolved(r32["g_target"], r64["g_target"])
        self.tie = cls["near_tie"] | (c["lattice"] & self.keep_img)

    def image(self, where, got):
        _record("image", f"{self.name} {where}", sc.per_ray_err(_np(got).reshape(self.r64["image"].shape), self.r64["image"],
                                                               self.keep_img), 1e-5 if self.c["lattice"] else FLOOR["image"])

    def grads(self, where, got, stop=False):
        w = f"{self.name} {where}"
        B, N = self.c["tgt"].shape[:2]
        if got.get("g_target") is not None:
            g = _np(got["g_target"]).reshape(B, N, 3)
            if not self.c["lattice"]:
                err32 = sc.per_ray_err(self.r32["g_target"], self.r64["g_target"], self.keep_end)
                _record("g_target", w, sc.per_ray_err(g, self.r64["g_target"], self.keep_end), sc.siddon_tol(err32, FLOOR["g_target"]))
            if self.uncut is not None and self.tie.any():
                s = np.abs(self.uncut).max()
                _record("g_target ties vs uncut", w, sc.per_ray_err(g, self.uncut, self.tie, scale=s), TIE_TOL)
        if got.get("g_source") is not None and self.uncut_src is not None:
            # per-pose sums, ties included, against the un-cut walk's per-ray source gradients summed in fp64
            ref, mag = self.uncut_src.sum(1), np.abs(self.uncut_src).sum(1).max()
            _record("g_source vs uncut", w, float(np.abs(_np(got["g_source"]) - ref).max() / max(mag, 1e-30)), TIE_TOL)
        if got.get("g_raylen") is not None:
            g = _np(got["g_raylen"]).reshape(B, N)
            if stop:
                assert not g.any(), w
            else:
                keep = _resolved(self.r32["g_raylen"], self.r64["g_raylen"]) if self.resolved else None
                bound = TIE_TOL if self.c["lattice"] else sc.siddon_tol(
                    sc.per_ray_err(self.r32["g_raylen"], self.r64["g_raylen"], keep), FLOOR["g_raylen"])
                _record("g_raylen", w, sc.per_ray_err(g, self.r64["g_raylen"], keep), bound)
        # sums over rays: the options compare them in a second run with gout zeroed on the rays they leave out (sums_vs_oracle)
        if got.get("g_volume") is not None and not stop and not self.resolved:
            bound = TIE_TOL if self.c["lattice"] else tc.tol(self.r32["g_volume"], self.r64["g_volume"], FLOOR["g_volume"])
            _record("g_volume", w, relerr(_np(got["g_volume"]), self.r64["g_volume"]), bound)

    def sens(self, where, sens, gout):
        """Per-ray source sensitivities gout x sens[4:7]: well-conditioned rays against the oracle, tie rays against the un-cut
        walk (the end-point ones, sens[0:3], are read through bwd_sens by grads)."""
        w = f"{self.name} {where}"
        B, N = self.c["tgt"].shape[:2]
        g = _np(sens).reshape(B, N, 8)[..., 4:7].astype(np.float64) * np.asarray(gout, np.float64).reshape(B, N, 1)
        if not self.c["lattice"]:
            err32 = sc.per_ray_err(self.r32["g_src_ray"], self.r64["g_src_ray"], self.keep_end)
            _record("g_src per ray", w, sc.per_ray_err(g, self.r64["g_src_ray"], self.keep_end), sc.siddon_tol(err32, FLOOR["g_target"]))
        if self.uncut_src is not None and self.tie.any():
            s = np.abs(self.uncut_src).max()
            _record("g_src ties vs uncut", w, sc.per_ray_err(g, self.uncut_src, self.tie, scale=s), TIE_TOL)

    def sums_vs_oracle(self, where, got, r64, r32, stop=False, gout=None):
        """Per-pose g_source and g_volume of a run whose gout is zero on every ray the comparison leaves out.  With gout given
        (max-reduction, align_corners) the volume gradient is checked by the adjoint identity <g_volume, vol> = sum gout x image
        instead of voxel by voxel: a midpoint on a lookup cell face between two voxels of zero density moves the scatter between
        them without changing the image or any per-ray gradient, so no per-ray comparison can tell that such a ray is unresolved."""
        w = f"{self.name} {where}"
        _record("g_source", w, relerr(_np(got["g_source"]), r64["g_source"]), tc.tol(r32["g_source"], r64["g_source"], FLOOR["g_source"]))
        if got.get("g_volume") is not None and not stop and gout is not None:
            lhs = float((_np(got["g_volume"]).astype(np.float64) * self.c["vol"]).sum())
            rhs = float((np.asarray(gout, np.float64) * r64["image"]).sum())
            _record("adjoint <g_vol, vol>", w, abs(lhs - rhs) / abs(rhs), TIE_TOL)
        elif got.get("g_volume") is not None and not stop:
            _record("g_volume", w, relerr(_np(got["g_volume"]), r64["g_volume"]),
                    tc.tol(r32["g_volume"], r64["g_volume"], FLOOR["g_volume"]))


def _resolved(a32, a64):
    """(B, N): rays on which the oracle's own fp32 and fp64 agree to 1e-5 of the maximum.  The ray classes model nearest sampling
    summed along the ray; with align_corners the lookup grid is not the crossing grid, and max-reduction and bilinear sampling
    have discontinuities of their own, so those comparisons also leave out the rays the oracle cannot resolve in fp32."""
    e = np.abs(np.asarray(a32, np.float64) - a64)
    if e.ndim == 3:
        e = e.max(-1)
    return e <= 1e-5 * np.abs(a64).max()


def _identities(where, c, img, sens):
    """Per ray: sum_a dI/dt_a d_a = -I and sum_a (dI/ds_a + dI/dt_a) d_a = 0, read from the sensitivities."""
    B, N = c["tgt"].shape[:2]
    s = _np(sens).astype(np.float64).reshape(B, N, 8)
    d = c["tgt"].astype(np.float64) - c["src"][:, None, :].astype(np.float64) + c["eps"]
    I = _np(img).astype(np.float64).reshape(B, N)
    scale = np.abs(s[..., :3] * d).sum(-1).max() + np.abs(I).max()
    _record("identity dI/dt.d = -I", where, float(np.abs((s[..., :3] * d).sum(-1) + I).max() / scale), 1e-5)
    _record("identity (ds+dt).d = 0", where, float(np.abs(((s[..., :3] + s[..., 4:7]) * d).sum(-1)).max() / scale), 1e-5)
    assert not s[..., 7].any()


def _bwd_sens(sens, gout, B, N, stop, pose=None, HW=None):
    got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N))
    _call("bwd_sens", _p(sens), _p(gout), _p(got["g_source"]), _p(got["g_target"]), _p(got["g_raylen"]), B, N, int(stop))
    return got


# ---- ray sets -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n in CASES if n not in ("brick_route/rotated", "lattice/pieces", "lattice/brick")])
def test_ray_set_kernels_vs_oracle(name):
    """fwd (sum / max x align_corners), fwd_general (nearest, bilinear), bwd and bwd_general, fwd_sens + bwd_sens, the sorted forms
    on a permuted ray order, fwd_mask / bwd_mask."""
    from oracle import oracle
    c = _case(name)
    vol_np, src_np, tgt_np, len_np = c["vol"], c["src"], c["tgt"], c["raylen"]
    dims, (B, N), sh, eps = vol_np.shape, tgt_np.shape[:2], c["shift"], c["eps"]
    g_all_np, g_end_np = _gouts(c)
    r64, r32 = _ref(c, g_all_np, per_ray=True)
    assert np.abs(r64["image"]).max() > 0
    vol, src, tgt, raylen, g_all = _t(vol_np), _t(src_np), _t(tgt_np), _t(len_np), _t(g_all_np)
    geo = (_p(vol), *dims, _p(src), _p(tgt), _p(raylen))
    # the un-cut walk: one thread walks each whole ray; its per-ray end-point gradients for gout = g_all
    out, sens0 = _nan(B, N), _nan(B, N, 8)
    _call("fwd_sens", *geo, _p(out), _p(sens0), B, N, sh, eps)
    s0 = _np(sens0).astype(np.float64)
    uncut, uncut_src = s0[..., :3] * g_all_np[..., None], s0[..., 4:7] * g_all_np[..., None]
    un = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
    _call("bwd", *geo, _p(g_all), *[_p(un[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, N, sh, eps, 0, 0)
    if c["lattice"]:   # the un-cut walks are the CPU-verified emulation of the same source, per ray
        from hostemu import emu
        e = emu.siddon_bwd(vol_np, src_np[:, None], tgt_np, len_np[:, None], g_all_np, eps=eps)
        _record("uncut vs emulation", f"{name} bwd", sc.per_ray_err(_np(un["g_target"]), e["g_target"]), 1e-6)
        e = emu.siddon_sens(vol_np, src_np[:, None], tgt_np, len_np[:, None], g_all_np, eps=eps, slab=0)
        _record("uncut vs emulation", f"{name} fwd_sens", sc.per_ray_err(uncut, e["g_target"]), 1e-6)
        _record("uncut vs emulation", f"{name} fwd_sens source", relerr(uncut_src.sum(1), e["g_source"].reshape(B, 3)), 1e-6)
    chk = Checker(c, name, r64, r32, uncut, uncut_src)
    chk.sens("fwd_sens (un-cut)", sens0, g_all_np)
    chk.grads("bwd", un)
    # the un-cut walk's per-pose source gradient over the well-conditioned rays, against the oracle
    e64, e32 = _ref(c, g_end_np)
    g_end = _t(g_end_np)
    chk.sums_vs_oracle("fwd_sens+bwd_sens (g_end)", _bwd_sens(sens0, g_end, B, N, 0), e64, e32)
    chk.image("fwd_sens (un-cut)", out)
    out.fill_(float("nan"))
    _call("fwd", *geo, _p(out), B, N, sh, eps, 0, 0)
    chk.image("fwd", out)
    for mode in (0, 1):
        out.fill_(float("nan"))
        _call("fwd_general", *geo, _p(out), B, N, sh, eps, 0, 0, mode)
        if mode == 0:
            chk.image("fwd_general/nearest", out)
        else:
            ref = oracle.siddon_bilinear(vol_np, src_np[:, None], tgt_np, len_np[:, None], voxel_shift=sh, eps=eps)["img"].reshape(B, N)
            _record("image", f"{name} fwd_general/bilinear", sc.per_ray_err(_np(out), ref, chk.keep_img), FLOOR["image"])
    # options of the plain walk (ordinary geometries)
    if not c["lattice"] and "planar" not in name:
        for reduce, ac in ((1, 0), (0, 1), (1, 1)):
            kw = dict(reduce="max" if reduce else "sum", align_corners=bool(ac))
            ref, ref32 = (oracle.siddon_fwd(vol_np, src_np[:, None], tgt_np, len_np[:, None], voxel_shift=sh, eps=eps, dtype=dt,
                                            **kw).reshape(B, N) for dt in (np.float64, np.float32))
            out.fill_(float("nan"))
            _call("fwd", *geo, _p(out), B, N, sh, eps, reduce, ac)
            _record("image", f"{name} fwd/r{reduce}a{ac}", sc.per_ray_err(_np(out), ref, chk.keep_img & _resolved(ref32, ref)),
                    FLOOR["image"])
        for label, kw, args in (("max", dict(reduce="max"), (0, 1, 0, 0)), ("ac", dict(align_corners=True), (0, 0, 1, 0)),
                                ("bilinear", dict(mode=1), (0, 0, 0, 1)), ("bilinear/stop", dict(mode=1, stop_grad=True), (1, 0, 0, 1))):
            q64, q32 = _ref(c, g_all_np, **kw)
            got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
            _call("bwd_general", *geo, _p(g_all), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, N, sh,
                  eps, *args)
            ochk = Checker(c, name, q64, q32, None, resolved=True)
            ochk.grads(f"bwd_general/{label}", got, stop=args[0] == 1)
            # sums over rays (g_source, g_volume): gout zeroed on every ray the per-ray comparison leaves out, kernel and oracle rerun
            keep = ochk.keep_end & _resolved(q32["g_raylen"], q64["g_raylen"]) & _resolved(q32["image"], q64["image"])
            g_opt_np = (g_all_np * keep).astype(np.float32)
            o64, o32 = _ref(c, g_opt_np, **kw)
            g_opt = _t(g_opt_np)
            got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
            _call("bwd_general", *geo, _p(g_opt), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, N, sh,
                  eps, *args)
            ochk.sums_vs_oracle(f"bwd_general/{label} (resolved rays)", got, o64, o32, stop=args[0] == 1,
                                gout=None if args[3] == 1 else g_opt_np)
    # stop_grad two-walk backward
    got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
    _call("bwd", *geo, _p(g_all), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, N, sh, eps, 1, 0)
    chk.grads("bwd/stop", got, stop=True)
    assert not got["g_volume"].any()
    # forward with sensitivities, in the caller's order and permuted (the sorted kernels take any order)
    perm = np.random.default_rng(3).permutation(N)
    inv = np.argsort(perm)
    tgt_p, len_p = _t(tgt_np[:, perm]), _t(len_np[:, perm])
    for kname in ("fwd_sens", "fwd_sens_sorted", "fwd_sorted"):
        out.fill_(float("nan"))
        sens = _nan(B, N, 8)
        if kname == "fwd_sens":
            _call(kname, *geo, _p(out), _p(sens), B, N, sh, eps)
        else:
            extra = (_p(sens),) if kname == "fwd_sens_sorted" else ()
            _call(kname, _p(vol), *dims, _p(src), _p(tgt_p), _p(len_p), _p(out), *extra, B, N, sh, eps)
            out = out[:, inv].contiguous()
            sens = sens[:, inv].contiguous()
        chk.image(kname, out)
        if kname == "fwd_sorted":
            continue
        _identities(f"{name} {kname}", c, out, sens)
        chk.sens(kname, sens, g_all_np)
        for stop in (0, 1):
            chk.grads(f"{kname}+bwd_sens/stop{stop}", _bwd_sens(sens, g_all, B, N, stop), stop=bool(stop))
        chk.sums_vs_oracle(f"{kname}+bwd_sens (g_end)", _bwd_sens(sens, g_end, B, N, 0), e64, e32)
    # label mask: a segment's label is its voxel's label, so the channel images are as well conditioned as the image
    if not c["lattice"]:
        C = 3
        ii = np.indices(dims)
        mask_np = ((ii[0] >= dims[0] // 2).astype(np.float32) + (ii[1] >= dims[1] // 3)).astype(np.float32)
        margs = (vol_np, mask_np, src_np[:, None], tgt_np, len_np[:, None])
        ref = oracle.siddon_fwd_mask(*margs, C, voxel_shift=sh, eps=eps, dtype=np.float64)
        mask = _t(mask_np)
        outc = _nan(B, C, N)
        _call("fwd_mask", _p(vol), _p(mask), *dims, _p(src), _p(tgt), _p(raylen), _p(outc), B, N, C, sh, eps)
        keep = np.repeat(chk.keep_img[:, None, :], C, 1).reshape(B * C, N)
        _record("image/mask", f"{name} fwd_mask", sc.per_ray_err(_np(outc).reshape(B * C, N), ref.reshape(B * C, N), keep), 1e-4)
        gm_np = (np.random.default_rng(9).random((B, C, N)) * ~sc.excluded(c["cls"], "g_target")[:, None, :]).astype(np.float32)
        m64 = oracle.siddon_bwd_mask(*margs, gm_np, voxel_shift=sh, eps=eps, dtype=np.float64)
        m32 = oracle.siddon_bwd_mask(*margs, gm_np, voxel_shift=sh, eps=eps, dtype=np.float32)
        got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
        gm = _t(gm_np)
        _call("bwd_mask", _p(vol), _p(mask), *dims, _p(src), _p(tgt), _p(raylen), _p(gm),
              *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, N, C, sh, eps, 0)
        mk = dict(g_target=m64["g_target"], g_raylen=m64["g_raylen"].reshape(B, N), g_volume=m64["g_volume"],
                  g_source=m64["g_source"].reshape(B, 3))
        mk32 = dict(g_target=m32["g_target"], g_raylen=m32["g_raylen"].reshape(B, N), g_volume=m32["g_volume"],
                    g_source=m32["g_source"].reshape(B, 3))
        mchk = Checker(c, name, mk, mk32, None)
        mchk.grads("bwd_mask", got)
        mchk.sums_vs_oracle("bwd_mask", got, mk, mk32)


# ---- full grids, bricks, pose-in --------------------------------------------------------------------------------------------------
GRID_CASES = [n for n, (g, s) in CASES.items() if g not in ("axis", "lattice_rays")]
GRID_IDS = [f"{n}/sens_pose-{_route(n)}" if CASES[n][0] in ("rotated", "inside", "planar", "lattice") else n for n in GRID_CASES]
FWD_GRID = (0, 46, 47, 15, 101, 103, 116, 164)
SENS_GRID = (0, 41, 38, 34, 42, 101, 103, 116)


@pytest.mark.parametrize("name", GRID_CASES, ids=GRID_IDS)
def test_grid_brick_and_pose_in_kernels_vs_oracle(name):
    """fwd_grid / fwd_sens_grid variants, bwd_grid, the mask grids, the brick kernels (ray tensors, pose-in, pixel subset, volume
    gradient) and the pose-in walks, with the route fwd_sens_pose takes named."""
    from oracle import oracle
    c = _case(name)
    vol_np, src_np, tgt_np, len_np, H, W = c["vol"], c["src"], c["tgt"], c["raylen"], c["H"], c["W"]
    dims, (B, N), sh, eps = vol_np.shape, tgt_np.shape[:2], c["shift"], c["eps"]
    g_all_np, g_end_np = _gouts(c)
    r64, r32 = _ref(c, g_all_np, per_ray=True)
    e64, e32 = _ref(c, g_end_np)
    vol, src, tgt, raylen, g_all, g_end = _t(vol_np), _t(src_np), _t(tgt_np), _t(len_np), _t(g_all_np), _t(g_end_np)
    geo = (_p(vol), *dims, _p(src), _p(tgt), _p(raylen))
    # the un-cut sensitivities walk (one slab of 512 planes)
    out, sens0 = _nan(B, N), _nan(B, N, 8)
    _call("fwd_sens_grid", *geo, _p(out), _p(sens0), B, H, W, sh, eps, 34)
    s0 = _np(sens0).astype(np.float64)
    uncut, uncut_src = s0[..., :3] * g_all_np[..., None], s0[..., 4:7] * g_all_np[..., None]
    if c["lattice"]:
        from hostemu import emu
        e = emu.siddon_sens(vol_np, src_np[:, None], tgt_np, len_np[:, None], g_all_np, eps=eps, slab=0)
        _record("uncut vs emulation", f"{name} fwd_sens_grid/34", sc.per_ray_err(uncut, e["g_target"]), 1e-6)
        _record("uncut vs emulation", f"{name} fwd_sens_grid/34 image", sc.per_ray_err(_np(out), e["img"].reshape(B, N)), 1e-6)
        _record("uncut vs emulation", f"{name} fwd_sens_grid/34 source", relerr(uncut_src.sum(1), e["g_source"].reshape(B, 3)), 1e-6)
    chk = Checker(c, name, r64, r32, uncut, uncut_src)
    chk.sens("fwd_sens_grid/34 (un-cut)", sens0, g_all_np)
    chk.sums_vs_oracle("fwd_sens_grid/34+bwd_sens (g_end)", _bwd_sens(sens0, g_end, B, N, 0), e64, e32)
    brick_ok = dims[2] % 4 == 0 and H >= 2 and W >= 2
    for v in FWD_GRID:
        out.fill_(float("nan"))
        _call("fwd_grid", *geo, _p(out), B, H, W, sh, eps, v)
        chk.image(f"fwd_grid/{v}", out)
    for v in SENS_GRID:
        if v == 42 and not brick_ok:
            continue
        out.fill_(float("nan"))
        sens = _nan(B, N, 8)
        _call("fwd_sens_grid", *geo, _p(out), _p(sens), B, H, W, sh, eps, v)
        chk.image(f"fwd_sens_grid/{v}", out)
        _identities(f"{name} fwd_sens_grid/{v}", c, out, sens)
        chk.sens(f"fwd_sens_grid/{v}", sens, g_all_np)
        chk.grads(f"fwd_sens_grid/{v}", _bwd_sens(sens, g_all, B, N, 0))
    for stop in (0, 1):
        got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
        _call("bwd_grid", *geo, _p(g_all), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, H, W, sh, eps,
              stop, 0)
        chk.grads(f"bwd_grid/stop{stop}", got, stop=bool(stop))
    got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=None)
    _call("bwd_grid", *geo, _p(g_end), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, H, W, sh, eps, 0, 0)
    chk.sums_vs_oracle("bwd_grid (g_end)", got, e64, e32)
    if not c["lattice"]:
        C = 3
        ii = np.indices(dims)
        mask_np = ((ii[0] >= dims[0] // 2).astype(np.float32) + (ii[2] >= dims[2] // 3)).astype(np.float32)
        margs = (vol_np, mask_np, src_np[:, None], tgt_np, len_np[:, None])
        ref = oracle.siddon_fwd_mask(*margs, C, voxel_shift=sh, eps=eps, dtype=np.float64)
        mask = _t(mask_np)
        outc = _nan(B, C, N)
        _call("fwd_mask_grid", _p(vol), _p(mask), *dims, _p(src), _p(tgt), _p(raylen), _p(outc), B, H, W, C, sh, eps)
        keep = np.repeat(chk.keep_img[:, None, :], C, 1).reshape(B * C, N)
        _record("image/mask", f"{name} fwd_mask_grid", sc.per_ray_err(_np(outc).reshape(B * C, N), ref.reshape(B * C, N), keep), 1e-4)
        gm_np = (np.random.default_rng(9).random((B, C, N)) * ~sc.excluded(c["cls"], "g_target")[:, None, :]).astype(np.float32)
        m64 = oracle.siddon_bwd_mask(*margs, gm_np, voxel_shift=sh, eps=eps, dtype=np.float64)
        m32 = oracle.siddon_bwd_mask(*margs, gm_np, voxel_shift=sh, eps=eps, dtype=np.float32)
        got = dict(g_source=_nan(B, 3), g_target=_nan(B, N, 3), g_raylen=_nan(B, N), g_volume=torch.zeros(dims, device=DEV))
        gm = _t(gm_np)
        _call("bwd_mask_grid", _p(vol), _p(mask), *dims, _p(src), _p(tgt), _p(raylen), _p(gm),
              *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume")], B, H, W, C, sh, eps, 0)
        mk = dict(g_target=m64["g_target"], g_raylen=m64["g_raylen"].reshape(B, N), g_volume=m64["g_volume"],
                  g_source=m64["g_source"].reshape(B, 3))
        mk32 = dict(g_target=m32["g_target"], g_raylen=m32["g_raylen"].reshape(B, N), g_volume=m32["g_volume"],
                    g_source=m32["g_source"].reshape(B, 3))
        mchk = Checker(c, name, mk, mk32, None)
        mchk.grads("bwd_mask_grid", got)
        mchk.sums_vs_oracle("bwd_mask_grid", got, mk, mk32)
    L, lib = _lib()
    if brick_ok:
        nbytes = int(lib.b200drr_siddon_brick_workspace_bytes(B, H, W))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        out.fill_(float("nan"))
        _call("fwd_brick", *geo, None, None, None, None, _p(out), _p(ws), nbytes, B, H, W, sh, eps, 0)
        chk.image("fwd_brick/rays", out)
        gv = _nan(*dims)
        _call("bwd_vol_brick", _p(g_all), *dims, _p(src), _p(tgt), _p(raylen), None, None, None, None, _p(gv), _p(ws), nbytes, B, H, W,
              sh, eps)
        chk.grads("bwd_vol_brick", dict(g_volume=gv))
        # a random pixel subset, in a random order
        rng = np.random.default_rng(5)
        pix = rng.permutation(N)[: max(N // 3, 2)]
        Ns = len(pix)
        index = np.full(N, -1, np.int32)
        index[pix] = np.arange(Ns, dtype=np.int32)
        corners = tgt_np.reshape(B, H, W, 3)[:, [0, 0, H - 1], [0, W - 1, 0]]
        nb = int(lib.b200drr_siddon_brick_workspace_bytes(B, 1, Ns))
        wss = torch.empty(nb, dtype=torch.uint8, device=DEV)
        outs = _nan(B, Ns)
        # named tensors: a temporary would be freed (and its block reused) before the launch
        tgt_s, len_s, index_t, corners_t = _t(tgt_np[:, pix]), _t(len_np[:, pix]), _t(index, np.int32), _t(corners)
        _call("fwd_brick_subset", _p(vol), *dims, _p(src), _p(tgt_s), _p(len_s), _p(index_t), _p(corners_t), _p(outs), _p(wss), nb, B, H,
              W, Ns, sh, eps, 0)
        _record("image", f"{name} fwd_brick_subset", sc.per_ray_err(_np(outs), r64["image"][:, pix], chk.keep_img[:, pix]),
                1e-5 if c["lattice"] else FLOOR["image"])
    if c["pose"] is None:
        return
    G, Wd, rows, cols = c["pose"]
    t64, l64, p = sc.pose_rays(G, Wd, rows, cols)
    # the pose-in kernels generate their rays in fp32: the reference rays are G p and |Wd p| in fp64.  G p is exact in fp32 for
    # every case here (siddon_cases.pose_matrices / grid_matrices / lattice_ties), so the pose-in rays are the ray tensors above and
    # the un-cut walk on those is their tie reference; the classes are those of the rays G p all the same
    assert (t64 == tgt_np).all()
    q = dict(c, tgt=t64.astype(np.float32), raylen=l64, cls=sc.classify(dims, src_np, t64, sh, eps))
    q64, q32 = _ref(q, g_all_np, per_ray=True)
    pchk = Checker(q, name, q64, q32, uncut, uncut_src)
    Gt, Wt, rt, ct = _t(G), _t(Wd), _t(rows), _t(cols)
    pgeo = (_p(vol), *dims, _p(src), _p(Gt), _p(Wt), _p(rt), _p(ct))
    if brick_ok:
        out.fill_(float("nan"))
        _call("fwd_brick", _p(vol), *dims, _p(src), None, None, _p(Gt), _p(Wt), _p(rt), _p(ct), _p(out), _p(ws), nbytes, B, H, W, sh,
              eps, 0)
        pchk.image("fwd_brick/pose", out)
    out.fill_(float("nan"))
    _call("fwd_pose", *pgeo, _p(out), B, H, W, sh, eps)
    pchk.image("fwd_pose", out)
    ws_t, ws_l = _nan(B, N, 3), _nan(B, N)
    pg = dict(g_source=_nan(B, 3), g_G=_nan(B, 3, 4), g_Wd=_nan(B, 3, 4), g_volume=torch.zeros(dims, device=DEV))
    _call("bwd_pose", *pgeo, _p(g_all), _p(pg["g_source"]), _p(pg["g_G"]), _p(pg["g_Wd"]), _p(pg["g_volume"]), _p(ws_t), _p(ws_l),
          B, H, W, sh, eps, 0)
    pchk.grads("bwd_pose", dict(g_target=ws_t, g_raylen=ws_l, g_volume=pg["g_volume"], g_source=pg["g_source"]))
    _pose_sums(f"{name} bwd_pose", pg, _np(ws_t), _np(ws_l), Wd, p)
    pg = dict(g_source=_nan(B, 3), g_G=_nan(B, 3, 4), g_Wd=_nan(B, 3, 4))
    _call("bwd_pose", *pgeo, _p(g_end), _p(pg["g_source"]), _p(pg["g_G"]), _p(pg["g_Wd"]), None, _p(ws_t), _p(ws_l), B, H, W, sh, eps,
          0)
    pchk.sums_vs_oracle("bwd_pose (g_end)", pg, e64, e32)
    # the pose-in sensitivities walk, on the route the library picks for this shape (asserted from the launched kernel)
    route = _route(name)
    # the brick route is also told by its scratch, which comes from the library's stream-ordered pool (cudaMallocFromPoolAsync):
    # the profiler has been seen to record the runtime calls of that launch but not its kernel
    for _ in range(3):   # the profiler occasionally drops a session's device activity records; the launch is then repeated
        out.fill_(float("nan"))
        sens = _nan(B, N, 8)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            _call("fwd_sens_pose", *pgeo, _p(out), _p(sens), B, H, W, sh, eps)
            torch.cuda.synchronize()
        names = sorted({e.name for e in prof.events()})
        slab = [n for n in names if "siddon_sens_slab_kernel" in n]
        maj = [n for n in slab if ", true" in n or "(bool)1" in n]
        brick = any("siddon_fwd_brick_kernel" in n or n == "cudaMallocFromPoolAsync" for n in names)
        seen = "brick" if brick else "pieces" if maj else "slabs" if slab else None
        if seen is not None:
            break
    print(f"fwd_sens_pose {name}: route {seen}")
    assert seen == route, (route, names)
    pchk.image(f"fwd_sens_pose/{route}", out)
    pchk.sens(f"fwd_sens_pose/{route}", sens, g_all_np)
    s_np = _np(sens)
    pchk.grads(f"fwd_sens_pose/{route}", dict(g_target=torch.as_tensor(s_np[..., :3] * g_all_np[..., None])))
    for stop in (0, 1):
        pg = dict(g_source=_nan(B, 3), g_G=_nan(B, 3, 4), g_Wd=_nan(B, 3, 4))
        _call("bwd_sens_pose", _p(sens), _p(g_all), _p(Wt), _p(rt), _p(ct), _p(pg["g_source"]), _p(pg["g_G"]), _p(pg["g_Wd"]), B, H, W,
              stop)
        pchk.grads(f"bwd_sens_pose/{route}/stop{stop}", dict(g_source=pg["g_source"]))     # against the un-cut walk
        gl = np.zeros((B, N)) if stop else s_np[..., 3] * g_all_np
        _pose_sums(f"{name} bwd_sens_pose/{route}/stop{stop}", pg, uncut, gl, Wd, p)


def _pose_sums(where, got, g_tgt, g_len, Wd, p):
    """g_G = sum_n g_tgt p^T and g_Wd = sum_n g_len (Wd p / |Wd p|) p^T in fp64 from per-ray gradients (the un-cut walk's end-point
    gradients, or bwd_pose's own per-ray workspace); errors over the sum of the magnitudes of the terms."""
    g_tgt, g_len = np.asarray(g_tgt, np.float64), np.asarray(g_len, np.float64)
    dl = np.einsum("bij,nj->bni", np.asarray(Wd, np.float64), p)
    u = dl / np.linalg.norm(dl, axis=-1, keepdims=True)
    terms = dict(g_G=g_tgt[..., :, None] * p[None, :, None, :], g_Wd=(g_len[..., None] * u)[..., :, None] * p[None, :, None, :])
    for k, t in terms.items():
        ref, mag = t.sum(1), np.abs(t).sum(1).max()
        _record(f"pose sum {k}", where, float(np.abs(_np(got[k]) - ref).max() / max(mag, 1e-30)), 1e-5)


def test_every_siddon_entry_point_ran():
    missing = [e for e in ENTRIES if e not in SEEN]
    for what, (ratio, err, bound, where) in sorted(WORST.items()):
        print(f"WORST {what:24s} err {err:.2e} bound {bound:.2e} ({ratio:.2f} of it) at {where}")
    assert not missing, missing
