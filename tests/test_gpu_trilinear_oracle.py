"""Every trilinear device path against the fp64 oracle on the same ray tensors: row-ordered, tiled and packed-corner launches,
slab-major cuts, forward-with-sensitivities, mask_to_channels, the pose-in training step, and the volume gradient, at shapes with
partial tiles, thin volumes, sources inside the volume, misses, axis-parallel rays and heavy scatter contention.

Kernels are called through the C ABI with `slab` / `variant` passed explicitly, so each path is pinned whatever the routing
thresholds are.  Images: max-abs error over the reference's max-abs <= 1e-4.  Gradients: the SURVEY 8c rule (trilinear_cases.tol);
end points and range partials on the smooth volume.  The geometries are checked to be what their names say on the CPU
(test_trilinear_cases_cpu.py)."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import trilinear_cases as tc
from conftest import relerr
from gpu_common import DEV
from test_gpu_production import _setup

pytestmark = pytest.mark.gpu

IMG_TOL = 1e-4
FLOOR = dict(g_volume=1e-4, g_raylen=1e-4, g_target=1e-3, g_source=1e-3, g_alpha=1e-3, g_G=1e-3, g_Wd=1e-3)
GRADS = ("g_volume", "g_raylen", "g_target", "g_source", "g_alpha")
# the trilinear entry points this module must reach (b200drr.h); the final test asserts each ran
ENTRIES = ("b200drr_trilinear_fwd", "b200drr_trilinear_bwd", "b200drr_trilinear_bwd_max", "b200drr_trilinear_fwd_grid",
           "b200drr_trilinear_bwd_grid", "b200drr_pack_corners", "b200drr_trilinear_fwd_packed", "b200drr_trilinear_bwd_packed",
           "b200drr_trilinear_fwd_sens", "b200drr_trilinear_fwd_sens_packed", "b200drr_trilinear_bwd_sens",
           "b200drr_trilinear_alpha_range_pose", "b200drr_trilinear_fwd_sens_pose", "b200drr_trilinear_bwd_sens_pose",
           "b200drr_trilinear_fwd_mask", "b200drr_trilinear_bwd_mask", "b200drr_trilinear_fwd_mask_grid",
           "b200drr_trilinear_bwd_mask_grid")
SEEN = set()
WORST = {}   # quantity -> (largest observed error / its bound, error, bound, where)


@pytest.fixture(autouse=True)
def _entry_points(monkeypatch):
    """Record which trilinear entry points run (the module's own calls included: renderers look them up per call)."""
    from diffdrr_b200 import _lib
    lib = _lib.load()
    for name in _lib.exported_symbols():
        if name.startswith("b200drr_trilinear") or name == "b200drr_pack_corners":
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


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    L, lib = _lib()
    L.check(getattr(lib, name)(*args, _stream()), name)


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32)).to(DEV)


def _record(what, where, err, bound):
    print(f"{what:24s} {where:40s} err {err:.2e} bound {bound:.2e}")
    if what not in WORST or err / bound > WORST[what][0]:
        WORST[what] = (err / bound, err, bound, where)
    assert err <= bound, (what, where, err, bound)


# ---- geometry ---------------------------------------------------------------------------------------------------------------------
SHAPES = {"A": tc.SHAPE_A, "B4": ((256, 256, 256), 200, 200, 4), "B9": ((256, 256, 256), 200, 200, 9),
          "thin": tc.SHAPE_THIN, "sliver": tc.SHAPE_SLIVER, "D": ((32, 32, 32), 128, 128, 16)}


@functools.lru_cache(maxsize=None)
def _case(shape, geom, shift):
    """-> (vol fp32 numpy, src (B, 3), tgt (B, N, 3), raylen (B, N), H, W, kinks (N,) bool or None); all fp32 numpy, smooth volume."""
    dims, H, W, B = SHAPES[shape]
    if geom == "rotated":
        _, _, src, tgt, raylen = _setup(dims, H, B, seed=1, kind="smooth", W=W)
        src, tgt, raylen = (x.cpu().numpy() for x in (src, tgt, raylen))
    elif geom == "axis":
        src, tgt, raylen = tc.axis(dims, H, W, shift)
    else:
        src, tgt, raylen = getattr(tc, geom)(dims, H, W, B, seed=2)
    return tc.volume(dims), src, tgt, raylen, H, W, tc.axis_kinks(H, W) if geom == "axis" else None


def _range(vol, src, tgt, shift, narrow):
    amin, amax = tc.range_of(vol.shape, src, tgt, shift)
    if narrow:   # explicit alphamin / alphamax inside the volume's own range
        amin, amax = amin + 0.3 * (amax - amin), amax - 0.2 * (amax - amin)
    return float(np.float32(amin)), float(np.float32(amax))


def _oracle(vol, src, tgt, raylen, gout, P, amin, amax, shift, want_vol=True, **kw):
    """fp64 and fp32 oracle: (img64, img32, grads64, grads32) with g_alpha = [g_alphamin, g_alphamax]."""
    from oracle import oracle
    args = (vol, src[:, None], tgt, raylen[:, None])
    fkw = dict(n_points=P, alphamin=amin, alphamax=amax, voxel_shift=shift, **kw)
    out = []
    for dt in (np.float64, np.float32):
        out.append(oracle.trilinear_fwd(*args, dtype=dt, **fkw).reshape(len(src), -1))
    for dt in (np.float64, np.float32):
        g = oracle.trilinear_bwd(*args, gout.reshape(len(src), 1, -1), dtype=dt, want_vol=want_vol, **fkw)
        g["g_alpha"] = np.array([g["g_alphamin"], g["g_alphamax"]])
        g["g_source"] = g["g_source"].reshape(len(src), 3)
        g["g_raylen"] = g["g_raylen"].reshape(len(src), -1)
        out.append(g)
    out[3]["g_alpha"] = tc.alpha_partials_f32(vol, src, tgt, raylen, gout, **fkw)
    out[2]["alpha_scale"] = tc.alpha_scale(out[2]["g_raylen"], raylen, amin, amax)
    return out


def _check_img(where, got, ref64):
    _record("image", where, relerr(got.cpu().numpy(), ref64), IMG_TOL)


def _check_grads(where, got, g64, g32, keys):
    for k in keys:
        if got.get(k) is None:
            continue
        x = got[k].cpu().numpy()
        if k == "g_alpha":   # measured against the size of the terms the partials sum (trilinear_cases.alpha_scale)
            s = g64["alpha_scale"]
            _record(k, where, float(np.abs(x - g64[k]).max()) / s, tc.tol(g32[k], g64[k], FLOOR[k], s))
        else:
            _record(k, where, relerr(x, g64[k]), tc.tol(g32[k], g64[k], FLOOR[k]))


def _grads(B, N, dims, vol=True):
    z = dict(g_source=torch.full((B, 3), float("nan"), device=DEV), g_target=torch.full((B, N, 3), float("nan"), device=DEV),
             g_raylen=torch.full((B, N), float("nan"), device=DEV), g_alpha=torch.zeros(2, device=DEV))
    z["g_volume"] = torch.zeros(dims, device=DEV) if vol else None
    return z


# ---- every launch of the same rays -------------------------------------------------------------------------------------------------
CASES = [  # (shape, geometry, n_points, voxel_shift, narrow range)
    ("A", "rotated", 500, 0.5, False), ("A", "rotated", 2, 0.5, False), ("A", "rotated", 77, 0.5, True),
    ("A", "rotated", 77, 0.0, False), ("A", "inside", 77, 0.5, False), ("A", "miss", 77, 0.5, False),
    ("A", "axis", 77, 0.5, True), ("A", "axis", 500, 0.0, True), ("A", "axis", 2, 0.5, True),
    ("B4", "rotated", 200, 0.5, False), ("B9", "rotated", 200, 0.5, False),
    ("thin", "rotated", 77, 0.5, False), ("thin", "axis", 77, 0.5, True),
    ("sliver", "rotated", 77, 0.5, False), ("sliver", "axis", 77, 0.0, True),
    ("D", "near_identical", 77, 0.5, False),
]


@pytest.mark.parametrize("shape,geom,P,shift,narrow", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_every_launch_vs_oracle(shape, geom, P, shift, narrow):
    """Images of fwd, fwd_grid, fwd_packed (slab 0 and two slab heights), fwd_sens (ray set and grid), fwd_sens_packed (slab 0 and
    two heights); gradients of bwd, bwd_grid (with g_vol), bwd_packed (slab 0 and two heights) and the sensitivities + bwd_sens."""
    vol_np, src_np, tgt_np, len_np, H, W, kinks = _case(shape, geom, shift)
    dims = vol_np.shape
    B, N = tgt_np.shape[:2]
    eps = 1e-8
    slabs = (16, 8) if dims[0] >= 16 else (1, 2)
    amin, amax = _range(vol_np, src_np, tgt_np, shift, narrow)
    gfull = np.random.default_rng(7).random((B, N), dtype=np.float32)
    # axis-parallel rays on an integer plane: end points and range partials are one-sided sub-gradients there (trilinear_cases.axis_kinks)
    gend = gfull if kinks is None else gfull * ~kinks[None, :]
    img64, _, g64, g32 = _oracle(vol_np, src_np, tgt_np, len_np, gfull, P, amin, amax, shift)
    # D: the end points of its long, nearly parallel rays are ill-conditioned in the oracle's own fp32 (~2 %), past TOL_CAP; the
    # case is there for the scatter contention of g_volume and the cross-CTA sums of g_source / the range partials
    passes = [("all", gfull, g64, g32, tuple(k for k in GRADS if not (shape == "D" and k == "g_target")))]
    if kinks is not None:   # image, g_volume, g_raylen on every ray; end points and range partials off the kinks
        _, _, e64, e32 = _oracle(vol_np, src_np, tgt_np, len_np, gend, P, amin, amax, shift, want_vol=False)
        passes = [("all", gfull, g64, g32, GRADS[:2]), ("end", gend, e64, e32, GRADS[2:])]
    assert np.abs(img64).max() > 0
    vol, src, tgt, raylen, arange = _t(vol_np), _t(src_np), _t(tgt_np), _t(len_np), _t([amin, amax])
    packed = torch.empty(int(_lib()[1].b200drr_packed_volume_floats(*dims)), device=DEV)
    _call("b200drr_pack_corners", _p(vol), *dims, _p(packed))
    geo = (*dims, _p(src), _p(tgt), _p(raylen))
    where = f"{shape}/{geom}/P{P}/s{shift}" + ("/narrow" if narrow else "")
    # images
    out = torch.empty(B, N, device=DEV)
    for name, args in [("fwd", ("b200drr_trilinear_fwd", _p(vol), *geo, _p(out), B, N, shift, eps, P, _p(arange), 0, 0)),
                       ("fwd_grid", ("b200drr_trilinear_fwd_grid", _p(vol), *geo, _p(out), B, H, W, shift, eps, P, _p(arange), 1))] + [
            (f"fwd_packed/slab{s}", ("b200drr_trilinear_fwd_packed", _p(packed), *geo, _p(out), B, H, W, shift, eps, P, _p(arange), s))
            for s in (0, *slabs)]:
        out.fill_(float("nan"))
        _call(*args)
        _check_img(f"{where} {name}", out, img64)
    # two-walk gradients, for the full and (axis) the kink-free upstream gradient
    for gname, g_np, r64, r32, keys in passes:
        gout = _t(g_np)
        for name in ["bwd", "bwd_grid"] + [f"bwd_packed/slab{s}" for s in (0, *slabs)]:
            got = _grads(B, N, dims, vol=not name.startswith("bwd_packed"))
            gp = [_p(got[k]) for k in ("g_source", "g_target", "g_raylen")]
            if name == "bwd":
                _call("b200drr_trilinear_bwd", _p(vol), *geo, _p(gout), *gp, _p(got["g_volume"]), _p(got["g_alpha"]), B, N, shift, eps, P,
                      _p(arange), 0)
            elif name == "bwd_grid":
                _call("b200drr_trilinear_bwd_grid", _p(vol), *geo, _p(gout), *gp, _p(got["g_volume"]), _p(got["g_alpha"]), B, H, W,
                      shift, eps, P, _p(arange), 1)
            else:
                _call("b200drr_trilinear_bwd_packed", _p(packed), *geo, _p(gout), *gp, _p(got["g_alpha"]), B, H, W, shift, eps, P,
                      _p(arange), int(name.split("slab")[1]))
            _check_grads(f"{where} {name}/{gname}", got, r64, r32, keys)
        # forward with sensitivities + elementwise backward
        for name in ["fwd_sens/rays", "fwd_sens/grid"] + [f"fwd_sens_packed/slab{s}" for s in (0, *slabs)]:
            sens = torch.full((B, N, 12), float("nan"), device=DEV)
            out.fill_(float("nan"))
            if name.startswith("fwd_sens/"):
                h, w = (H, W) if name.endswith("grid") else (0, 0)
                _call("b200drr_trilinear_fwd_sens", _p(vol), *geo, _p(out), _p(sens), B, N, h, w, shift, eps, P, _p(arange), 0)
            else:
                _call("b200drr_trilinear_fwd_sens_packed", _p(packed), *geo, _p(out), _p(sens), B, H, W, shift, eps, P, _p(arange),
                      int(name.split("slab")[1]))
            if gname == "all":
                _check_img(f"{where} {name}", out, img64)
            got = _grads(B, N, dims, vol=False)
            _call("b200drr_trilinear_bwd_sens", _p(sens), _p(gout), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen")],
                  _p(got["g_alpha"]), B, N)
            _check_grads(f"{where} {name}/{gname}", got, r64, r32, keys)


# ---- options of the plain kernels ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", ["rotated", "inside", "axis"])
@pytest.mark.parametrize("opt", ["align_corners", "max"])
def test_row_kernels_align_corners_and_max_vs_oracle(geom, opt):
    """align_corners=True (fwd, bwd, fwd_sens on a ray set) and reducefn="max" (fwd, bwd_max) with the volume gradient."""
    shift, P = 0.5, 77
    vol_np, src_np, tgt_np, len_np, H, W, kinks = _case("A", geom, shift)
    dims = vol_np.shape
    B, N = tgt_np.shape[:2]
    amin, amax = _range(vol_np, src_np, tgt_np, shift, geom == "axis")
    ac, red = (1, 0) if opt == "align_corners" else (0, 1)
    gout_np = np.random.default_rng(8).random((B, N), dtype=np.float32)
    if kinks is not None:
        gout_np = gout_np * ~kinks[None, :]
    kw = dict(align_corners=bool(ac), reduce="max" if red else "sum")
    img64, _, g64, g32 = _oracle(vol_np, src_np, tgt_np, len_np, gout_np, P, amin, amax, shift, **kw)
    vol, src, tgt, raylen, arange, gout = _t(vol_np), _t(src_np), _t(tgt_np), _t(len_np), _t([amin, amax]), _t(gout_np)
    geo = (*dims, _p(src), _p(tgt), _p(raylen))
    where = f"A/{geom}/{opt}"
    out = torch.full((B, N), float("nan"), device=DEV)
    _call("b200drr_trilinear_fwd", _p(vol), *geo, _p(out), B, N, shift, 1e-8, P, _p(arange), red, ac)
    _check_img(f"{where} fwd", out, img64)
    got = _grads(B, N, dims)
    name = "b200drr_trilinear_bwd_max" if red else "b200drr_trilinear_bwd"
    _call(name, _p(vol), *geo, _p(gout), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume", "g_alpha")], B, N,
          0.5, 1e-8, P, _p(arange), ac)
    _check_grads(f"{where} {name[8:]}", got, g64, g32, GRADS)
    if ac:
        sens = torch.empty(B, N, 12, device=DEV)
        _call("b200drr_trilinear_fwd_sens", _p(vol), *geo, _p(out), _p(sens), B, N, 0, 0, shift, 1e-8, P, _p(arange), 1)
        _check_img(f"{where} fwd_sens", out, img64)
        got = _grads(B, N, dims, vol=False)
        _call("b200drr_trilinear_bwd_sens", _p(sens), _p(gout), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_alpha")],
              B, N)
        _check_grads(f"{where} fwd_sens", got, g64, g32, ("g_raylen", "g_target", "g_source", "g_alpha"))


# ---- mask_to_channels --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,geom", [("A", "rotated"), ("A", "inside"), ("thin", "rotated")])
def test_mask_kernels_vs_oracle(shape, geom):
    """fwd_mask / bwd_mask (row order) and fwd_mask_grid / bwd_mask_grid (pixel tiles) with the volume gradient."""
    from oracle import oracle
    shift, P, C = 0.5, 77, 3
    vol_np, src_np, tgt_np, len_np, H, W, _ = _case(shape, geom, shift)
    dims = vol_np.shape
    B, N = tgt_np.shape[:2]
    # two label faces (half-integer planes of pix): few samples land within round-off of one, where the nearest label is a tie
    ii = np.indices(dims)
    mask_np = ((ii[0] >= dims[0] // 2).astype(np.float32) + (ii[1] >= dims[1] // 3)).astype(np.float32)
    amin, amax = _range(vol_np, src_np, tgt_np, shift, False)
    gout_np = np.random.default_rng(9).random((B, C, N), dtype=np.float32)
    args = (vol_np, mask_np, src_np[:, None], tgt_np, len_np[:, None])
    ref = oracle.trilinear_fwd_mask(*args, C, n_points=P, alphamin=amin, alphamax=amax, dtype=np.float64)
    g = [oracle.trilinear_bwd_mask(*args, gout_np, n_points=P, alphamin=amin, alphamax=amax, dtype=dt) for dt in (np.float64, np.float32)]
    for x in g:
        x["g_alpha"] = np.array([x["g_alphamin"], x["g_alphamax"]])
        x["g_source"] = x["g_source"].reshape(B, 3)
        x["g_raylen"] = x["g_raylen"].reshape(B, N)
    g[0]["alpha_scale"] = tc.alpha_scale(g[0]["g_raylen"], len_np, amin, amax)
    g[1]["g_alpha"] = tc.alpha_partials_f32(vol_np, src_np, tgt_np, len_np, gout_np, mask=mask_np, n_points=P, alphamin=amin,
                                            alphamax=amax)
    vol, mask, src, tgt, raylen, arange, gout = (_t(x) for x in (vol_np, mask_np, src_np, tgt_np, len_np, [amin, amax], gout_np))
    geo = (_p(vol), _p(mask), *dims, _p(src), _p(tgt), _p(raylen))
    out = torch.full((B, C, N), float("nan"), device=DEV)
    for name, extent in (("b200drr_trilinear_fwd_mask", (B, N, C)), ("b200drr_trilinear_fwd_mask_grid", (B, H, W, C))):
        out.fill_(float("nan"))
        _call(name, *geo, _p(out), *extent, shift, 1e-8, P, _p(arange), 0)
        # labels are sampled NEAREST: a sample within round-off of a half-integer plane may take the neighbouring label, a jump of
        # the image; allowed on a handful of rays as test_gpu_production allows near-plane rays
        err = np.abs(out.cpu().numpy() - ref) / np.abs(ref).max()
        print(f"{name[8:]} {shape}/{geom}: max {err.max():.2e}, rays over 1e-4: {(err > IMG_TOL).sum()}")
        assert (err > IMG_TOL).sum() <= 5 and err.max() < 1e-3 and float(np.sqrt((err ** 2).mean())) < 1e-5
    for name, extent in (("b200drr_trilinear_bwd_mask", (B, N, C)), ("b200drr_trilinear_bwd_mask_grid", (B, H, W, C))):
        got = _grads(B, N, dims)
        _call(name, *geo, _p(gout), *[_p(got[k]) for k in ("g_source", "g_target", "g_raylen", "g_volume", "g_alpha")], *extent,
              shift, 1e-8, P, _p(arange), 0)
        _check_grads(f"{shape}/{geom} {name[8:]}", got, g[0], g[1], GRADS)


# ---- pose-in training step -----------------------------------------------------------------------------------------------------
def _pose_drr(dtype=torch.float32):
    from diffdrr_b200 import DRR, synthetic
    dims, H, W, _ = tc.SHAPE_A
    return DRR(synthetic.make_subject(tc.volume(dims)), **synthetic.detector_kwargs(H, W), renderer="trilinear").to(DEV).to(dtype)


def _poses(B=3):
    from diffdrr_b200 import synthetic
    rot, xyz = synthetic.make_poses(B, seed=11)   # asymmetric: unique arg-min / arg-max rays of the sampling range
    return rot.to(DEV), xyz.to(DEV)


def test_pose_in_kernels_vs_oracle_on_their_own_rays():
    """alpha_range_pose + fwd_sens_pose (slab 0, 16, 8) + bwd_sens_pose through the C ABI.  The module's rays are rebuilt from the
    same matrices; the image is compared with the oracle on them (up to the few rays that run within round-off of a voxel plane,
    as in test_gpu_production), g_G / g_Wd with the oracle's g_target / g_raylen contracted with the detector coordinates."""
    from diffdrr_b200 import geometry
    from diffdrr_b200.pose import convert
    drr = _pose_drr()
    dims, H, W, B = tc.SHAPE_A
    N, P = H * W, 150
    rot, xyz = _poses(B)
    with torch.no_grad():
        pose = convert(rot, xyz, parameterization="euler_angles", convention="ZXY")
        Q, r, Ainv = drr._pose_constants()
        src, G, Wd = (x.contiguous() for x in geometry.pose_rays(pose.matrix, Q, r, Ainv))
        rows, cols = drr._grid_axes(None)
        p = torch.stack(torch.broadcast_tensors(cols[None, :], rows[:, None], torch.ones(1, 1, device=DEV), torch.ones(1, 1, device=DEV)),
                        -1).reshape(N, 4)
        tgt = torch.einsum("bij,nj->bni", G, p).contiguous()
        dl = torch.einsum("bij,nj->bni", Wd, p)
        raylen = dl.norm(dim=-1).contiguous()
    rng_, arg = torch.empty(2, device=DEV), torch.empty(2, dtype=torch.int64, device=DEV)
    scratch = torch.empty(2, dtype=torch.int64, device=DEV)
    _call("b200drr_trilinear_alpha_range_pose", *dims, _p(src), _p(G), _p(Wd), _p(rows), _p(cols), _p(rng_), _p(arg), _p(scratch), B, H, W,
          0.5, 1e-8)
    src_np, tgt_np, len_np = src.cpu().numpy(), tgt.cpu().numpy(), raylen.cpu().numpy()
    lo, hi = tc.entry_exit(dims, src_np, tgt_np)
    lo, hi = np.clip(lo, 0, None).ravel(), np.clip(hi, None, 1).ravel()
    amin, amax = (float(x) for x in rng_.cpu())
    assert abs(amin - lo.min()) < 2e-6 and abs(amax - hi.max()) < 2e-6
    a = arg.cpu().numpy()
    assert abs(lo[a[0]] - lo.min()) < 2e-6 and abs(hi[a[1]] - hi.max()) < 2e-6
    vol_np = tc.volume(dims)
    gout_np = np.random.default_rng(10).random((B, N), dtype=np.float32)
    img64, _, g64, g32 = _oracle(vol_np, src_np, tgt_np, len_np, gout_np, P, amin, amax, 0.5, want_vol=False)
    pn, dln, Ln = p.double().cpu().numpy(), dl.double().cpu().numpy(), np.linalg.norm(dl.double().cpu().numpy(), axis=-1)
    for g in (g64, g32):   # target = G p, raylen = |Wd p|  =>  g_G = sum g_tgt p^T,  g_Wd = sum g_len (Wd p / L) p^T
        g["g_G"] = np.einsum("bni,nj->bij", g["g_target"].astype(np.float64), pn)
        g["g_Wd"] = np.einsum("bn,bni,nj->bij", g["g_raylen"].astype(np.float64) / Ln, dln, pn)
    packed = drr.renderer._packed_volume(drr.density)
    gout = _t(gout_np)
    for slab in (0, 16, 8):
        out = torch.full((B, N), float("nan"), device=DEV)
        sens = torch.full((B, N, 12), float("nan"), device=DEV)
        _call("b200drr_trilinear_fwd_sens_pose", _p(packed), *dims, _p(src), _p(G), _p(Wd), _p(rows), _p(cols), _p(out), _p(sens), B, H, W,
              0.5, 1e-8, P, _p(rng_), slab)
        err = np.abs(out.cpu().numpy() - img64) / np.abs(img64).max()
        print(f"pose-in image slab {slab}: max {err.max():.2e}, rays over 1e-4: {(err > IMG_TOL).sum()}")
        assert (err > IMG_TOL).sum() <= 5 and err.max() < 1e-3 and float(np.sqrt((err ** 2).mean())) < 1e-5
        got = dict(g_source=torch.empty(B, 3, device=DEV), g_G=torch.empty(B, 3, 4, device=DEV), g_Wd=torch.empty(B, 3, 4, device=DEV),
                   g_alpha=torch.zeros(2, device=DEV))
        _call("b200drr_trilinear_bwd_sens_pose", _p(sens), _p(gout), _p(Wd), _p(rows), _p(cols), _p(got["g_source"]), _p(got["g_G"]),
              _p(got["g_Wd"]), _p(got["g_alpha"]), B, H, W)
        _check_grads(f"pose-in slab{slab}", got, g64, g32, ("g_source", "g_G", "g_Wd", "g_alpha"))


def test_pose_in_module_gradients_vs_the_fp64_module():
    """DRR.forward's pose-in training step (fp32) against the same DRR in torch.float64 (csrc/literal.cu, pinned to the
    reference at 1e-9 by test_gpu_fp64.py): image and the pose gradients."""
    import diffdrr_b200.drr as drr_mod
    rot, xyz = _poses(3)
    w = torch.rand(3, 1, tc.SHAPE_A[1], tc.SHAPE_A[2], device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    res = []
    for dtype in (torch.float32, torch.float64):
        drr = _pose_drr(dtype)
        r, x = rot.to(dtype).clone().requires_grad_(True), xyz.to(dtype).clone().requires_grad_(True)
        if dtype == torch.float32:
            assert drr_mod._TRILINEAR_POSE_IN and drr._pose_in_trilinear_ok(False, dict(n_points=150), (r, x))
        img = drr(r, x, parameterization="euler_angles", convention="ZXY", n_points=150)
        (img * w.to(dtype)).sum().backward()
        res.append((img.detach(), r.grad, x.grad))
    assert "b200drr_trilinear_fwd_sens_pose" in SEEN and "b200drr_trilinear_bwd_sens_pose" in SEEN
    err = ((res[0][0].double() - res[1][0]).abs() / res[1][0].abs().max()).cpu().numpy()
    assert (err > IMG_TOL).sum() <= 5 and err.max() < 1e-3
    for name, a, b in (("pose grad rot", res[0][1], res[1][1]), ("pose grad xyz", res[0][2], res[1][2])):
        _record(name, "A pose-in vs fp64 DRR", relerr(a.cpu().numpy(), b.cpu().numpy()), 2e-3)


# ---- large case: adjoint identity ---------------------------------------------------------------------------------------------
def test_volume_gradient_is_the_adjoint_of_the_forward_at_512():
    """<A v, w> = <v, A^T w> for fwd_grid / bwd_grid's g_vol at 512^3 -> 256^2, two rotated poses (no oracle at this size)."""
    D, H, B, P = 512, 256, 2, 300
    _, vol, src, tgt, raylen = _setup(D, H, B, seed=5, kind="rand")
    amin, amax = tc.range_of((D, D, D), src.cpu().numpy(), tgt.cpu().numpy())
    arange = _t([amin, amax])
    w = torch.rand(B, H * H, device=DEV, generator=torch.Generator(DEV).manual_seed(4))
    out = torch.empty(B, H * H, device=DEV)
    geo = (D, D, D, _p(src), _p(tgt), _p(raylen))
    _call("b200drr_trilinear_fwd_grid", _p(vol), *geo, _p(out), B, H, H, 0.5, 1e-8, P, _p(arange), 1)
    g_vol = torch.zeros_like(vol)
    _call("b200drr_trilinear_bwd_grid", _p(vol), *geo, _p(w), None, None, None, _p(g_vol), None, B, H, H, 0.5, 1e-8, P, _p(arange), 1)
    lhs = float((out.double() * w.double()).sum())
    rhs = float((vol.double() * g_vol.double()).sum())
    _record("adjoint <Av,w>", "512^3 bwd_grid", abs(lhs - rhs) / abs(lhs), 1e-4)


def test_every_trilinear_entry_point_ran():
    missing = [e for e in ENTRIES if e not in SEEN]
    for what, (ratio, err, bound, where) in sorted(WORST.items()):
        print(f"WORST {what:20s} err {err:.2e} bound {bound:.2e} ({ratio:.2f} of it) at {where}")
    assert not missing, missing
