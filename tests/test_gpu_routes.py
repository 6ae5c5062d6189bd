"""Which C entry points each renderer call launches, with which arguments.

Every `b200drr_*` launch of a renderer call is recorded through a proxy of the ctypes handle: the entry point's name, its
integer and float arguments by value, and its pointer arguments as null (`0`) or non-null (`p`).  The matrix below reaches
every forward and backward branch of the renderers' autograd functions and of `DRR.jacobian`; EXPECTED is the trace the
library produced when this file was written, so a change to the routing -- a kernel swapped, an argument or a threshold
moved, a buffer that became null -- shows up as a diff of one case.  Raised errors are part of the trace."""
import ctypes
import itertools

import pytest
import torch

from gpu_common import DEV

pytestmark = pytest.mark.gpu

_SKIP = ("_workspace_bytes", "_packed_volume_floats", "b200drr_error_string")


def _arg(a):
    if a is None:
        return "0"
    if isinstance(a, ctypes.c_void_p):
        return "0" if a.value is None else "p"
    if isinstance(a, float):
        return repr(a)
    return str(int(a))


class _Recorder:
    """Transparent stand-in for the ctypes library handle that logs every launch."""

    def __init__(self, lib):
        self._real = lib
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith("b200drr_") or name.endswith(_SKIP):
            return fn

        def launch(*args):
            self.calls.append(f"{name[len('b200drr_'):]}({','.join(_arg(a) for a in args)})")
            return fn(*args)

        launch.__name__ = name
        return launch


@pytest.fixture
def recorder(monkeypatch):
    from diffdrr_b200 import _lib, renderers

    rec = _Recorder(_lib.load())
    monkeypatch.setattr(_lib, "_lib", rec)
    monkeypatch.setattr(renderers, "_FUSED_SENSITIVITIES", True)
    monkeypatch.setattr(renderers, "_PACKED_SLAB_SENS", renderers._PACKED_SLAB_SENS)
    yield rec


DIMS = (40, 48, 56)   # D2 % 8 == 0: 16-byte rows for the brick kernel's TMA map with fp32 and 16-bit voxels
_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "f64": torch.float64}
_GRADS = ("none", "rays", "vol", "both")


def _case(kind, dtype="f32", rays="grid", grads="none", **opt):
    opt = dict(sorted(opt.items()))
    cid = "-".join([kind, dtype, rays, grads] + [f"{k}={v}" for k, v in opt.items()])
    return cid, dict(kind=kind, dtype=dtype, rays=rays, grads=grads, **opt)


def _cases():
    out = []
    add = lambda *a, **k: out.append(_case(*a, **k))  # noqa: E731
    ray_sets = ("grid", "small", "large", "subset")
    # ---- Siddon on ray tensors
    for dt, rays, grads, brick in itertools.product(("f32", "f16", "bf16"), ray_sets, _GRADS, (0, 1)):
        if dt != "f32" and grads in ("vol", "both") and brick:
            continue
        add("siddon", dt, rays, grads, brick=brick)
    for rays, grads in itertools.product(ray_sets, _GRADS):
        add("siddon", "f64", rays, grads, brick=1)
        add("siddon", "f32", rays, grads, brick=1, mode="bilinear")
    for opt in (dict(reduce="max"), dict(reduce="callable"), dict(align=1), dict(mask=1), dict(stop=1), dict(fused=0)):
        for rays, grads in itertools.product(("grid", "small", "large"), _GRADS):
            add("siddon", "f32", rays, grads, brick=1, **opt)
    for opt in (dict(reduce="max"), dict(reduce="callable"), dict(align=1), dict(stop=1), dict(mode="bilinear"),
                dict(mask=1)):
        for grads in _GRADS:
            add("siddon", "f64", "grid", grads, brick=1, **opt)
    for grads in _GRADS:
        add("siddon", "f32", "grid", grads, brick=1, mode="bilinear", reduce="max")
        add("siddon", "f32", "grid", grads, brick=1, mode="bilinear", align=1)
        add("siddon", "f16", "grid", grads, fused=0)
    # ---- Trilinear on ray tensors
    for dt, rays, grads, pack in itertools.product(("f32", "f16", "bf16", "f64"), ("grid", "small", "large"), _GRADS,
                                                    (0, 1)):
        add("trilinear", dt, rays, grads, pack=pack)
    for opt in (dict(reduce="max"), dict(reduce="callable"), dict(align=1), dict(mask=1), dict(fused=0)):
        for rays, grads in itertools.product(("grid", "small"), _GRADS):
            add("trilinear", "f32", rays, grads, pack=1, **opt)
            add("trilinear", "f64", rays, grads, pack=1, **opt)
    for grads in _GRADS:
        add("trilinear", "f16", "grid", grads, pack=1, fused=0)
    # ---- pose-in rendering through the DRR module
    for dt, grads, fused, brick in itertools.product(("f32", "f16"), _GRADS, (1, 0), (0, 1)):
        add("siddon_pose", dt, "pose", grads, fused=fused, brick=brick, B=2)
    for grads in _GRADS:
        add("siddon_pose", "f32", "pose", grads, stop=1, brick=1, B=2)
        add("siddon_pose", "f32", "pose", grads, brick=1, B=1)
    for dt, grads, B in itertools.product(("f32", "f16", "bf16"), _GRADS, (2, 8)):
        add("trilinear_pose", dt, "pose", grads, B=B)
    for grads in ("rays", "both"):
        add("trilinear_pose", "f32", "pose", grads, B=8, slab=16)
        add("trilinear_pose", "f32", "pose", grads, B=2, fused=0)
    # ---- DRR.jacobian
    for dt, B in itertools.product(("f32", "f16", "bf16"), (1, 2, 8)):
        add("siddon_jac", dt, "pose", "none", B=B)
        add("trilinear_jac", dt, "pose", "none", B=B)
    add("siddon_jac", "f32", "pose", "none", B=2, stop=1)
    return out


CASES = _cases()


def _volume():
    from diffdrr_b200 import synthetic

    return torch.as_tensor(synthetic.make_volume(DIMS, "smooth", seed=3)).to(DEV)


def _drr(renderer, H, B=2, p_subsample=None, **kw):
    from diffdrr_b200 import DRR, synthetic

    torch.manual_seed(0)
    vol = synthetic.make_volume(DIMS, "smooth", seed=3)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer=renderer, p_subsample=p_subsample,
              **kw).to(DEV)
    rot, xyz = synthetic.make_poses(B, seed=1)
    return drr, rot.to(DEV), xyz.to(DEV)


def _rays(renderer, rays):
    """Voxel-space rays (src (B,1,3), tgt (B,N,3), ray lengths (B,1,N)), the detector_shape hint and the ray_subset hint."""
    from diffdrr_b200.pose import convert

    H = {"grid": 16, "small": 16, "large": 40, "subset": 48}[rays]
    drr, rot, xyz = _drr(renderer, H, p_subsample=0.25 if rays == "subset" else None)
    pose = convert(rot, xyz, parameterization="euler_angles", convention="ZXY")
    with torch.no_grad():
        src, tgt = drr.detector(pose, None)
        img = (tgt - src).norm(dim=-1).unsqueeze(1)
        hint = None
        if rays == "subset":
            det = drr.detector
            hint = (det.pixel_index(), drr.affine_inverse(det.corner_targets(pose, None)), det.height, det.width,
                    len(det.subsamples[-1]))
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
    if rays == "small":
        tgt, img = tgt[:, ::3].contiguous(), img[..., ::3].contiguous()
    return src, tgt, img, ((H, H) if rays == "grid" else None), hint


def _labels(vol):
    return (vol > 0.3).float() + (vol > 0.6).float()


def _ray_call(c, rec):
    """Render through a Siddon / Trilinear module on ray tensors; returns the output and the leaves that want gradients."""
    from callable_reducers import ramp_weighted

    from diffdrr_b200 import Siddon, Trilinear

    dtype = _DT[c["dtype"]]
    ray_dtype = torch.float64 if dtype == torch.float64 else torch.float32
    src, tgt, img, shape, hint = _rays(c["kind"], c["rays"])
    src, tgt, img = src.to(ray_dtype), tgt.to(ray_dtype), img.to(ray_dtype)
    vol32 = _volume()
    vol = vol32.to(dtype)
    reducefn = {"sum": "sum", "max": "max", "callable": ramp_weighted}[c.get("reduce", "sum")]
    want_rays, want_vol = c["grads"] in ("rays", "both"), c["grads"] in ("vol", "both")
    leaves = []
    if want_vol:
        vol.requires_grad_(True)
        leaves.append(vol)
    if want_rays:
        src, tgt, img = (x.clone().requires_grad_(True) for x in (src, tgt, img))
        leaves += [src, tgt, img]
    kw = dict(align_corners=bool(c.get("align", 0)), mask=_labels(vol32) if c.get("mask") else None)
    rec.calls.clear()
    if c["kind"] == "siddon":
        r = Siddon(mode=c.get("mode", "nearest"), reducefn=reducefn,
                   stop_gradients_through_grid_sample=bool(c.get("stop", 0)))
        r.detector_shape, r.ray_subset = shape, hint
        out = r(vol, src, tgt, img, **kw)
    else:
        r = Trilinear(reducefn=reducefn)
        r.detector_shape, r.pack_corners = shape, bool(c.get("pack", 1))
        out = r(vol, src, tgt, img, n_points=40, **kw)
    return out, leaves


def _module(c):
    renderer = c["kind"].split("_")[0]
    kw = dict(stop_gradients_through_grid_sample=True) if c.get("stop") else {}
    return _drr(renderer, 16, B=c["B"], **kw)


def _pose_call(c, rec):
    drr, rot, xyz = _module(c)
    if c["dtype"] != "f32":
        drr.density = drr.density.to(_DT[c["dtype"]])
    leaves = []
    if c["grads"] in ("vol", "both"):
        drr.density = drr.density.detach().clone().requires_grad_(True)
        leaves.append(drr.density)
    if c["grads"] in ("rays", "both"):
        rot, xyz = rot.requires_grad_(True), xyz.requires_grad_(True)
        leaves += [rot, xyz]
    kw = dict(n_points=40) if c["kind"] == "trilinear_pose" else {}
    rec.calls.clear()
    return drr(rot, xyz, parameterization="euler_angles", convention="ZXY", **kw), leaves


def _jacobian_call(c, rec):
    drr, rot, xyz = _module(c)
    if c["dtype"] != "f32":
        drr.density = drr.density.to(_DT[c["dtype"]])
    kw = dict(n_points=40) if c["kind"] == "trilinear_jac" else {}
    rec.calls.clear()
    drr.jacobian(rot, xyz, parameterization="euler_angles", convention="ZXY", **kw)


def run_case(c, rec, monkeypatch):
    """The trace of one case: every launch of its forward and backward, then the error it raised, if any."""
    from diffdrr_b200 import renderers

    if c.get("brick"):
        monkeypatch.setattr(renderers, "_BRICK_MIN_BRICKS", 1)
        monkeypatch.setattr(renderers, "_BRICK_FULL_GRID_MIN_LOAD", 0.0)
    else:
        monkeypatch.setattr(renderers, "_BRICK_MIN_BRICKS", 10 ** 9)
    monkeypatch.setattr(renderers, "_FUSED_SENSITIVITIES", bool(c.get("fused", 1)))
    monkeypatch.setattr(renderers, "_PACKED_SLAB_SENS", c.get("slab", 0))
    renderers._brick_ws.clear()
    try:
        if c["kind"].endswith("_jac"):
            _jacobian_call(c, rec)
        else:
            out, leaves = (_pose_call if c["kind"].endswith("_pose") else _ray_call)(c, rec)
            if leaves:
                out.float().sum().backward()
    except (NotImplementedError, ValueError) as e:
        rec.calls.append(f"raise {type(e).__name__}: {e}")
    torch.cuda.synchronize()
    return list(rec.calls)


@pytest.mark.parametrize("case", [c for _, c in CASES], ids=[i for i, _ in CASES])
def test_route(case, recorder, monkeypatch):
    cid = _case(**case)[0]
    assert run_case(case, recorder, monkeypatch) == EXPECTED[cid]


def test_every_case_is_recorded():
    assert sorted(EXPECTED) == sorted(i for i, _ in CASES)


EXPECTED = {
    "siddon-f32-grid-none-brick=0": [
        "siddon_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-none-brick=1": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-rays-brick=0": [
        "siddon_fwd_sens_grid(p,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,256,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1": [
        "siddon_fwd_sens_grid(p,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,256,0,0)",
    ],
    "siddon-f32-grid-vol-brick=0": [
        "siddon_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,p,2,16,16,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-vol-brick=1": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0)",
    ],
    "siddon-f32-grid-both-brick=0": [
        "siddon_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-both-brick=1": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,0,2,16,16,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-none-brick=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-none-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-rays-brick=0": [
        "siddon_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,86,0,0)",
    ],
    "siddon-f32-small-rays-brick=1": [
        "siddon_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,86,0,0)",
    ],
    "siddon-f32-small-vol-brick=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-vol-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-both-brick=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-both-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-none-brick=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-f32-large-none-brick=1": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-f32-large-rays-brick=0": [
        "siddon_fwd_sens_sorted(p,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,1600,0,0)",
    ],
    "siddon-f32-large-rays-brick=1": [
        "siddon_fwd_sens_sorted(p,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,1600,0,0)",
    ],
    "siddon-f32-large-vol-brick=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-vol-brick=1": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-both-brick=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-both-brick=1": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-none-brick=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-none-brick=1": [
        "siddon_fwd_brick_subset(p,40,48,56,p,p,p,p,p,p,p,23552,2,48,48,576,0.5,1e-08,0,0)",
    ],
    "siddon-f32-subset-rays-brick=0": [
        "siddon_fwd_sens(p,40,48,56,p,p,p,p,p,2,576,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,576,0,0)",
    ],
    "siddon-f32-subset-rays-brick=1": [
        "siddon_fwd_sens(p,40,48,56,p,p,p,p,p,2,576,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,576,0,0)",
    ],
    "siddon-f32-subset-vol-brick=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-vol-brick=1": [
        "siddon_fwd_brick_subset(p,40,48,56,p,p,p,p,p,p,p,23552,2,48,48,576,0.5,1e-08,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-both-brick=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-both-brick=1": [
        "siddon_fwd_brick_subset(p,40,48,56,p,p,p,p,p,p,p,23552,2,48,48,576,0.5,1e-08,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f16-grid-none-brick=0": [
        "siddon_fwd_grid_v16(p,1,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f16-grid-none-brick=1": [
        "siddon_fwd_brick_v16(p,1,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f16-grid-rays-brick=0": [
        "siddon_fwd_sens_grid_v16(p,1,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,256,0,0)",
    ],
    "siddon-f16-grid-rays-brick=1": [
        "siddon_fwd_sens_grid_v16(p,1,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,256,0,0)",
    ],
    "siddon-f16-grid-vol-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-grid-both-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-small-none-brick=0": [
        "siddon_fwd_v16(p,1,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f16-small-none-brick=1": [
        "siddon_fwd_v16(p,1,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f16-small-rays-brick=0": [
        "siddon_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,86,0,0)",
    ],
    "siddon-f16-small-rays-brick=1": [
        "siddon_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,86,0,0)",
    ],
    "siddon-f16-small-vol-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-small-both-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-large-none-brick=0": [
        "siddon_fwd_sorted_v16(p,1,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-f16-large-none-brick=1": [
        "siddon_fwd_sorted_v16(p,1,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-f16-large-rays-brick=0": [
        "siddon_fwd_sens_sorted_v16(p,1,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,1600,0,0)",
    ],
    "siddon-f16-large-rays-brick=1": [
        "siddon_fwd_sens_sorted_v16(p,1,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,1600,0,0)",
    ],
    "siddon-f16-large-vol-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-large-both-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-subset-none-brick=0": [
        "siddon_fwd_v16(p,1,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f16-subset-none-brick=1": [
        "siddon_fwd_brick_subset_v16(p,1,40,48,56,p,p,p,p,p,p,p,23552,2,48,48,576,0.5,1e-08,0,0)",
    ],
    "siddon-f16-subset-rays-brick=0": [
        "siddon_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,576,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,576,0,0)",
    ],
    "siddon-f16-subset-rays-brick=1": [
        "siddon_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,576,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,576,0,0)",
    ],
    "siddon-f16-subset-vol-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f16-subset-both-brick=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-grid-none-brick=0": [
        "siddon_fwd_grid_v16(p,2,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-bf16-grid-none-brick=1": [
        "siddon_fwd_brick_v16(p,2,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-bf16-grid-rays-brick=0": [
        "siddon_fwd_sens_grid_v16(p,2,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,256,0,0)",
    ],
    "siddon-bf16-grid-rays-brick=1": [
        "siddon_fwd_sens_grid_v16(p,2,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,256,0,0)",
    ],
    "siddon-bf16-grid-vol-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-grid-both-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-small-none-brick=0": [
        "siddon_fwd_v16(p,2,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-bf16-small-none-brick=1": [
        "siddon_fwd_v16(p,2,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-bf16-small-rays-brick=0": [
        "siddon_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,86,0,0)",
    ],
    "siddon-bf16-small-rays-brick=1": [
        "siddon_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,86,0,0)",
    ],
    "siddon-bf16-small-vol-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-small-both-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-large-none-brick=0": [
        "siddon_fwd_sorted_v16(p,2,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-bf16-large-none-brick=1": [
        "siddon_fwd_sorted_v16(p,2,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-bf16-large-rays-brick=0": [
        "siddon_fwd_sens_sorted_v16(p,2,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,1600,0,0)",
    ],
    "siddon-bf16-large-rays-brick=1": [
        "siddon_fwd_sens_sorted_v16(p,2,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,1600,0,0)",
    ],
    "siddon-bf16-large-vol-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-large-both-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-subset-none-brick=0": [
        "siddon_fwd_v16(p,2,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-bf16-subset-none-brick=1": [
        "siddon_fwd_brick_subset_v16(p,2,40,48,56,p,p,p,p,p,p,p,23552,2,48,48,576,0.5,1e-08,0,0)",
    ],
    "siddon-bf16-subset-rays-brick=0": [
        "siddon_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,576,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,576,0,0)",
    ],
    "siddon-bf16-subset-rays-brick=1": [
        "siddon_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,576,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,p,2,576,0,0)",
    ],
    "siddon-bf16-subset-vol-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-bf16-subset-both-brick=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f64-grid-none-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-none-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,1,0)",
    ],
    "siddon-f64-grid-rays-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-grid-vol-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,2,256,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-vol-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,256,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-grid-both-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-both-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-small-none-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-none-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,1,0)",
    ],
    "siddon-f64-small-rays-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-rays-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,86,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-small-vol-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-vol-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-small-both-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-both-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-large-none-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-none-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,1,0)",
    ],
    "siddon-f64-large-rays-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-rays-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,1600,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-large-vol-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-vol-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-large-both-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-both-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-subset-none-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-none-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,1,0)",
    ],
    "siddon-f64-subset-rays-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-rays-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,576,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-subset-vol-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-vol-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,576,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f64-subset-both-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,2,576,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-subset-both-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,576,0.5,1e-08,0,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,576,0.5,1e-08,0,0,0,1,0)",
    ],
    "siddon-f32-grid-none-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-grid-vol-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,256,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-grid-both-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-small-none-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,1,0,0)",
    ],
    "siddon-f32-small-rays-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,86,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-small-vol-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-small-both-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-large-none-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,1,0,0)",
    ],
    "siddon-f32-large-rays-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,1600,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-large-vol-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-large-both-brick=1-reduce=max": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,1,0,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,1,0,0,0)",
    ],
    "siddon-f32-grid-none-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,p,p,p,0,0,2,256,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-grid-vol-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-grid-both-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-small-none-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0,0)",
    ],
    "siddon-f32-small-rays-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,p,p,p,0,0,2,86,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-small-vol-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-small-both-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,p,p,p,p,0,2,86,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-large-none-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0,0)",
    ],
    "siddon-f32-large-rays-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,p,p,p,0,0,2,1600,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-large-vol-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,0,0,0,p,0,2,1600,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-large-both-brick=1-reduce=callable": [
        "segments_fwd(0,0,p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,0,p,40,48,56,p,p,p,p,p,p,p,p,0,2,1600,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f32-grid-none-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
    ],
    "siddon-f32-grid-rays-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-grid-vol-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,256,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-grid-both-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-small-none-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,1,0)",
    ],
    "siddon-f32-small-rays-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,86,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-small-vol-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-small-both-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-large-none-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,1,0)",
    ],
    "siddon-f32-large-rays-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,1600,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-large-vol-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-large-both-align=1-brick=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,0,1,0,0)",
    ],
    "siddon-f32-grid-none-brick=1-mask=1": [
        "siddon_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,0)",
    ],
    "siddon-f32-grid-rays-brick=1-mask=1": [
        "siddon_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,0)",
        "siddon_bwd_mask_grid(p,p,40,48,56,p,p,p,p,p,p,p,0,2,16,16,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-vol-brick=1-mask=1": [
        "siddon_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,0)",
        "siddon_bwd_mask_grid(p,p,40,48,56,p,p,p,p,0,0,0,p,2,16,16,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-both-brick=1-mask=1": [
        "siddon_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,0)",
        "siddon_bwd_mask_grid(p,p,40,48,56,p,p,p,p,p,p,p,p,2,16,16,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-small-none-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,0)",
    ],
    "siddon-f32-small-rays-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,0)",
        "siddon_bwd_mask(p,p,40,48,56,p,p,p,p,p,p,p,0,2,86,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-small-vol-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,0)",
        "siddon_bwd_mask(p,p,40,48,56,p,p,p,p,0,0,0,p,2,86,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-small-both-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,0)",
        "siddon_bwd_mask(p,p,40,48,56,p,p,p,p,p,p,p,p,2,86,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-large-none-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,1600,3,0.5,1e-08,0)",
    ],
    "siddon-f32-large-rays-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,1600,3,0.5,1e-08,0)",
        "siddon_bwd_mask(p,p,40,48,56,p,p,p,p,p,p,p,0,2,1600,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-large-vol-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,1600,3,0.5,1e-08,0)",
        "siddon_bwd_mask(p,p,40,48,56,p,p,p,p,0,0,0,p,2,1600,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-large-both-brick=1-mask=1": [
        "siddon_fwd_mask(p,p,40,48,56,p,p,p,p,2,1600,3,0.5,1e-08,0)",
        "siddon_bwd_mask(p,p,40,48,56,p,p,p,p,p,p,p,p,2,1600,3,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-none-brick=1-stop=1": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1-stop=1": [
        "siddon_fwd_sens_grid(p,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,0,2,256,1,0)",
    ],
    "siddon-f32-grid-vol-brick=1-stop=1": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,0,2,16,16,0.5,1e-08,1,0,0)",
    ],
    "siddon-f32-grid-both-brick=1-stop=1": [
        "siddon_fwd_sens_grid(p,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_sens(p,p,p,p,0,2,256,1,0)",
    ],
    "siddon-f32-small-none-brick=1-stop=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-rays-brick=1-stop=1": [
        "siddon_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,0,2,86,1,0)",
    ],
    "siddon-f32-small-vol-brick=1-stop=1": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,0,2,86,0.5,1e-08,1,0,0)",
    ],
    "siddon-f32-small-both-brick=1-stop=1": [
        "siddon_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,0,2,86,1,0)",
    ],
    "siddon-f32-large-none-brick=1-stop=1": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-f32-large-rays-brick=1-stop=1": [
        "siddon_fwd_sens_sorted(p,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,0,2,1600,1,0)",
    ],
    "siddon-f32-large-vol-brick=1-stop=1": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,0,2,1600,0.5,1e-08,1,0,0)",
    ],
    "siddon-f32-large-both-brick=1-stop=1": [
        "siddon_fwd_sens_sorted(p,40,48,56,p,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd_sens(p,p,p,p,0,2,1600,1,0)",
    ],
    "siddon-f32-grid-none-brick=1-fused=0": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1-fused=0": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,0,2,16,16,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-grid-vol-brick=1-fused=0": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0)",
    ],
    "siddon-f32-grid-both-brick=1-fused=0": [
        "siddon_fwd_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,p,p,0,0,0,0,p,p,10752,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,0,2,16,16,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-none-brick=1-fused=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-rays-brick=1-fused=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,0,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-vol-brick=1-fused=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-small-both-brick=1-fused=0": [
        "siddon_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-none-brick=1-fused=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
    ],
    "siddon-f32-large-rays-brick=1-fused=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,0,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-vol-brick=1-fused=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,0,0,0,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f32-large-both-brick=1-fused=0": [
        "siddon_fwd_sorted(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,0)",
        "siddon_bwd(p,40,48,56,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,0,0,0)",
    ],
    "siddon-f64-grid-none-brick=1-reduce=max": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
    ],
    "siddon-f64-grid-rays-brick=1-reduce=max": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
        "raise NotImplementedError: fp64 Siddon: backward is implemented for reducefn='sum'",
    ],
    "siddon-f64-grid-vol-brick=1-reduce=max": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
        "raise NotImplementedError: fp64 Siddon: backward is implemented for reducefn='sum'",
    ],
    "siddon-f64-grid-both-brick=1-reduce=max": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,0)",
        "raise NotImplementedError: fp64 Siddon: backward is implemented for reducefn='sum'",
    ],
    "siddon-f64-grid-none-brick=1-reduce=callable": [
        "segments_fwd(0,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
    ],
    "siddon-f64-grid-rays-brick=1-reduce=callable": [
        "segments_fwd(0,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,1,p,40,48,56,p,p,p,p,p,p,p,0,0,2,256,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f64-grid-vol-brick=1-reduce=callable": [
        "segments_fwd(0,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,1,p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f64-grid-both-brick=1-reduce=callable": [
        "segments_fwd(0,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0,0)",
        "segments_bwd(0,1,p,40,48,56,p,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,0,0,0,0)",
    ],
    "siddon-f64-grid-none-align=1-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
    ],
    "siddon-f64-grid-rays-align=1-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,1,0)",
    ],
    "siddon-f64-grid-vol-align=1-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,2,256,0.5,1e-08,0,1,0)",
    ],
    "siddon-f64-grid-both-align=1-brick=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,0,1,0)",
    ],
    "siddon-f64-grid-none-brick=1-stop=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
    ],
    "siddon-f64-grid-rays-brick=1-stop=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,0,0,2,256,0.5,1e-08,1,0,0)",
    ],
    "siddon-f64-grid-vol-brick=1-stop=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,0,2,256,0.5,1e-08,1,0,0)",
    ],
    "siddon-f64-grid-both-brick=1-stop=1": [
        "siddon_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,0,0)",
        "siddon_bwd_f64(p,40,48,56,p,p,p,p,p,p,0,0,2,256,0.5,1e-08,1,0,0)",
    ],
    "siddon-f64-grid-none-brick=1-mode=bilinear": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-rays-brick=1-mode=bilinear": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-vol-brick=1-mode=bilinear": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-both-brick=1-mode=bilinear": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-none-brick=1-mask=1": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-rays-brick=1-mask=1": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-vol-brick=1-mask=1": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f64-grid-both-brick=1-mask=1": [
        "raise NotImplementedError: fp64 Siddon is implemented for mode='nearest' without mask_to_channels",
    ],
    "siddon-f32-grid-none-brick=1-mode=bilinear-reduce=max": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,1,0)",
    ],
    "siddon-f32-grid-none-align=1-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,1,0)",
    ],
    "siddon-f16-grid-none-fused=0": [
        "siddon_fwd_grid_v16(p,1,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon-f32-grid-rays-brick=1-mode=bilinear-reduce=max": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,1,0)",
        "raise NotImplementedError: backward through Siddon(mode='bilinear', reducefn='max') is not implemented",
    ],
    "siddon-f32-grid-rays-align=1-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,0,2,256,0.5,1e-08,0,0,1,1,0)",
    ],
    "siddon-f16-grid-rays-fused=0": [
        "raise NotImplementedError: ray gradients from a torch.float16 volume come from the fused sensitivities walk only",
    ],
    "siddon-f32-grid-vol-brick=1-mode=bilinear-reduce=max": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,1,0)",
        "raise NotImplementedError: backward through Siddon(mode='bilinear', reducefn='max') is not implemented",
    ],
    "siddon-f32-grid-vol-align=1-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,0,0,0,p,2,256,0.5,1e-08,0,0,1,1,0)",
    ],
    "siddon-f16-grid-vol-fused=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon-f32-grid-both-brick=1-mode=bilinear-reduce=max": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,1,0,1,0)",
        "raise NotImplementedError: backward through Siddon(mode='bilinear', reducefn='max') is not implemented",
    ],
    "siddon-f32-grid-both-align=1-brick=1-mode=bilinear": [
        "siddon_fwd_general(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,0,1,1,0)",
        "siddon_bwd_general(p,40,48,56,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,0,0,1,1,0)",
    ],
    "siddon-f16-grid-both-fused=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f32-grid-none-pack=0": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-none-pack=1": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_packed(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-grid-rays-pack=0": [
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,256,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-f32-grid-rays-pack=1": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_sens_packed(p,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-f32-grid-vol-pack=0": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,p,0,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-vol-pack=1": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,p,0,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-both-pack=0": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-both-pack=1": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-small-none-pack=0": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-small-none-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-small-rays-pack=0": [
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-f32-small-rays-pack=1": [
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-f32-small-vol-pack=0": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-vol-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-both-pack=0": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-both-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-large-none-pack=0": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-large-none-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-large-rays-pack=0": [
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,1600,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,1600,0)",
    ],
    "trilinear-f32-large-rays-pack=1": [
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,1600,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,1600,0)",
    ],
    "trilinear-f32-large-vol-pack=0": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-large-vol-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-large-both-pack=0": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-large-both-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f16-grid-none-pack=0": [
        "trilinear_fwd_grid_v16(p,1,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f16-grid-none-pack=1": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,1,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f16-grid-rays-pack=0": [
        "trilinear_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,256,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-f16-grid-rays-pack=1": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "trilinear_fwd_sens_packed_v16(p,1,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-f16-grid-vol-pack=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-grid-vol-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-grid-both-pack=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-grid-both-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-small-none-pack=0": [
        "trilinear_fwd_v16(p,1,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f16-small-none-pack=1": [
        "trilinear_fwd_v16(p,1,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f16-small-rays-pack=0": [
        "trilinear_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-f16-small-rays-pack=1": [
        "trilinear_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-f16-small-vol-pack=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-small-vol-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-small-both-pack=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-small-both-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-large-none-pack=0": [
        "trilinear_fwd_v16(p,1,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f16-large-none-pack=1": [
        "trilinear_fwd_v16(p,1,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f16-large-rays-pack=0": [
        "trilinear_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,1600,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,1600,0)",
    ],
    "trilinear-f16-large-rays-pack=1": [
        "trilinear_fwd_sens_v16(p,1,40,48,56,p,p,p,p,p,2,1600,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,1600,0)",
    ],
    "trilinear-f16-large-vol-pack=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-large-vol-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-large-both-pack=0": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-large-both-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-grid-none-pack=0": [
        "trilinear_fwd_grid_v16(p,2,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-bf16-grid-none-pack=1": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,2,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-bf16-grid-rays-pack=0": [
        "trilinear_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,256,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-bf16-grid-rays-pack=1": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "trilinear_fwd_sens_packed_v16(p,2,40,48,56,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-bf16-grid-vol-pack=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-grid-vol-pack=1": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-grid-both-pack=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-grid-both-pack=1": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-small-none-pack=0": [
        "trilinear_fwd_v16(p,2,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-bf16-small-none-pack=1": [
        "trilinear_fwd_v16(p,2,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-bf16-small-rays-pack=0": [
        "trilinear_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-bf16-small-rays-pack=1": [
        "trilinear_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-bf16-small-vol-pack=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-small-vol-pack=1": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-small-both-pack=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-small-both-pack=1": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-large-none-pack=0": [
        "trilinear_fwd_v16(p,2,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-bf16-large-none-pack=1": [
        "trilinear_fwd_v16(p,2,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-bf16-large-rays-pack=0": [
        "trilinear_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,1600,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,1600,0)",
    ],
    "trilinear-bf16-large-rays-pack=1": [
        "trilinear_fwd_sens_v16(p,2,40,48,56,p,p,p,p,p,2,1600,0,0,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,1600,0)",
    ],
    "trilinear-bf16-large-vol-pack=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-large-vol-pack=1": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-large-both-pack=0": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-bf16-large-both-pack=1": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f64-grid-none-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-grid-none-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-grid-rays-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-rays-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-vol-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-vol-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-both-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-both-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-none-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-small-none-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-small-rays-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-rays-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-vol-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-vol-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-both-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-both-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-large-none-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-large-none-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-large-rays-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-large-rays-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-large-vol-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-large-vol-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-large-both-pack=0": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-large-both-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,1600,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-grid-none-pack=1-reduce=max": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
    ],
    "trilinear-f64-grid-none-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
    ],
    "trilinear-f32-grid-rays-pack=1-reduce=max": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
        "trilinear_bwd_max(p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-rays-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
        "raise NotImplementedError: fp64 trilinear: backward is implemented for reducefn='sum'",
    ],
    "trilinear-f32-grid-vol-pack=1-reduce=max": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
        "trilinear_bwd_max(p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-vol-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
        "raise NotImplementedError: fp64 trilinear: backward is implemented for reducefn='sum'",
    ],
    "trilinear-f32-grid-both-pack=1-reduce=max": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
        "trilinear_bwd_max(p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-both-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,1,0,0)",
        "raise NotImplementedError: fp64 trilinear: backward is implemented for reducefn='sum'",
    ],
    "trilinear-f32-small-none-pack=1-reduce=max": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
    ],
    "trilinear-f64-small-none-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
    ],
    "trilinear-f32-small-rays-pack=1-reduce=max": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
        "trilinear_bwd_max(p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-rays-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
        "raise NotImplementedError: fp64 trilinear: backward is implemented for reducefn='sum'",
    ],
    "trilinear-f32-small-vol-pack=1-reduce=max": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
        "trilinear_bwd_max(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-vol-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
        "raise NotImplementedError: fp64 trilinear: backward is implemented for reducefn='sum'",
    ],
    "trilinear-f32-small-both-pack=1-reduce=max": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
        "trilinear_bwd_max(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-both-pack=1-reduce=max": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,1,0,0)",
        "raise NotImplementedError: fp64 trilinear: backward is implemented for reducefn='sum'",
    ],
    "trilinear-f32-grid-none-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-none-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-grid-rays-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,0,p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-grid-rays-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,1,p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-grid-vol-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,0,p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-grid-vol-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,1,p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-grid-both-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,0,p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-grid-both-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,1,p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-small-none-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-none-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-rays-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,0,p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-small-rays-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,1,p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-small-vol-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,0,p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-small-vol-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,1,p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-small-both-pack=1-reduce=callable": [
        "segments_fwd(1,0,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,0,p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-small-both-pack=1-reduce=callable": [
        "segments_fwd(1,1,p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
        "segments_bwd(1,1,p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-grid-none-align=1-pack=1": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
    ],
    "trilinear-f64-grid-none-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
    ],
    "trilinear-f32-grid-rays-align=1-pack=1": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,256,0,0,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,256,0)",
    ],
    "trilinear-f64-grid-rays-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-vol-align=1-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f64-grid-vol-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-both-align=1-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f64-grid-both-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-small-none-align=1-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
    ],
    "trilinear-f64-small-none-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
    ],
    "trilinear-f32-small-rays-align=1-pack=1": [
        "trilinear_fwd_sens(p,40,48,56,p,p,p,p,p,2,86,0,0,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_sens(p,p,p,p,p,p,2,86,0)",
    ],
    "trilinear-f64-small-rays-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-small-vol-align=1-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f64-small-vol-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-small-both-align=1-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f64-small-both-align=1-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,1,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f32-grid-none-mask=1-pack=1": [
        "trilinear_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-none-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-grid-rays-mask=1-pack=1": [
        "trilinear_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_mask_grid(p,p,40,48,56,p,p,p,p,p,p,p,0,p,2,16,16,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-rays-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-grid-vol-mask=1-pack=1": [
        "trilinear_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_mask_grid(p,p,40,48,56,p,p,p,p,0,0,0,p,0,2,16,16,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-vol-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-grid-both-mask=1-pack=1": [
        "trilinear_fwd_mask_grid(p,p,40,48,56,p,p,p,p,2,16,16,3,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_mask_grid(p,p,40,48,56,p,p,p,p,p,p,p,p,p,2,16,16,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-both-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-small-none-mask=1-pack=1": [
        "trilinear_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-none-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-small-rays-mask=1-pack=1": [
        "trilinear_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_mask(p,p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-rays-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-small-vol-mask=1-pack=1": [
        "trilinear_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_mask(p,p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-vol-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-small-both-mask=1-pack=1": [
        "trilinear_fwd_mask(p,p,40,48,56,p,p,p,p,2,86,3,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_mask(p,p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,3,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-both-mask=1-pack=1": [
        "raise NotImplementedError: fp64 trilinear is implemented without mask_to_channels",
    ],
    "trilinear-f32-grid-none-fused=0-pack=1": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_packed(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-none-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-grid-rays-fused=0-pack=1": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_packed(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_packed(p,40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-grid-rays-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-grid-vol-fused=0-pack=1": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,p,0,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f64-grid-vol-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-grid-both-fused=0-pack=1": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear-f64-grid-both-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,256,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,256,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-none-fused=0-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f64-small-none-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
    ],
    "trilinear-f32-small-rays-fused=0-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-rays-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,0,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-vol-fused=0-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-vol-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,0,0,0,p,0,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f32-small-both-fused=0-pack=1": [
        "trilinear_fwd(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f64-small-both-fused=0-pack=1": [
        "trilinear_fwd_f64(p,40,48,56,p,p,p,p,2,86,0.5,1e-08,40,p,0,0,0)",
        "trilinear_bwd_f64(p,40,48,56,p,p,p,p,p,p,p,p,p,2,86,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f16-grid-none-fused=0-pack=1": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,1,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear-f16-grid-rays-fused=0-pack=1": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "raise NotImplementedError: ray gradients from a torch.float16 volume come from the fused sensitivities march only",
    ],
    "trilinear-f16-grid-vol-fused=0-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear-f16-grid-both-fused=0-pack=1": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f32-pose-none-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f32-pose-none-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f32-pose-none-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f32-pose-none-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f32-pose-rays-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,2,16,16,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-rays-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,2,16,16,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-rays-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,0,p,p,2,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-rays-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,0,p,p,2,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-vol-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f32-pose-vol-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f32-pose-vol-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f32-pose-vol-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f32-pose-both-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-both-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,0,p,p,2,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-both-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-both-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,0,p,p,2,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f16-pose-none-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose_v16(p,1,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f16-pose-none-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick_v16(p,1,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f16-pose-none-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_pose_v16(p,1,40,48,56,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f16-pose-none-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick_v16(p,1,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f16-pose-rays-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,2,16,16,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f16-pose-rays-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,2,16,16,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f16-pose-rays-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: pose gradients from a torch.float16 volume come from the fused sensitivities walk only",
    ],
    "siddon_pose-f16-pose-rays-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: pose gradients from a torch.float16 volume come from the fused sensitivities walk only",
    ],
    "siddon_pose-f16-pose-vol-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-vol-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-vol-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-vol-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-both-B=2-brick=0-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-both-B=2-brick=1-fused=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-both-B=2-brick=0-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f16-pose-both-B=2-brick=1-fused=0": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "siddon_pose-f32-pose-none-B=2-brick=1-stop=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
    ],
    "siddon_pose-f32-pose-none-B=1-brick=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f32-pose-rays-B=2-brick=1-stop=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,2,16,16,1,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-rays-B=1-brick=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,1,16,16,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,1,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,1,0)",
    ],
    "siddon_pose-f32-pose-vol-B=2-brick=1-stop=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,10752,2,16,16,0.5,1e-08,0,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,0,p,p,2,16,16,0.5,1e-08,1,0)",
    ],
    "siddon_pose-f32-pose-vol-B=1-brick=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,5632,1,16,16,0.5,1e-08,0)",
    ],
    "siddon_pose-f32-pose-both-B=2-brick=1-stop=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_bwd_sens_pose(p,p,p,p,p,p,p,p,2,16,16,1,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "siddon_pose-f32-pose-both-B=1-brick=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_pose(p,40,48,56,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "siddon_bwd_vol_brick(p,40,48,56,p,0,0,p,p,p,p,p,p,5632,1,16,16,0.5,1e-08,0)",
        "siddon_bwd_pose(p,40,48,56,p,p,p,p,p,p,p,p,p,0,p,p,1,16,16,0.5,1e-08,0,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,1,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,1,0)",
    ],
    "trilinear_pose-f32-pose-none-B=2": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_packed(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear_pose-f32-pose-none-B=8": [
        "pack_corners(p,40,48,56,p,0)",
        "trilinear_fwd_packed(p,40,48,56,p,p,p,p,8,16,16,0.5,1e-08,40,p,16,0)",
    ],
    "trilinear_pose-f32-pose-rays-B=2": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "trilinear_pose-f32-pose-rays-B=8": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,8,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,8,0)",
    ],
    "trilinear_pose-f32-pose-vol-B=2": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,p,0,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear_pose-f32-pose-vol-B=8": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,8,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,0,0,0,p,0,8,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear_pose-f32-pose-both-B=2": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear_pose-f32-pose-both-B=8": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,8,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear_pose-f16-pose-none-B=2": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,1,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear_pose-f16-pose-none-B=8": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,1,40,48,56,p,p,p,p,8,16,16,0.5,1e-08,40,p,16,0)",
    ],
    "trilinear_pose-f16-pose-rays-B=2": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "trilinear_pose-f16-pose-rays-B=8": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,8,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,8,0)",
    ],
    "trilinear_pose-f16-pose-vol-B=2": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-f16-pose-vol-B=8": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-f16-pose-both-B=2": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-f16-pose-both-B=8": [
        "raise NotImplementedError: a torch.float16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-bf16-pose-none-B=2": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,2,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
    ],
    "trilinear_pose-bf16-pose-none-B=8": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "trilinear_fwd_packed_v16(p,2,40,48,56,p,p,p,p,8,16,16,0.5,1e-08,40,p,16,0)",
    ],
    "trilinear_pose-bf16-pose-rays-B=2": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "trilinear_pose-bf16-pose-rays-B=8": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,8,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,8,0)",
    ],
    "trilinear_pose-bf16-pose-vol-B=2": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-bf16-pose-vol-B=8": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-bf16-pose-both-B=2": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-bf16-pose-both-B=8": [
        "raise NotImplementedError: a torch.bfloat16 volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are supported; optimise an fp32 volume for volume gradients)",
    ],
    "trilinear_pose-f32-pose-rays-B=8-slab=16": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,16,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,8,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,8,0)",
    ],
    "trilinear_pose-f32-pose-rays-B=2-fused=0": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_bwd_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,0)",
        "pose_rays_bwd(p,p,p,p,p,p,p,2,0)",
        "euler_pose_bwd(p,p,2,0,1,1.0,p,p,p,2,0)",
    ],
    "trilinear_pose-f32-pose-both-B=8-slab=16": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,8,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "trilinear_pose-f32-pose-both-B=2-fused=0": [
        "trilinear_fwd_grid(p,40,48,56,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
        "trilinear_bwd_grid(p,40,48,56,p,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,1,0)",
    ],
    "siddon_jac-f32-pose-none-B=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,1,16,16,6,0,0)",
    ],
    "trilinear_jac-f32-pose-none-B=1": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,1,16,16,6,0)",
    ],
    "siddon_jac-f32-pose-none-B=2": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,2,16,16,6,0,0)",
    ],
    "trilinear_jac-f32-pose-none-B=2": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,6,0)",
    ],
    "siddon_jac-f32-pose-none-B=8": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,8,16,16,6,0,0)",
    ],
    "trilinear_jac-f32-pose-none-B=8": [
        "pack_corners(p,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,6,0)",
    ],
    "siddon_jac-f16-pose-none-B=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,1,16,16,6,0,0)",
    ],
    "trilinear_jac-f16-pose-none-B=1": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,1,16,16,6,0)",
    ],
    "siddon_jac-f16-pose-none-B=2": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,2,16,16,6,0,0)",
    ],
    "trilinear_jac-f16-pose-none-B=2": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,6,0)",
    ],
    "siddon_jac-f16-pose-none-B=8": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "siddon_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,8,16,16,6,0,0)",
    ],
    "trilinear_jac-f16-pose-none-B=8": [
        "pack_corners_v16(p,1,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,1,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,6,0)",
    ],
    "siddon_jac-bf16-pose-none-B=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "siddon_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,1,16,16,6,0,0)",
    ],
    "trilinear_jac-bf16-pose-none-B=1": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,1,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,1,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,1,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,1,16,16,6,0)",
    ],
    "siddon_jac-bf16-pose-none-B=2": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,2,16,16,6,0,0)",
    ],
    "trilinear_jac-bf16-pose-none-B=2": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,2,16,16,6,0)",
    ],
    "siddon_jac-bf16-pose-none-B=8": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "siddon_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,8,16,16,6,0,0)",
    ],
    "trilinear_jac-bf16-pose-none-B=8": [
        "pack_corners_v16(p,2,40,48,56,p,0)",
        "euler_pose_fwd(p,p,2,0,1,1.0,p,8,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,8,0)",
        "trilinear_alpha_range_pose(40,48,56,p,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,0)",
        "trilinear_fwd_sens_pose_v16(p,2,40,48,56,p,p,p,p,p,p,p,8,16,16,0.5,1e-08,40,p,0,0)",
        "trilinear_jac_sens_pose(p,p,p,p,p,p,p,p,p,8,16,16,6,0)",
    ],
    "siddon_jac-f32-pose-none-B=2-stop=1": [
        "euler_pose_fwd(p,p,2,0,1,1.0,p,2,0)",
        "pose_rays_fwd(p,p,p,p,p,p,p,2,0)",
        "siddon_fwd_sens_pose(p,40,48,56,p,p,p,p,p,p,p,2,16,16,0.5,1e-08,0)",
        "siddon_jac_sens_pose(p,p,p,p,p,p,p,p,2,16,16,6,1,0)",
    ],
}
