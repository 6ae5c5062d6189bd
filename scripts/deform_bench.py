#!/usr/bin/env python
"""deform_bench.py -- deformable renders (DRR.render_deformed, DESIGN.md 6i) against their floor and against torch.

512^3 density (U[0,1) noise), 256^2 detector, n_points = 500, a smooth shared world-mm displacement field of ~5 mm on a 32^3 and a
64^3 lattice, B in {1, 16} poses, fp32 and bf16 densities.  Per configuration, alternated for --rounds rounds, median of
CUDA-event-timed calls after warm-up:
  def_fwd          render_deformed forward (no_grad);
  def_train        forward + backward to the camera pose and the field (the field scatter included);
  def_train_nofld  forward + backward to the camera pose only: the backward launches with g_field = NULL and skips the scatter, so
                   def_train - def_train_nofld is the scatter's cost;
  tri_fwd          the plain Trilinear forward drr(rot, xyz) on the same rays: the floor (same density bytes, no field);
  torch_fwd        what a user would otherwise write: grid_sample of the field at the samples, then grid_sample of the density, one
                   pose at a time (fp32 density only); torch_train the same with backward to the field (B = 1 only: at B = 16 the
                   saved sample tensors of all poses would not fit).
The image is compared with the torch composition (on the up-cast density for bf16) and the largest difference is reported.
flushes_per_ray: how often a ray adds its 8 x 3 field registers to the lattice gradient, counted by the host emulation
(tests/hostemu/hostemu_deform.cpp, the kernels' own per-ray code) on every 8th row and column of the B = 1 rays; each flush is
at most 8 vector reductions of 16 B.  Bytes model: 32 B (16 B for a 16-bit density) per sample whose pulled-back point lies in the
zero-padded volume -- one packed-corner cell -- plus the field lattice once; `hbm_share_def_fwd` is those bytes over def_fwd time
over the H100 SXM data sheet's 3.35 TB/s, a statement about the packed copy's byte bound and nothing about achieved DRAM
bandwidth (L2 serves the cells neighbouring rays share, and the field's 8 float4 reads per sample are L2 traffic it leaves out).
Prints one JSON line; writes nothing but the host emulation's library (built once under tests/hostemu/).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deform_cases import smooth_field  # noqa: E402
from diffdrr_b200 import DRR, synthetic  # noqa: E402
from diffdrr_b200.deform import voxel_field  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.renderers import _dims_tensor, _get_alpha_minmax  # noqa: E402

KW = dict(parameterization="euler_angles", convention="ZXY")
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def _time(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def _norm(p, dims):
    """voxel coordinates (..., 3) -> grid_sample coordinates (align_corners=False), last axis ordered (D2, D1, D0)."""
    return (2.0 * (p + 0.5) / dims - 1.0).flip(-1)


def _rays(drr, rot, xyz):
    source, target = drr.detector(convert(rot, xyz, **KW), None)
    raylen = (target - source).norm(dim=-1)
    src, tgt = drr.affine_inverse(source), drr.affine_inverse(target)
    dims = _dims_tensor(drr.density.shape, src.device, torch.float32)
    amin, amax = _get_alpha_minmax(src, tgt, dims, 0.5, 1e-8)
    return src, tgt, raylen, amin.min(), amax.max()


def torch_composition(drr, rot, xyz, field, n_points):
    """render_deformed in torch ops, one pose at a time -> (image (B, 1, H, W), samples whose pulled-back point is in the padded
    volume).  Differentiable in `field`."""
    vol = drr.density.float()
    dims = _dims_tensor(vol.shape, vol.device, torch.float32)
    src, tgt, raylen, amin, amax = _rays(drr, rot, xyz)
    alpha = torch.linspace(0, 1, n_points, device=vol.device) * (amax - amin) + amin
    U = voxel_field(drr, field)[..., :3].movedim(-1, 1)                                            # (Bf, 3, g0, g1, g2)
    out, inside = [], 0
    for b in range(src.shape[0]):
        d = tgt[b] - src[b] + 1e-8
        x = src[b, :, None, :] + alpha[None, :, None] * d[:, None, :]                              # (N, P, 3)
        u = torch.nn.functional.grid_sample(U[b if U.shape[0] > 1 else 0][None], _norm(x, dims)[None, None], mode="bilinear",
                                            padding_mode="zeros", align_corners=False)[0, :, 0]     # (3, N, P)
        y = x + u.movedim(0, -1)
        inside += int(((y > -1) & (y < dims)).all(-1).sum())
        v = torch.nn.functional.grid_sample(vol[None, None], _norm(y, dims)[None, None], mode="bilinear", padding_mode="zeros",
                                            align_corners=False)[0, 0, 0]                         # (N, P)
        out.append(raylen[b] * ((amax - amin) / (n_points - 1)) * v.sum(-1))
    det = drr.detector
    return torch.stack(out).view(-1, 1, det.height, det.width), inside


def flushes_per_ray(drr, rot, xyz, field, n_points, every=8):
    """Mean and largest number of flushes per ray of the host emulation on every `every`-th row and column of pose 0."""
    from hostemu import emu_deform
    src, tgt, raylen, amin, amax = _rays(drr, rot[:1], xyz[:1])
    det = drr.detector
    tgt = tgt.view(1, det.height, det.width, 3)[:, ::every, ::every].reshape(1, -1, 3)
    raylen = raylen.view(1, det.height, det.width)[:, ::every, ::every].reshape(1, -1)
    U = voxel_field(drr, field)[..., :3].movedim(-1, 1)
    vol = drr.density.float().cpu().numpy()
    res = emu_deform.deform(vol, src[:, 0].cpu().numpy(), tgt.cpu().numpy(), raylen.cpu().numpy(), U.cpu().numpy(), n_points,
                            float(amin), float(amax), gout=np.ones(raylen.shape, np.float32))
    return float(res["flushes"].mean()), int(res["flushes"].max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--n-points", type=int, default=500)
    ap.add_argument("--lattices", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deform_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    D, H, P = args.vol, args.det, args.n_points
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    results = []
    for g in args.lattices:
        field = torch.from_numpy(smooth_field(np.random.default_rng(g), 1, (g, g, g), 5.0)[0]).to(dev)
        for dtype in (torch.float32, torch.bfloat16):
            drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
            if dtype != torch.float32:
                drr.density = drr.density.to(dtype)
            for B in args.batches:
                rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))

                def deformed(r=rot, x=xyz, u=field):
                    return drr.render_deformed(r, x, field=u, n_points=P, **KW)

                def tri(r=rot, x=xyz, u=None):
                    return drr(r, x, n_points=P, **KW)

                def train(fn, field_grad=True):
                    r, x = (t.clone().requires_grad_(True) for t in (rot, xyz))
                    u = field.clone().requires_grad_(field_grad)
                    return lambda: fn(r, x, u).sum().backward()

                def torch_train():
                    u = field.clone().requires_grad_(True)
                    torch_composition(drr, rot, xyz, u, P)[0].sum().backward()

                res = dict(lattice=g, B=B, density=str(dtype).replace("torch.", ""))
                with torch.no_grad():
                    img = deformed()
                    comp, inside = torch_composition(drr, rot, xyz, field, P)
                    res["max_abs_diff_vs_torch"] = float((img - comp).abs().max())
                    res["rel_err_vs_torch"] = float((img - comp).abs().max() / comp.abs().max())
                    res["moved"] = float((img - tri()).abs().max() / comp.abs().max())
                    del comp
                t = {k: [] for k in ("def_fwd", "tri_fwd", "def_train", "def_train_nofld", "torch_fwd", "torch_train")}
                steps = dict(def_train=train(deformed), def_train_nofld=train(deformed, field_grad=False))
                for _ in range(args.rounds):
                    with torch.no_grad():
                        t["def_fwd"].append(_time(deformed, args.warmup, args.iters))
                        t["tri_fwd"].append(_time(tri, args.warmup, args.iters))
                        if dtype == torch.float32:
                            t["torch_fwd"].append(_time(lambda: torch_composition(drr, rot, xyz, field, P), 1, 2))
                    t["def_train"].append(_time(steps["def_train"], args.warmup, args.iters))
                    t["def_train_nofld"].append(_time(steps["def_train_nofld"], args.warmup, args.iters))
                    if dtype == torch.float32 and B == 1:
                        t["torch_train"].append(_time(torch_train, 1, 2))
                res["ms"] = {k: float(np.median(v)) for k, v in t.items() if v}
                cell = 32 if dtype == torch.float32 else 16
                res["samples_in_volume"] = inside
                res["model_bytes"] = inside * cell + g ** 3 * 16
                res["hbm_share_def_fwd"] = res["model_bytes"] / (res["ms"]["def_fwd"] * 1e-3) / HBM_BYTES_PER_S
                if B == 1:
                    res["flushes_per_ray_mean"], res["flushes_per_ray_max"] = flushes_per_ray(drr, rot, xyz, field, P)
                results.append(res)
                print(json.dumps(res), file=sys.stderr, flush=True)
            del drr
            torch.cuda.empty_cache()
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=D, det=H, n_points=P, results=results)))


if __name__ == "__main__":
    main()
