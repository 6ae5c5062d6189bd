#!/usr/bin/env python
"""deform_bproj_bench.py -- the deformable render's transpose in the density (b200drr_deform_bproj, DESIGN.md 6l) on the GPU.

Setup: 512^3 fp32 density (U[0,1) noise) that requires grad, 256^2 detector, n_points = 500, a smooth ~5 mm world-mm field on a
32^3 and a 64^3 lattice, shared by the poses (B = 1 and 16) or one per pose (B = 16).  Per configuration, alternated for --rounds
rounds, the median of CUDA-event-timed calls after warm-up:
  fwd          b200drr_deform_fwd on the module's rays (rays precomputed; the plain-gather instantiation a density that
               requires grad takes);
  bproj        b200drr_deform_bproj on the same rays: the density-only backward (its memset included);
  dens_bwd     the same through autograd: torch.autograd.grad(img, V) on a retained graph;
  recon_step   one reconstruction step through the module: render_deformed(..., density=V) + the backward to V;
  joint_bwd    the backward of a joint density + field fit: b200drr_deform_bproj + b200drr_deform_bwd with only g_field;
  tri_fwd      the plain Trilinear renderer's forward on the same rays (field ignored), density requiring grad;
  tri_bwd      its volume-gradient backward (autograd on a retained graph): the same 8 reductions per in-volume sample;
  torch_step   (B = 1) the torch composition -- grid_sample of the field, then of the density, summed per ray -- forward and
               backward to the density.
The reduction count is 8 per sample whose pulled-back point lies in the zero-padded volume (counted with deform_bench.py's torch
composition; corners outside the volume are skipped, so it is an upper bound), and `bproj_reductions_per_s` is that count over
the bproj time.  At B = 1 the image and the density gradient are compared with the torch composition's.  The first configuration
also lists, from torch.profiler, every CUDA kernel and memset a density-only backward launches.

Prints one JSON line with the card's name and power limit; writes nothing.
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deform_bench import torch_composition  # noqa: E402
from deform_cases import smooth_field  # noqa: E402
from diffdrr_b200 import DRR, _lib, synthetic  # noqa: E402
from diffdrr_b200 import deform as dm  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream  # noqa: E402

KW = dict(parameterization="euler_angles", convention="ZXY")


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


def _relerr(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def launches(fn):
    """Names of the CUDA kernels and memsets `fn` launches (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sorted(set(names)), len(names)


def costs(args, dev):
    D, H, P = args.vol, args.det, args.n_points
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
    r, lib = drr.renderer, _lib.load()
    V = drr.density.detach().clone().requires_grad_(True)
    results, listed = [], False
    for g in args.lattices:
        for B, per_pose in ((1, False), (16, False), (16, True)):
            if B not in args.batches:
                continue
            field = torch.from_numpy(smooth_field(np.random.default_rng(g), B if per_pose else 1, (g, g, g), 5.0)).to(dev)
            field = field if per_pose else field[0]
            rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
            w = torch.randn(B, 1, H, H, device=dev)
            with torch.no_grad():
                source, marches = dm._marches(drr, (rot, xyz), B, "euler_angles", "ZXY", False, None, None, None, vol=V)
                tgt, lens, arange, grid = marches[0]
                U = dm.voxel_field(drr, field)
            src = source.reshape(B, 3).contiguous()
            raylen = lens.reshape(B, -1).contiguous()
            gout = w.reshape(B, -1).contiguous()
            g_vol = torch.empty_like(V)
            consts = (float(r.voxel_shift), float(r.eps), P, grid)

            def fwd():
                with torch.no_grad():
                    return dm._DeformFunction.apply(V, None, source, tgt, lens, U, arange, *consts)

            def bproj():
                _lib.check(lib.b200drr_deform_bproj(*V.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(U), U.shape[0], *U.shape[1:4],
                                                    _ptr(gout), _ptr(g_vol), B, H * H, H, H, consts[0], consts[1], P, _ptr(arange),
                                                    _stream()), "b200drr_deform_bproj")

            img = dm._DeformFunction.apply(V, None, source, tgt, lens, U, arange, *consts)

            def dens_bwd():
                return torch.autograd.grad(img, V, w.view(B, 1, -1), retain_graph=True)[0]

            def recon_step():
                out = drr.render_deformed(rot, xyz, field=field, n_points=P, density=V, **KW)
                return torch.autograd.grad(out, V, w)[0]

            def joint_bwd():
                bproj()
                dm.field_vjp(drr, None, source, tgt, lens, U, gout, arange, P, grid)

            amin, amax = (float(a) for a in arange)

            def tri_fwd():
                with torch.no_grad():
                    return r(V, source, tgt, lens, n_points=P, alphamin=amin, alphamax=amax)

            tri = r(V, source, tgt, lens, n_points=P, alphamin=amin, alphamax=amax)

            def tri_bwd():
                return torch.autograd.grad(tri, V, w.view(B, 1, -1), retain_graph=True)[0]

            res = dict(lattice=g, B=B, field="per-pose" if per_pose else "shared")
            if not listed:   # what a density-only backward launches
                names, count = launches(dens_bwd)
                res["dens_bwd_launches"], res["dens_bwd_launch_count"] = names, count
                listed = True
            saved = drr.density
            drr.density = V   # the composition reads drr.density
            try:
                with torch.set_grad_enabled(B == 1):   # only B = 1 goes backward through it
                    comp, inside = torch_composition(drr, rot, xyz, field, P)
                if B == 1:
                    gc = torch.autograd.grad(comp, V, w)[0]
                    res["img_relerr_vs_torch"] = _relerr(fwd().view(comp.shape), comp.detach())
                    res["grad_relerr_vs_torch"] = _relerr(dens_bwd(), gc)

                    def torch_step():
                        out, _ = torch_composition(drr, rot, xyz, field, P)
                        return torch.autograd.grad(out, V, w)[0]
                del comp
            finally:
                drr.density = saved
            fns = dict(fwd=fwd, bproj=bproj, dens_bwd=dens_bwd, recon_step=recon_step, joint_bwd=joint_bwd, tri_fwd=tri_fwd,
                       tri_bwd=tri_bwd)
            t = {k: [] for k in fns}
            if B == 1:
                t["torch_step"] = []
            for _ in range(args.rounds):
                for k, fn in fns.items():
                    t[k].append(_time(fn, args.warmup, args.iters))
                if B == 1:
                    drr.density = V
                    try:
                        t["torch_step"].append(_time(torch_step, 1, 2))
                    finally:
                        drr.density = saved
            res["ms"] = {k: float(np.median(v)) for k, v in t.items()}
            res["samples_in_volume"] = inside
            res["reductions"] = 8 * inside
            res["bproj_reductions_per_s"] = 8 * inside / (res["ms"]["bproj"] * 1e-3)
            res["bproj_over_tri_bwd"] = res["ms"]["bproj"] / res["ms"]["tri_bwd"]
            res["dens_bwd_over_fwd"] = res["ms"]["dens_bwd"] / res["ms"]["fwd"]
            results.append(res)
            print(json.dumps(res), file=sys.stderr, flush=True)
            del img, tri
            torch.cuda.empty_cache()
    return results


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
        raise SystemExit("deform_bproj_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    results = costs(args, dev)
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=args.vol, det=args.det, n_points=args.n_points, results=results)))


if __name__ == "__main__":
    main()
