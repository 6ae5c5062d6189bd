#!/usr/bin/env python
"""polyrigid_bproj_bench.py -- the blended-rigid render's transpose in the density (b200drr_polyrigid_bproj, DESIGN.md 6o) on the GPU.

Setup: 512^3 fp32 density (U[0,1) noise) that requires grad, 256^2 detector, n_points = 500, K = 2 and 8 labelled blocks blended
on a 64^3 weight lattice (polyrigid_bench.py's scene), motions of about 0.05 rad and 5 mm shared by the poses (B = 1 and 16) or
one set per pose (B = 16).  Per configuration, alternated for --rounds rounds, the median of CUDA-event-timed calls after warm-up:
  fwd          b200drr_polyrigid_fwd on the module's rays (rays precomputed; the plain-gather instantiation a density that
               requires grad takes);
  bproj        b200drr_polyrigid_bproj on the same rays: the density-only backward (its memset included);
  recon_step   one reconstruction step through the module: render_polyrigid(..., density=V) + the backward to V;
  joint_bwd    the backward of a joint density + motion fit on a retained graph: b200drr_polyrigid_bproj + b200drr_polyrigid_bwd;
  deform_bproj b200drr_deform_bproj on the same rays with a zero 64^3 field;
  tri_bwd      the plain Trilinear renderer's volume-gradient backward on the same rays (autograd on a retained graph);
  torch_step   (B = 1) the torch composition (polyrigid_bench.py's: grid_sample of the weights, blend, grid_sample of the density)
               forward and backward to the density.
The reduction count is 8 per sample whose pulled-back point lies in the zero-padded volume (counted with the torch composition;
corners outside the volume are skipped, so it is an upper bound), and `bproj_reductions_per_s` is that count over the bproj time.
At B = 1 the image and the density gradient are compared with the torch composition's.  The first configuration also lists, from
torch.profiler, how many CUDA kernels and memsets one reconstruction step launches, and every one its backward launches.

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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from polyrigid_bench import _label_volume, torch_composition  # noqa: E402
from diffdrr_b200 import DRR, _lib, polyrigid_weights, synthetic  # noqa: E402
from diffdrr_b200 import deform as dm  # noqa: E402
from diffdrr_b200 import polyrigid as pr  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
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
    """Names of the CUDA kernels and memsets `fn` launches (torch.profiler), in launch order."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _motions(K, B, per_pose, dev):
    gen = torch.Generator().manual_seed(K)
    n = B if per_pose else 1
    X = convert((torch.rand(n * K, 3, generator=gen) * 2 - 1) * 0.05, (torch.rand(n * K, 3, generator=gen) * 2 - 1) * 5.0,
                parameterization="euler_angles", convention="XYZ").matrix.to(dev)
    return X.view(B, K, 4, 4) if per_pose else X


def costs(args, dev):
    D, H, P, g = args.vol, args.det, args.n_points, args.lattice
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    spacing = tuple(float(synthetic.make_affine(D)[a, a]) for a in range(3))
    lib = _lib.load()
    results, listed = [], False
    for K in args.structures:
        drr = DRR(synthetic.make_subject(vol, mask=_label_volume(D, K)), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
        r = drr.renderer
        W = polyrigid_weights(drr.mask, tuple(range(1, K + 1)), grid=(g, g, g), sigma=6.0, spacing=spacing)
        wp = pr._packed_weights(drr, W)
        V = drr.density.detach().clone().requires_grad_(True)
        zero_field = torch.zeros(1, g, g, g, 4, device=dev)
        for B, per_pose in ((1, False), (16, False), (16, True)):
            if B not in args.batches:
                continue
            X = _motions(K, B, per_pose, dev)
            rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
            w = torch.randn(B, 1, H, H, device=dev)
            with torch.no_grad():
                source, marches = dm._marches(drr, (rot, xyz), B, "euler_angles", "ZXY", False, None, None, None, vol=V)
                tgt, lens, arange, grid = marches[0]
                M = pr.voxel_maps(drr, X)
                M = (M if M.dim() == 4 else M[None]).contiguous()
            src = source.reshape(B, 3).contiguous()
            raylen = lens.reshape(B, -1).contiguous()
            gout = w.reshape(B, -1).contiguous()
            g_vol = torch.empty_like(V)
            consts = ((g, g, g), float(r.voxel_shift), float(r.eps), P, grid)

            def fwd():
                with torch.no_grad():
                    return pr._PolyrigidFunction.apply(V, None, source, tgt, lens, M, arange, wp, *consts)

            def bproj():
                _lib.check(lib.b200drr_polyrigid_bproj(*V.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(M), M.shape[0], K, _ptr(wp),
                                                       g, g, g, _ptr(gout), _ptr(g_vol), B, H * H, H, H, consts[1], consts[2], P,
                                                       _ptr(arange), _stream()), "b200drr_polyrigid_bproj")

            def recon_step():
                out = drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=P, density=V, **KW)
                return torch.autograd.grad(out, V, w)[0]

            Mg = M.clone().requires_grad_(True)
            img = pr._PolyrigidFunction.apply(V, None, source, tgt, lens, Mg, arange, wp, *consts)

            def joint_bwd():
                return torch.autograd.grad(img, (V, Mg), w.view(B, 1, -1), retain_graph=True)

            def deform_bproj():
                _lib.check(lib.b200drr_deform_bproj(*V.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(zero_field), 1, g, g, g,
                                                    _ptr(gout), _ptr(g_vol), B, H * H, H, H, consts[1], consts[2], P, _ptr(arange),
                                                    _stream()), "b200drr_deform_bproj")

            amin, amax = (float(a) for a in arange)
            tri = r(V, source, tgt, lens, n_points=P, alphamin=amin, alphamax=amax)

            def tri_bwd():
                return torch.autograd.grad(tri, V, w.view(B, 1, -1), retain_graph=True)[0]

            res = dict(K=K, B=B, motions="per-pose" if per_pose else "shared")
            if not listed:   # what one reconstruction step launches: the forward with its ray and map set-up, then the backward
                res["recon_step_launch_count"] = len(launches(recon_step))
                out = drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=P, density=V, **KW)
                res["recon_bwd_launches"] = launches(lambda: torch.autograd.grad(out, V, w))
                del out
                listed = True
            saved = drr.density
            drr.density = V   # the composition reads drr.density
            try:
                with torch.set_grad_enabled(B == 1):   # only B = 1 goes backward through it
                    comp, inside = torch_composition(drr, rot, xyz, X, W, P)
                if B == 1:
                    gc = torch.autograd.grad(comp, V, w)[0]
                    res["img_relerr_vs_torch"] = _relerr(fwd().view(comp.shape), comp.detach())
                    bproj()
                    res["grad_relerr_vs_torch"] = _relerr(g_vol, gc)

                    def torch_step():
                        out, _ = torch_composition(drr, rot, xyz, X, W, P)
                        return torch.autograd.grad(out, V, w)[0]
                del comp
            finally:
                drr.density = saved
            fns = dict(fwd=fwd, bproj=bproj, recon_step=recon_step, joint_bwd=joint_bwd, deform_bproj=deform_bproj, tri_bwd=tri_bwd)
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
            res["bproj_reductions_per_s"] = 8 * inside / (res["ms"]["bproj"] * 1e-3)
            res["bproj_over_deform_bproj"] = res["ms"]["bproj"] / res["ms"]["deform_bproj"]
            res["bproj_over_tri_bwd"] = res["ms"]["bproj"] / res["ms"]["tri_bwd"]
            if B == 1:
                res["torch_step_over_recon_step"] = res["ms"]["torch_step"] / res["ms"]["recon_step"]
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
    ap.add_argument("--lattice", type=int, default=64)
    ap.add_argument("--structures", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("polyrigid_bproj_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    results = costs(args, dev)
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=args.vol, det=args.det, n_points=args.n_points, lattice=args.lattice,
                          results=results)))


if __name__ == "__main__":
    main()
