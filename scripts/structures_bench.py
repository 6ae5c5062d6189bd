#!/usr/bin/env python
"""structures_bench.py -- piecewise-rigid renders (DRR.render_structures, DESIGN.md 6f) against the composition they replace.

512^3 density (U[0,1) noise, 0.5 mm voxels) with K in {2, 8, 24} vertebra-sized labelled blocks (80 x 80 x 60 voxels, 40 x 40 x 30
mm) on a 4 x 3 x 2 grid plus background, 256^2 detector, B in {1, 16} poses, small random motions shared by the poses.
  new:          one render_structures call (K + 1 channels);
  composition:  K + 1 renders through DRR's fused pose-in path, channel k on density * (mask == label k) with pose X_k^-1 P, then
                a sum (the masked copies are made once, outside the timed region);
each forward only (no_grad) and forward + backward to the camera pose and the motions, alternated for --rounds rounds, median of
CUDA-event-timed calls after warm-up.  Outputs of the two paths are compared at the timed sizes.  Voxel visits are bounds from
shapes: per (pose, slot) the pixels of the footprint rectangle times the walked box's D0 + D1 + D2, against B H W (D0 + D1 + D2)
per channel for the composition; the background slot (a gated whole-volume walk) is reported on its own.  Prints one JSON line;
writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from diffdrr_b200 import DRR, synthetic  # noqa: E402
from diffdrr_b200.pose import RigidTransform, convert  # noqa: E402
from diffdrr_b200.structures import _mask_state, _rigid_inverse  # noqa: E402

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


def _label_volume(D, K):
    lab = torch.zeros(D, D, D, dtype=torch.float32)
    cells = [(i, j, k) for i in range(4) for j in range(3) for k in range(2)][:K]
    for n, (i, j, k) in enumerate(cells):
        o = (i * D // 4 + 20, j * D // 3 + 40, k * D // 2 + 90)
        lab[o[0]:o[0] + 80, o[1]:o[1] + 80, o[2]:o[2] + 60] = n + 1
    return lab


def _footprint_visits(drr, src, G, boxes, S, H, W):
    """Upper bound on voxel visits per slot: footprint-rectangle pixels x (sum of the box's extents), torch restatement of the
    kernel's box_corner_uv / footprint_rect."""
    rows, cols = drr._grid_axes(None)
    BS = G.shape[0]
    lo, hi = boxes[:, :3].float() - 0.5, boxes[:, 3:].float() - 0.5
    bits = torch.tensor([[(k >> a) & 1 for a in range(3)] for k in range(8)], device=G.device, dtype=torch.float32)
    corners = lo[:, None] + bits[None] * (hi - lo)[:, None]                                # (S, 8, 3)
    corners = corners.repeat(BS // S, 1, 1)                                               # (BS, 8, 3)
    M = torch.stack([G[:, :, 0], G[:, :, 1], G[:, :, 2] + G[:, :, 3] - src], dim=-1)      # (BS, 3, 3)
    y = torch.linalg.solve(M.double()[:, None].expand(-1, 8, -1, -1), (corners - src[:, None]).double()[..., None])[..., 0]
    ok = (y[..., 2] > 0).all(dim=1)
    u, v = y[..., 0] / y[..., 2], y[..., 1] / y[..., 2]
    dc, dr = (cols[-1] - cols[0]) / (W - 1), (rows[-1] - rows[0]) / (H - 1)
    pw, ph = (u - cols[0]) / dc, (v - rows[0]) / dr
    w0 = (pw.amin(1).floor() - 1).clamp(0, W - 1)
    w1 = (pw.amax(1).ceil() + 1).clamp(-1, W - 1)
    h0 = (ph.amin(1).floor() - 1).clamp(0, H - 1)
    h1 = (ph.amax(1).ceil() + 1).clamp(-1, H - 1)
    area = ((w1 - w0 + 1).clamp_min(0) * (h1 - h0 + 1).clamp_min(0))
    area = torch.where(ok, area, torch.full_like(area, H * W))
    extent = (boxes[:, 3:] - boxes[:, :3]).clamp_min(0).sum(1).double().repeat(BS // S)
    return (area * extent).view(BS // S, S).sum(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--structures", type=int, nargs="+", default=[2, 8, 24])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    D, H = args.vol, args.det
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    results = []
    for K in args.structures:
        lab = _label_volume(D, K)
        drr = DRR(synthetic.make_subject(vol, mask=lab), **synthetic.detector_kwargs(H)).to(dev)
        labels = tuple(range(1, K + 1))
        mask = drr.mask
        masked = [drr.density * (mask == k) for k in labels] + [drr.density * (mask == 0)]
        # one module whose density buffer is swapped for each masked copy (same affine and detector as drr)
        base = DRR(synthetic.make_subject(vol[:2, :2, :2]), **synthetic.detector_kwargs(H))
        base._affine.copy_(drr._affine)
        base._affine_inverse.copy_(drr._affine_inverse)
        base = base.to(dev)
        g = torch.Generator().manual_seed(K)
        X = convert((torch.rand(K, 3, generator=g) * 2 - 1) * 0.05, (torch.rand(K, 3, generator=g) * 2 - 1) * 5.0,
                    parameterization="euler_angles", convention="XYZ").matrix.to(dev)
        for B in args.batches:
            rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))

            def new(rot=rot, xyz=xyz, Xm=X):
                return drr.render_structures(rot, xyz, motions=Xm, labels=labels, **KW).sum(1, keepdim=True)

            def comp(rot=rot, xyz=xyz, Xm=X):
                P = convert(rot, xyz, **KW).matrix
                out = 0
                for k in range(K + 1):
                    base.density = masked[k]
                    Pk = _rigid_inverse(Xm[k]) @ P if k < K else P
                    out = out + base(RigidTransform(Pk))
                return out

            def train(fn):
                r, x, Xm = rot.clone().requires_grad_(True), xyz.clone().requires_grad_(True), X.clone().requires_grad_(True)

                def step():
                    fn(r, x, Xm).sum().backward()
                return step

            with torch.no_grad():
                a, b = new(), comp()
            err = float((a - b).abs().max() / b.abs().max())
            t = {"new_fwd": [], "comp_fwd": [], "new_train": [], "comp_train": []}
            steps = {"new_train": train(new), "comp_train": train(comp)}
            for _ in range(args.rounds):
                with torch.no_grad():
                    t["new_fwd"].append(_time(new, args.warmup, args.iters))
                    t["comp_fwd"].append(_time(comp, args.warmup, args.iters))
                t["new_train"].append(_time(steps["new_train"], args.warmup, args.iters))
                t["comp_train"].append(_time(steps["comp_train"], args.warmup, args.iters))
            with torch.no_grad():
                state = _mask_state(drr)
                P = convert(rot, xyz, **KW).matrix
                Ps = torch.cat([_rigid_inverse(X) @ P[:, None], P[:, None]], dim=1).reshape(-1, 4, 4)
                src, G, _, _, _ = drr._pose_in_inputs(RigidTransform(Ps), None)
                boxes = torch.cat([state["boxes"][list(labels)], torch.tensor([[0, 0, 0, D, D, D]], device=dev, dtype=torch.int32)])
                visits = _footprint_visits(drr, src, G, boxes, K + 1, H, H)
            whole = float(B * H * H * 3 * D)
            results.append(dict(K=K, B=B, rel_err_vs_composition=err,
                                ms={k: float(np.median(v)) for k, v in t.items()},
                                visit_bound_structures=float(visits[:K].sum()), visit_bound_background=float(visits[K]),
                                visit_bound_composition=whole * (K + 1)))
            print(json.dumps(results[-1]), file=sys.stderr, flush=True)
        del masked, drr, base
        torch.cuda.empty_cache()
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=D, det=H, results=results)))


if __name__ == "__main__":
    main()
