#!/usr/bin/env python
"""svf_bench.py -- the scaling-and-squaring exponential (diffdrr_b200.svf, DESIGN.md 6m) and the log-Euclidean blended render.

exp:     the exponential of a smooth velocity (steps = 10) on lattices of 32^3, 64^3 and 128^3 nodes, Bf in {1, 16}: the kernels
         (svf_fwd: forward only; svf_train: forward + backward) against the same scaling and squaring written with
         torch.nn.functional.grid_sample (border padding, align_corners=True: the same clamped trilinear lookup), whose output is
         compared with the kernels'.  Byte model per node and step: one float4 read and one written (32 B compulsory) and 8 corner
         float4 reads that L2 mostly serves; `gbs` is the compulsory bytes over svf_fwd time.
render:  render_polyrigid(blend="log_euclidean") against blend="linear" at scripts/polyrigid_bench.py's configuration (512^3 ->
         256^2, n_points = 500, 64^3 lattice, K in {2, 8}, B in {1, 16}), forward (no_grad) and forward + backward to the camera
         pose and the motions; `assembly_share` is the velocity assembly's (polyrigid_velocity) share of the log-Euclidean forward.
Alternated rounds, median of CUDA-event-timed calls after warm-up.  Prints one JSON line; writes nothing.
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

from diffdrr_b200 import DRR, polyrigid_weights, svf, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402

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


def _alternate(fns, rounds, warmup, iters):
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            times[k].append(_time(fn, warmup, iters))
    return {k: float(np.median(v)) for k, v in times.items()}


def grid_sample_exp(U, steps, dims):
    """The scaling and squaring of the kernels in torch ops: U (Bf, g0, g1, g2, 4) voxel units -> (Bf, g0, g1, g2, 3)."""
    g = U.shape[1:4]
    sc = torch.tensor([g[a] / dims[a] for a in range(3)], device=U.device)
    idx = torch.stack(torch.meshgrid(*[torch.arange(n, device=U.device, dtype=torch.float32) for n in g], indexing="ij"), -1)
    den = torch.tensor([max(n - 1, 1) for n in g], device=U.device, dtype=torch.float32)
    u = U[..., :3]
    for k in range(steps):
        s = 2.0**-steps if k == 0 else 1.0
        q = 2.0 * (idx + s * u * sc) / den - 1.0
        look = torch.nn.functional.grid_sample(u.permute(0, 4, 1, 2, 3), q.flip(-1), mode="bilinear", padding_mode="border",
                                               align_corners=True).permute(0, 2, 3, 4, 1)
        u = s * (u + look)
    return u


def bench_exp(args, dev):
    rows = []
    for n in args.lattices:
        for Bf in args.fields:
            dims = (4 * n, 4 * n, 4 * n)
            gen = torch.Generator().manual_seed(n + Bf)
            coarse = torch.randn(Bf, 3, 4, 4, 4, generator=gen) * (0.1 * dims[0])
            v = torch.nn.functional.interpolate(coarse, size=(n, n, n), mode="trilinear", align_corners=True)
            U = torch.nn.functional.pad(v.permute(0, 2, 3, 4, 1), (0, 1)).contiguous().to(dev)
            gout = torch.randn(U.shape, generator=gen).to(dev)
            gout[..., 3] = 0
            Ug = U.clone().requires_grad_(True)
            Ut = U.clone().requires_grad_(True)
            with torch.no_grad():
                ours = svf._SquaringFunction.apply(U, args.steps, dims)[..., :3]
                ref = grid_sample_exp(U, args.steps, dims)
                err = float((ours - ref).abs().max() / ref.abs().max())

            def svf_fwd():
                with torch.no_grad():
                    svf._SquaringFunction.apply(U, args.steps, dims)

            def svf_train():
                Ug.grad = None
                svf._SquaringFunction.apply(Ug, args.steps, dims).backward(gout)

            def gs_fwd():
                with torch.no_grad():
                    grid_sample_exp(U, args.steps, dims)

            def gs_train():
                Ut.grad = None
                grid_sample_exp(Ut, args.steps, dims).backward(gout[..., :3])

            t = _alternate(dict(svf_fwd=svf_fwd, svf_train=svf_train, gs_fwd=gs_fwd, gs_train=gs_train), args.rounds, args.warmup,
                           args.iters)
            nodes = Bf * n**3
            rows.append(dict(lattice=n, Bf=Bf, steps=args.steps, max_rel_diff_vs_grid_sample=err, **{k: round(x, 4) for k, x in t.items()},
                             gbs=round(32.0 * nodes * args.steps / (t["svf_fwd"] * 1e-3) / 1e9, 1),
                             fwd_speedup=round(t["gs_fwd"] / t["svf_fwd"], 2), train_speedup=round(t["gs_train"] / t["svf_train"], 2)))
            print(json.dumps(rows[-1]), file=sys.stderr)
    return rows


def _label_volume(D, K):
    lab = torch.zeros(D, D, D, dtype=torch.float32)
    cells = [(i, j) for i in range(4) for j in range(2)][:K]
    for n, (i, j) in enumerate(cells):
        o = (i * D // 4 + D // 32, j * D // 2 + D // 8, D // 3)
        lab[o[0]:o[0] + D // 6, o[1]:o[1] + D // 6, o[2]:o[2] + D // 8] = n + 1
    return lab


def bench_render(args, dev):
    D, H, P, g = args.vol, args.det, args.n_points, args.lattice
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    spacing = tuple(float(synthetic.make_affine(D)[a, a]) for a in range(3))
    rows = []
    for K in args.structures:
        drr = DRR(synthetic.make_subject(vol, mask=_label_volume(D, K)), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
        W = polyrigid_weights(drr.mask, tuple(range(1, K + 1)), grid=(g, g, g), sigma=6.0, spacing=spacing)
        gen = torch.Generator().manual_seed(K)
        X = convert((torch.rand(K, 3, generator=gen) * 2 - 1) * 0.05, (torch.rand(K, 3, generator=gen) * 2 - 1) * 5.0,
                    parameterization="euler_angles", convention="XYZ").matrix.to(dev)
        for B in args.batches:
            rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=1))
            kw = dict(weights=W, n_points=P, **KW)
            rot_g, xyz_g, X_g = (t.clone().requires_grad_(True) for t in (rot, xyz, X))

            def fwd(blend):
                def f():
                    with torch.no_grad():
                        drr.render_polyrigid(rot, xyz, motions=X, blend=blend, **kw)
                return f

            def train(blend):
                def f():
                    for t in (rot_g, xyz_g, X_g):
                        t.grad = None
                    drr.render_polyrigid(rot_g, xyz_g, motions=X_g, blend=blend, **kw).sum().backward()
                return f

            def assembly():
                with torch.no_grad():
                    svf.polyrigid_velocity(drr, X, W)

            with torch.no_grad():
                a = drr.render_polyrigid(rot, xyz, motions=X, blend="log_euclidean", **kw)
                b = drr.render_polyrigid(rot, xyz, motions=X, blend="linear", **kw)
                diff = float((a - b).abs().max() / b.abs().max())
            t = _alternate(dict(log_fwd=fwd("log_euclidean"), lin_fwd=fwd("linear"), log_train=train("log_euclidean"),
                                lin_train=train("linear"), assembly=assembly), args.rounds, args.warmup, args.iters)
            rows.append(dict(K=K, B=B, **{k: round(x, 3) for k, x in t.items()},
                             assembly_share=round(t["assembly"] / t["log_fwd"], 3), max_rel_diff_log_vs_linear=diff))
            print(json.dumps(rows[-1]), file=sys.stderr)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lattices", type=int, nargs="+", default=[32, 64, 128])
    ap.add_argument("--fields", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--n-points", type=int, default=500)
    ap.add_argument("--lattice", type=int, default=64)
    ap.add_argument("--structures", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--skip-render", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("svf_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = dict(gpu=smi.stdout.strip(), exp=bench_exp(args, dev))
    if not args.skip_render:
        out["render"] = bench_render(args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
