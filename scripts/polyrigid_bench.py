#!/usr/bin/env python
"""polyrigid_bench.py -- blended-rigid renders (DRR.render_polyrigid, DESIGN.md 6h) against their floor and against torch.

512^3 density (U[0,1) noise), 256^2 detector, n_points = 500, K in {2, 8} labelled blocks with a 64^3 weight lattice
(polyrigid_weights, sigma 6 mm), B in {1, 16} poses, fp32 and bf16 densities.  Per configuration, alternated for --rounds rounds,
median of CUDA-event-timed calls after warm-up:
  poly_fwd / poly_train   render_polyrigid forward (no_grad), and forward + backward to the camera pose and the motions;
  tri_fwd / tri_train     the plain Trilinear forward and training step on the same rays: the floor (same density bytes, no blend);
  torch_fwd               what a user would otherwise write: grid_sample of the weights at the samples, blend, grid_sample of the
                          density (fp32 density only, one pose at a time; its output is compared with render_polyrigid's).
Bytes model: 32 B (16 B for a 16-bit density) per sample whose pulled-back point lies in the zero-padded volume -- one packed-corner
cell -- plus the weight lattice once; `hbm_share` is those bytes over poly_fwd time over the H100 SXM data sheet's 3.35 TB/s.  The
model counts compulsory density bytes only: cells shared by neighbouring rays are counted once per sample although L2 serves many
of them, and the ~8 K weight reads per sample are L2 traffic it leaves out, so the share says how close the march is to the
packed copy's byte bound and nothing about achieved DRAM bandwidth.  Prints one JSON line; writes nothing.
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

from diffdrr_b200 import DRR, polyrigid_weights, synthetic  # noqa: E402
from diffdrr_b200.polyrigid import voxel_maps  # noqa: E402
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


def _label_volume(D, K):
    lab = torch.zeros(D, D, D, dtype=torch.float32)
    cells = [(i, j, k) for i in range(4) for j in range(2) for k in range(1)][:K]
    for n, (i, j, k) in enumerate(cells):
        o = (i * D // 4 + D // 32, j * D // 2 + D // 8, D // 3)
        lab[o[0]:o[0] + D // 6, o[1]:o[1] + D // 6, o[2]:o[2] + D // 8] = n + 1
    return lab


def _norm(p, dims):
    """voxel coordinates (..., 3) -> grid_sample coordinates (align_corners=False), last axis ordered (D2, D1, D0)."""
    return (2.0 * (p + 0.5) / dims - 1.0).flip(-1)


def torch_composition(drr, rot, xyz, X, W, n_points):
    """render_polyrigid in torch ops, one pose at a time -> (image (B, 1, H, W), samples whose pulled-back point is in the padded
    volume)."""
    vol = drr.density.float()
    dims = _dims_tensor(vol.shape, vol.device, torch.float32)
    source, target = drr.detector(convert(rot, xyz, **KW), None)
    raylen = (target - source).norm(dim=-1)
    src, tgt = drr.affine_inverse(source), drr.affine_inverse(target)
    amin, amax = _get_alpha_minmax(src, tgt, dims, 0.5, 1e-8)
    amin, amax = amin.min(), amax.max()
    alpha = torch.linspace(0, 1, n_points, device=vol.device) * (amax - amin) + amin
    M = voxel_maps(drr, X)
    out, inside = [], 0
    for b in range(src.shape[0]):
        d = tgt[b] - src[b] + 1e-8
        x = src[b, :, None, :] + alpha[None, :, None] * d[:, None, :]                              # (N, P, 3)
        w = torch.nn.functional.grid_sample(W[None], _norm(x, dims)[None, None], mode="bilinear", padding_mode="zeros",
                                            align_corners=False)[0, :, 0]                         # (K, N, P)
        Mb = M if M.dim() == 3 else M[b]
        y = x.clone()
        for k in range(Mb.shape[0]):
            y += w[k, ..., None] * (x @ Mb[k, :, :3].T + Mb[k, :, 3] - x)
        inside += int(((y > -1) & (y < dims)).all(-1).sum())
        v = torch.nn.functional.grid_sample(vol[None, None], _norm(y, dims)[None, None], mode="bilinear", padding_mode="zeros",
                                            align_corners=False)[0, 0, 0]                         # (N, P)
        out.append(raylen[b] * ((amax - amin) / (n_points - 1)) * v.sum(-1))
    det = drr.detector
    return torch.stack(out).view(-1, 1, det.height, det.width), inside


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
        raise SystemExit("polyrigid_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    D, H, P, g = args.vol, args.det, args.n_points, args.lattice
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    spacing = tuple(float(synthetic.make_affine(D)[a, a]) for a in range(3))
    results = []
    for K in args.structures:
        lab = _label_volume(D, K)
        labels = tuple(range(1, K + 1))
        gen = torch.Generator().manual_seed(K)
        X = convert((torch.rand(K, 3, generator=gen) * 2 - 1) * 0.05, (torch.rand(K, 3, generator=gen) * 2 - 1) * 5.0,
                    parameterization="euler_angles", convention="XYZ").matrix.to(dev)
        for dtype in (torch.float32, torch.bfloat16):
            drr = DRR(synthetic.make_subject(vol, mask=lab), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
            W = polyrigid_weights(drr.mask, labels, grid=(g, g, g), sigma=6.0, spacing=spacing)
            if dtype != torch.float32:
                drr.density = drr.density.to(dtype)
            for B in args.batches:
                rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))

                def poly(r=rot, x=xyz, Xm=X):
                    return drr.render_polyrigid(r, x, motions=Xm, weights=W, n_points=P, **KW)

                def tri(r=rot, x=xyz, Xm=None):
                    return drr(r, x, n_points=P, **KW)

                def train(fn):
                    r, x, Xm = (t.clone().requires_grad_(True) for t in (rot, xyz, X))
                    return lambda: fn(r, x, Xm).sum().backward()

                res = dict(K=K, B=B, density=str(dtype).replace("torch.", ""))
                with torch.no_grad():
                    img = poly()
                    comp, inside = torch_composition(drr, rot, xyz, X, W, P)
                    res["rel_err_vs_torch"] = float((img - comp).abs().max() / comp.abs().max())
                    res["moved"] = float((img - tri()).abs().max() / comp.abs().max())
                t = {k: [] for k in ("poly_fwd", "tri_fwd", "poly_train", "tri_train", "torch_fwd")}
                steps = dict(poly_train=train(poly), tri_train=train(tri))
                for _ in range(args.rounds):
                    with torch.no_grad():
                        t["poly_fwd"].append(_time(poly, args.warmup, args.iters))
                        t["tri_fwd"].append(_time(tri, args.warmup, args.iters))
                        if dtype == torch.float32:
                            t["torch_fwd"].append(_time(lambda: torch_composition(drr, rot, xyz, X, W, P), 1, 2))
                    t["poly_train"].append(_time(steps["poly_train"], args.warmup, args.iters))
                    t["tri_train"].append(_time(steps["tri_train"], args.warmup, args.iters))
                res["ms"] = {k: float(np.median(v)) for k, v in t.items() if v}
                cell = 32 if dtype == torch.float32 else 16
                res["samples_in_volume"] = inside
                res["model_bytes"] = inside * cell + W.numel() * 4
                res["hbm_share_poly_fwd"] = res["model_bytes"] / (res["ms"]["poly_fwd"] * 1e-3) / HBM_BYTES_PER_S
                res["flop_per_sample_model"] = 40 + 20 * K
                results.append(res)
                print(json.dumps(res), file=sys.stderr, flush=True)
            del drr
            torch.cuda.empty_cache()
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=D, det=H, n_points=P, lattice=g, results=results)))


if __name__ == "__main__":
    main()
