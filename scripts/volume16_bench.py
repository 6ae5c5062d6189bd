#!/usr/bin/env python
"""volume16_bench.py -- the Siddon projector on a 512^3 volume stored as fp32, fp16 and bf16 (DESIGN.md 4.5), at bench.py's
configuration (512^3 -> 256^2, 16 poses from synthetic.make_poses(16, seed=0), a U[0,1) volume).

Per storage type, alternating fp32 / fp16 / bf16 for --rounds rounds, warmed up, CUDA-event timed:
  - the kernels-only training step: b200drr_siddon_fwd_sens_grid (variant 0) + b200drr_siddon_bwd_sens, as bench.py times it
    (16-bit: b200drr_siddon_fwd_sens_grid_v16);
  - the inference forward through the module (DRR(rot, xyz) under no_grad) at B = 16 and at B = 1;
  - BASELINE config 3: 512^3 -> 512^2, 64 poses, Trilinear with 500 points, forward + backward to the pose through the module
    (the pose-in march over the packed-corner copy: 32 B per sample in fp32, 16 B per sample for 16-bit storage).
The roofline share counts ALGORITHMIC bytes: one voxel read per Siddon visit at the storage size (4 B fp32, 2 B 16-bit) plus the
per-ray traffic bench.py counts, over the HBM peak.  Prints one JSON line; writes nothing.
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

from diffdrr_b200 import DRR, _lib, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.renderers import _VOL16, _ptr, _stream, siddon_visits  # noqa: E402

HBM_PEAK_GBS = 3350.0  # H100 SXM (HBM3) data sheet


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-config3", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    D, H, B = args.vol, args.det, args.batch
    N = H * H
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    lib = _lib.load()

    gen = torch.Generator(device=dev).manual_seed(0)
    vol32 = torch.rand(D, D, D, device=dev, generator=gen)
    vols = {"float32": vol32, "float16": vol32.to(torch.float16), "bfloat16": vol32.to(torch.bfloat16)}
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H), renderer="siddon").to(dev)
    rot, xyz = synthetic.make_poses(B, seed=0)
    rot, xyz = rot.to(dev), xyz.to(dev)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot, xyz, parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).unsqueeze(1).contiguous()
        src, tgt = drr.affine_inverse(src).reshape(B, 3).contiguous(), drr.affine_inverse(tgt).contiguous()
    visits = int(siddon_visits((D, D, D), src, tgt).sum().item())
    out, sens, gout = torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev), torch.rand(B, N, device=dev, generator=gen)
    g_src, g_tgt, g_len = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev)

    def step(vol):
        if vol.dtype == torch.float32:
            _lib.check(lib.b200drr_siddon_fwd_sens_grid(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens),
                                                        B, H, H, 0.5, 1e-8, 0, _stream()), "fwd_sens_grid")
        else:
            _lib.check(lib.b200drr_siddon_fwd_sens_grid_v16(_ptr(vol), _VOL16[vol.dtype], D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                            _ptr(out), _ptr(sens), B, H, H, 0.5, 1e-8, 0, _stream()), "fwd_sens_grid_v16")
        _lib.check(lib.b200drr_siddon_bwd_sens(_ptr(sens), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), B, N, 0, _stream()),
                   "bwd_sens")

    def infer(b):
        def run():
            with torch.no_grad():
                drr(rot[:b], xyz[:b], parameterization="euler_angles", convention="ZXY")
        return run

    res = {k: {"train_step_ms": [], "fwd_b16_ms": [], "fwd_b1_ms": []} for k in vols}
    for _ in range(args.rounds):
        for name, vol in vols.items():
            drr.density = vol
            res[name]["train_step_ms"].append(_time(lambda: step(vol), args.warmup, args.iters))
            res[name]["fwd_b16_ms"].append(_time(infer(B), args.warmup, args.iters))
            res[name]["fwd_b1_ms"].append(_time(infer(1), args.warmup, args.iters * 5))
    if not args.no_config3:  # BASELINE config 3, same volume: trilinear fwd + bwd(pose) through the module
        B3, H3, P3 = 64, 512, 500
        tri = DRR(subj, **synthetic.detector_kwargs(H3), renderer="trilinear").to(dev)
        rot3, xyz3 = synthetic.make_poses(B3, seed=0)
        rot3, xyz3 = rot3.to(dev).requires_grad_(True), xyz3.to(dev).requires_grad_(True)

        def tri_step():
            img = tri(rot3, xyz3, parameterization="euler_angles", convention="ZXY", n_points=P3)
            img.sum().backward()

        for name in vols:
            res[name]["config3_ms"] = []
        for _ in range(args.rounds):
            for name, vol in vols.items():
                tri.density = vol
                res[name]["config3_ms"].append(_time(tri_step, 1, 3))
        tri.renderer.invalidate_packed()
    summary = {}
    for name in vols:
        esz = 4 if name == "float32" else 2
        train_bytes = esz * visits + (16 + 4 + 32) * B * N + (32 + 4 + 12 + 4 + 4) * B * N
        fwd_bytes = esz * visits + (4 + 16) * B * N
        r = res[name]
        t_train, t_fwd = float(np.median(r["train_step_ms"])), float(np.median(r["fwd_b16_ms"]))
        summary[name] = {
            **{k: [round(x, 4) for x in v] for k, v in r.items()},
            "train_drr_per_s": B / (t_train * 1e-3), "fwd_b16_drr_per_s": B / (t_fwd * 1e-3),
            "fwd_b1_drr_per_s": 1.0 / (float(np.median(r["fwd_b1_ms"])) * 1e-3),
            "train_roofline_frac": train_bytes / (t_train * 1e-3) / 1e9 / HBM_PEAK_GBS,
            "fwd_b16_roofline_frac": fwd_bytes / (t_fwd * 1e-3) / 1e9 / HBM_PEAK_GBS,
        }
        if "config3_ms" in r:
            t3 = float(np.median(r["config3_ms"]))
            summary[name]["config3_drr_per_s"] = 64 / (t3 * 1e-3)
            # algorithmic: one packed-cell read per sample (8 corners: 32 B fp32, 16 B 16-bit); the training step marches once
            summary[name]["config3_roofline_frac"] = (8 * esz * 64 * 512 * 512 * 500) / (t3 * 1e-3) / 1e9 / HBM_PEAK_GBS
    print(json.dumps({"gpu": smi.stdout.strip(), "workload": f"{D}^3 -> {H}^2, {B} poses, Siddon",
                      "roofline_basis": "algorithmic bytes: one voxel read per visit at the storage size (4 B fp32, 2 B fp16/bf16) "
                                        "+ per-ray traffic; trilinear: one packed cell per sample (32 B fp32, 16 B fp16/bf16), all 500 "
                                        "samples counted; HBM peak 3350 GB/s (data sheet)",
                      "visits": visits, "results": summary}), flush=True)


if __name__ == "__main__":
    main()
