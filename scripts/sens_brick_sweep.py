"""Training-step kernels (image + per-ray sensitivities, b200drr_siddon_fwd_sens_grid) at 512^3 -> 256^2 over the batch size:
the slab-major kernel (variant 41), the major-axis pieces (variant 116: 16 pieces per ray) and the brick kernel's sensitivities
mode (variant 42).  Kernels alternate in blocks of --block back-to-back launches (1 = launch by launch), --reps blocks each;
every launch is timed with CUDA events.
Prints one JSON line per batch size (median / min us per launch, largest difference of the image and of each sensitivity
component to the slab kernel's, relative to that output's maximum) and the card it ran on; the batch threshold of
siddon_sens_brick_route (csrc/siddon_brick.cu) comes from this table.

    python scripts/sens_brick_sweep.py [--batches 1 2 4 8 16 32] [--reps 20] [--block 1] [--out results.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from diffdrr_b200 import DRR, _lib, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402

KERNELS = {"slab": 41, "pieces": 116, "brick": 42}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2, 4, 8, 16, 32])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--block", type=int, default=1, help="back-to-back launches of one kernel before the next kernel's block")
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.load()
    D, H = args.vol, args.det
    N = H * H
    vol = torch.rand(D, D, D, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H), renderer="siddon").to(dev)
    stream = torch.cuda.current_stream()
    p = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
    rows = []
    info = {"card": card(), "shape": f"{D}^3 -> {H}^2", "block": args.block}
    print(json.dumps(info), flush=True)
    for B in args.batches:
        rot, xyz = synthetic.make_poses(max(B, 2), seed=0)
        with torch.no_grad():
            src, tgt = drr.detector(convert(rot[:B].to(dev), xyz[:B].to(dev), parameterization="euler_angles", convention="ZXY"),
                                    None)
            raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
            src = drr.affine_inverse(src).reshape(B, 3).contiguous()
            tgt = drr.affine_inverse(tgt).contiguous()
        bufs = {k: (torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev)) for k in KERNELS}

        def launch(k):
            out, sens = bufs[k]
            _lib.check(lib.b200drr_siddon_fwd_sens_grid(p(vol), D, D, D, p(src), p(tgt), p(raylen), p(out), p(sens), B, H, H, 0.5,
                                                        1e-8, KERNELS[k], ctypes.c_void_p(stream.cuda_stream)), k)

        for k in KERNELS:  # warm-up (module load, allocator pool)
            launch(k)
            launch(k)
        times = {k: [] for k in KERNELS}
        for _ in range(args.reps):
            for k in KERNELS:
                for _ in range(args.block):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    launch(k)
                    e1.record(stream)
                    times[k].append((e0, e1))
        torch.cuda.synchronize()
        row = {"B": B}
        for k in KERNELS:
            us = np.array([a.elapsed_time(b) * 1e3 for a, b in times[k]])
            row[k] = {"median_us": float(np.median(us)), "min_us": float(us.min())}
        ref_out, ref_sens = bufs["slab"]
        for k in ("pieces", "brick"):
            out, sens = bufs[k]
            img = float((out - ref_out).abs().max() / ref_out.abs().max())
            comp = [float((sens[..., c] - ref_sens[..., c]).abs().max() / ref_sens[..., c].abs().max().clamp_min(1e-30))
                    for c in range(7)]
            row[k]["max_image_diff"] = img
            row[k]["max_sens_diff"] = max(comp)
        row["brick_speedup_vs_slab"] = row["slab"]["median_us"] / row["brick"]["median_us"]
        rows.append(row)
        print(json.dumps(row), flush=True)
        del bufs
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"info": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
