#!/usr/bin/env python
"""Kernel-selection sweep behind the defaults of renderers.py (_BRICK_FULL_GRID_MIN_LOAD) and csrc/siddon.cu
(small_batch_pieces, the slab height of the sensitivities walk): 512^3 fp32 CT -> 256^2 detector, the bench workload, at
1..32 poses.  Median CUDA-event time per launch (us) of every candidate decomposition, one JSON line per batch size.

    python scripts/tune_thresholds.py [--reps 15]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from diffdrr_b200 import DRR, _lib, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream  # noqa: E402

# b200drr_siddon_fwd_grid / _fwd_sens_grid variant ids (csrc/siddon.cu): 1xx = xx major-axis pieces, the rest slab heights
FWD = {"default": 0, "pieces12": 112, "pieces16": 116, "slab16": 46, "slab24": 47, "slab32": 15}
SENS = {"default": 0, "pieces8": 108, "pieces12": 112, "pieces16": 116, "slab16": 41, "slab24": 40, "slab32": 39, "slab48": 38,
        "slab64": 37, "slab96": 35, "unslabbed": 34}


def median_us(fn, reps):
    for _ in range(3):
        fn()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return round(1e3 * float(np.median([a.elapsed_time(b) for a, b in evs])), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.load()
    D, det = 512, 256
    N = det * det
    vol = torch.rand(D, D, D, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(det)).to(dev)
    print(json.dumps({"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True).stdout.strip()}), flush=True)
    for B in (1, 2, 4, 8, 16, 32):
        rot, xyz = synthetic.make_poses(B, seed=0)
        with torch.no_grad():
            src, tgt = drr.detector(convert(rot.to(dev), xyz.to(dev), parameterization="euler_angles", convention="ZXY"), None)
            raylen = (tgt - src).norm(dim=-1).unsqueeze(1).contiguous()
            src, tgt = drr.affine_inverse(src).reshape(B, 3).contiguous(), drr.affine_inverse(tgt).contiguous()
        out = torch.empty(B, N, device=dev)
        sens = torch.empty(B, N, 8, device=dev)
        ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(B, det, det), dtype=torch.uint8, device=dev)
        row = {"poses": B}

        def fwd(v):
            _lib.check(lib.b200drr_siddon_fwd_grid(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, det, det,
                                                   0.5, 1e-8, v, _stream()), "fwd_grid")

        def brick():
            _lib.check(lib.b200drr_siddon_fwd_brick(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), None, None, None, None,
                                                    _ptr(out), _ptr(ws), ws.numel(), B, det, det, 0.5, 1e-8, 0, _stream()), "brick")

        def sens_walk(v):
            _lib.check(lib.b200drr_siddon_fwd_sens_grid(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens),
                                                        B, det, det, 0.5, 1e-8, v, _stream()), "fwd_sens_grid")

        row["fwd_us"] = {name: median_us(lambda v=v: fwd(v), args.reps) for name, v in FWD.items()}
        row["fwd_us"]["brick"] = median_us(brick, args.reps)
        row["sens_us"] = {name: median_us(lambda v=v: sens_walk(v), args.reps) for name, v in SENS.items()}
        print(json.dumps(row), flush=True)
        del out, sens, ws


if __name__ == "__main__":
    main()
