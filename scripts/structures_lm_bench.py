#!/usr/bin/env python
"""structures_lm_bench.py -- Levenberg-Marquardt over structures (StructuresLevenbergMarquardt, DESIGN.md 6g).

1. The block-sparse normal-equations kernel (b200drr_ncc_normal_structures) against the dense float64 torch statement (the
   composite Jacobian (B, H W, 6K) and Jz built explicitly, then A = Jz^T Jz), time and peak memory, on the J and footprints of
   a real render: 512^3 density (U[0,1) noise) with K in {2, 8, 24} vertebra-sized blocks (80 x 80 x 60 voxels; the layout of
   structures_bench.py), 256^2 detector, B in {1, 16} poses, small random motions, shared.  Pixel reads are counted from the
   footprints: the kernel reads each pair's overlap, the dense statement B H W pixels of every structure.
2. One LM step split into its parts: structures_jacobian (render + J), the normal equations, the solve, the trial render.
3. LM against Adam (the optimiser of test_gpu_structures.test_registration_recovers_two_structures) in steps and wall time to
   0.02 rad and 2 mm, on that test's problem (128^3, 96^2, three views) and on the same scene at 512^3, 256^2.
CUDA-event medians after warm-up; prints one JSON line; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, StructuresLevenbergMarquardt, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.structures import se3_exp, structures_jacobian  # noqa: E402
from structures_bench import _label_volume, _time  # noqa: E402

KW = dict(parameterization="euler_angles", convention="ZXY")


def dense_system(x, t, J, K, eps=1e-5):
    """The float64 torch statement of the global-NCC system with the dense composite Jacobian."""
    B, HW = x.shape[0], x[0].numel()
    Jd = J[:, :K].reshape(B, K, HW, 6).permute(0, 2, 1, 3).reshape(B, HW, 6 * K).double()
    x, t = x.double().flatten(1), t.double().flatten(1)
    mu, mt = x.mean(-1, keepdim=True), t.mean(-1, keepdim=True)
    s = ((x - mu).square().mean(-1, keepdim=True) + eps).sqrt()
    z, zt = (x - mu) / s, (t - mt) / ((t - mt).square().mean(-1, keepdim=True) + eps).sqrt()
    Jz = (Jd - Jd.mean(1, keepdim=True) - z[..., None] * (z[..., None] * Jd).mean(1, keepdim=True)) / s[..., None]
    return Jz.mT @ Jz / HW, (Jz.mT @ (z - zt)[..., None])[..., 0] / HW


def overlap_pixels(rects, K):
    r = rects[:, :K].long().cpu()
    w0, w1, h0, h1 = (r[..., i] for i in range(4))
    ow = (torch.minimum(w1[:, :, None], w1[:, None]) - torch.maximum(w0[:, :, None], w0[:, None]) + 1).clamp_min(0)
    oh = (torch.minimum(h1[:, :, None], h1[:, None]) - torch.maximum(h0[:, :, None], h0[:, None]) + 1).clamp_min(0)
    area = ow * oh
    return int(torch.triu(area).sum()), int(torch.triu(area > 0, diagonal=1).sum())


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def kernel_and_step(args, dev):
    D, H = args.vol, args.det
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    out = []
    for K in args.structures:
        drr = DRR(synthetic.make_subject(vol, mask=_label_volume(D, K)), **synthetic.detector_kwargs(H)).to(dev)
        labels = tuple(range(1, K + 1))
        g = torch.Generator().manual_seed(K)
        mot = lambda s: convert((torch.rand(K, 3, generator=g) * 2 - 1) * 0.05 * s, (torch.rand(K, 3, generator=g) * 2 - 1) * 5.0 * s,  # noqa: E731,E501
                                parameterization="euler_angles", convention="XYZ").matrix.to(dev)
        X, X_true = mot(1.0), mot(1.0)
        for B in args.batches:
            rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
            with torch.no_grad():
                target = drr.render_structures(rot, xyz, motions=X_true, labels=labels, **KW).sum(1, keepdim=True)
            lm = StructuresLevenbergMarquardt(drr, rot, xyz, X.clone(), labels, target, **KW)
            jac = lambda: structures_jacobian(drr, rot, xyz, motions=X, labels=labels, stop_grad=False,  # noqa: E731
                                              return_footprints=True, **KW)
            img, J, rects = jac()
            x = img.sum(1).contiguous()
            A, gv = lm.normal_equations(img, J, rects)
            Ad, gd = dense_system(x, target[:, 0], J, K)
            err = float((A - Ad).abs().max() / Ad.abs().max())
            ms = {k: [] for k in ("render_J", "normal_kernel", "normal_dense", "solve", "trial", "step")}
            Am = A.mean(0, keepdim=True)
            D_ = torch.diag_embed(torch.diagonal(Am, dim1=-2, dim2=-1))
            with torch.no_grad():
                for _ in range(args.rounds):
                    ms["render_J"].append(_time(jac, args.warmup, args.iters))
                    ms["normal_kernel"].append(_time(lambda: lm.normal_equations(img, J, rects), args.warmup, args.iters))
                    ms["normal_dense"].append(_time(lambda: dense_system(x, target[:, 0], J, K), 1, max(2, args.iters // 4)))
                    ms["solve"].append(_time(lambda: torch.linalg.solve_ex(Am + 1e-3 * D_, -gv.mean(0)[None, :, None]),
                                             args.warmup, args.iters))
                    ms["trial"].append(_time(lambda: drr.render_structures(rot, xyz, motions=X, labels=labels, **KW),
                                             args.warmup, args.iters))
                    ms["step"].append(_time(lm.step, args.warmup, args.iters))
            mem_k = peak(lambda: lm.normal_equations(img, J, rects))
            mem_d = peak(lambda: dense_system(x, target[:, 0], J, K))
            px, pairs = overlap_pixels(rects, K)
            out.append(dict(K=K, B=B, rel_err_kernel_vs_dense=err, ms={k: float(np.median(v)) for k, v in ms.items()},
                            peak_MiB_kernel=mem_k, peak_MiB_dense=mem_d, kernel_pair_pixels=px, overlapping_pairs=pairs,
                            dense_pixels=B * H * H * K))
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
        del drr
        torch.cuda.empty_cache()
    return out


def _about(w, t, centre):
    E = se3_exp(torch.cat([w, torch.zeros_like(w)], -1).double())
    R = E[..., :3, :3].to(w.dtype)
    top = torch.cat([R, (centre + t - (R @ centre[..., None])[..., 0])[..., None]], dim=-1)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], device=w.device).expand(*w.shape[:-1], 1, 4)
    return torch.cat([top, bottom], dim=-2)


def _errors(X, X_true, centre):
    M = X.double() @ torch.linalg.inv(X_true.double())
    cos = ((M[..., 0, 0] + M[..., 1, 1] + M[..., 2, 2] - 1) / 2).clamp(-1, 1)
    c = torch.cat([centre.double(), torch.ones_like(centre[..., :1]).double()], -1)[..., None]
    return float(torch.arccos(cos).max()), float(((X.double() - X_true.double()) @ c)[..., :3, 0].norm(dim=-1).max())


def convergence(n, H, dev, lm_cap=40, adam_cap=1000):
    """The scene of test_registration_recovers_two_structures at n^3 (blocks scaled with n), H^2 detector."""
    s = n / 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    rng = np.random.default_rng(3)
    lab = np.zeros((n, n, n), np.float32)
    lab[int(30 * s):int(58 * s), int(40 * s):int(70 * s), int(36 * s):int(60 * s)] = 1
    lab[int(70 * s):int(100 * s), int(60 * s):int(86 * s), int(66 * s):int(96 * s)] = 2
    vol = (vol + (lab > 0) * (1.0 + 0.5 * rng.random((n, n, n)))).astype(np.float32)
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(H)).to(dev)
    aff = torch.as_tensor(synthetic.make_affine(n), dtype=torch.float32)
    centre = torch.stack([torch.as_tensor(np.argwhere(lab == k).mean(0), dtype=torch.float32) for k in (1, 2)])
    centre = (centre @ aff[:3, :3].T + aff[:3, 3]).to(dev)
    rot = torch.tensor([[0.0, 0.0, 0.0], [math.pi / 2, 0.0, 0.0], [0.0, math.pi / 2, 0.0]], device=dev)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=dev).expand(3, 3).contiguous()
    w_true = torch.tensor([[0.05, -0.03, 0.04], [-0.04, 0.05, 0.03]], device=dev)
    t_true = torch.tensor([[8.0, -6.0, 5.0], [-7.0, 9.0, -4.0]], device=dev)
    X_true = _about(w_true, t_true, centre)
    with torch.no_grad():
        target = drr.render_structures(rot, xyz, motions=X_true, labels=(1, 2), **KW).sum(1, keepdim=True)
    res = {}
    # LM
    X = torch.eye(4, device=dev).expand(2, 4, 4).clone()
    lm = StructuresLevenbergMarquardt(drr, rot, xyz, X, (1, 2), target, **KW)
    torch.cuda.synchronize()
    t0, steps, errs = time.perf_counter(), None, None
    for k in range(1, lm_cap + 1):
        lm.step()
        errs = _errors(X, X_true, centre)
        if errs[0] < 0.02 and errs[1] < 2.0:
            steps = k
            break
    res["lm"] = dict(steps=steps, s=time.perf_counter() - t0, rad=errs[0], mm=errs[1])
    # Adam, as the test runs it
    w = torch.full((2, 3), 1e-4, device=dev, requires_grad=True)
    t = torch.zeros(2, 3, device=dev, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[w], lr=5e-3), dict(params=[t], lr=0.5)])
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.996)
    ncc = NormalizedCrossCorrelation2d()
    torch.cuda.synchronize()
    t0, steps = time.perf_counter(), None
    for k in range(1, adam_cap + 1):
        opt.zero_grad()
        img = drr.render_structures(rot, xyz, motions=_about(w, t, centre), labels=(1, 2), **KW).sum(1, keepdim=True)
        (-ncc(img, target).mean()).backward()
        opt.step()
        sched.step()
        with torch.no_grad():
            errs = _errors(_about(w, t, centre), X_true, centre)
        if errs[0] < 0.02 and errs[1] < 2.0:
            steps = k
            break
    res["adam"] = dict(steps=steps, s=time.perf_counter() - t0, rad=errs[0], mm=errs[1])
    print(json.dumps(dict(n=n, H=H, **res)), file=sys.stderr, flush=True)
    return dict(n=n, H=H, **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--structures", type=int, nargs="+", default=[2, 8, 24])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--skip-convergence", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    kernel = kernel_and_step(args, dev)
    conv = [] if args.skip_convergence else [convergence(128, 96, dev), convergence(args.vol, args.det, dev)]
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=args.vol, det=args.det, kernel_and_step=kernel, convergence=conv)))


if __name__ == "__main__":
    main()
