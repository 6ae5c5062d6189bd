#!/usr/bin/env python
"""polyrigid_lm_bench.py -- the blended-rigid motion Jacobian and its Levenberg-Marquardt (DESIGN.md 6j) against the render.

Part 1, kernels: polyrigid_bench.py's problem -- 512^3 density (U[0,1) noise), 256^2 detector, n_points = 500, K in {2, 8}
labelled blocks with a 64^3 weight lattice, B in {1, 16} poses, fp32 and bf16 densities.  Per configuration, alternated for
--rounds rounds, median of CUDA-event-timed calls after warm-up:
  jac          DRR.polyrigid_jacobian with footprints (one march: image, J (B, K, H, W, 6), rects)
  normal       PolyrigidLevenbergMarquardt.normal_equations on that output (b200drr_ncc_normal_structures, P = 6K)
  solve        the damped float64 solve of the (shared: view-averaged) system
  step         one PolyrigidLevenbergMarquardt.step() (shared motions)
  fwd / train  render_polyrigid forward (no_grad) -- the step's trial render is this call -- and forward + backward to the camera
               pose and the motions, on the same rays.
Byte model of the J kernel: J and img written (B K H W 24 + B H W 4 bytes) plus the forward's compulsory cell reads (32 B, 16 B
for a 16-bit density, per sample whose pulled-back point lies in the padded volume, counted by polyrigid_bench.torch_composition);
`jac_bytes_per_s` is that over jac time, and `hbm_share_jac` that over the H100 SXM data sheet's 3.35 TB/s.  L2-served cell
reuse and the weight lattice's reads are left out, as in polyrigid_bench.py.

Part 2, registration: test_gpu_polyrigid_lm.py's two-structure scene (128^3, three orthogonal views, 96^2, 32^3 lattice,
n_points = 250, shared motions) and the same scene at 512^3 (blocks and lattice scaled with it).  Steps and wall time (host clock
around synchronised steps, errors read after every step) to 0.02 rad / 2 mm from the identity, for PolyrigidLevenbergMarquardt and
for the Adam loop of test_gpu_polyrigid.test_registration_recovers_two_structures (500 steps at most).

Prints the card's name and power limit and one JSON line; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
sys.path.insert(0, _HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, PolyrigidLevenbergMarquardt, polyrigid_weights, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from polyrigid_bench import _label_volume, _time, torch_composition  # noqa: E402

KW = dict(parameterization="euler_angles", convention="ZXY")
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def kernels(args, dev):
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
        inside = {}
        for dtype in (torch.float32, torch.bfloat16):
            drr = DRR(synthetic.make_subject(vol, mask=lab), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
            W = polyrigid_weights(drr.mask, labels, grid=(g, g, g), sigma=6.0, spacing=spacing)
            if dtype != torch.float32:
                drr.density = drr.density.to(dtype)
            for B in args.batches:
                rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
                with torch.no_grad():
                    target = drr.render_polyrigid(rot, xyz, motions=torch.eye(4, device=dev).expand(K, 4, 4).contiguous(), weights=W,
                                                  n_points=P, **KW)
                    if B not in inside:
                        inside[B] = torch_composition(drr, rot, xyz, X, W, P)[1]
                lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X.clone(), W, target, n_points=P, **KW)
                img, J, rects = drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=P, return_footprints=True, **KW)
                A, gv = lm.normal_equations(img, J, rects)
                A, gv = A.mean(0, keepdim=True), gv.mean(0, keepdim=True)
                Dg = torch.diag_embed(torch.diagonal(A, dim1=-2, dim2=-1).clamp_min(1e-12))
                lam = torch.full((1,), 1e-3, dtype=torch.float64, device=dev)
                r, x, Xm = (t.clone().requires_grad_(True) for t in (rot, xyz, X))
                ops = dict(
                    jac=lambda: drr.polyrigid_jacobian(rot, xyz, motions=X, weights=W, n_points=P, return_footprints=True, **KW),
                    normal=lambda: lm.normal_equations(img, J, rects),
                    solve=lambda: torch.linalg.solve_ex(A + lam[:, None, None] * Dg, -gv.unsqueeze(-1)),
                    step=lm.step,
                    fwd=lambda: drr.render_polyrigid(rot, xyz, motions=X, weights=W, n_points=P, **KW),
                    train=lambda: drr.render_polyrigid(r, x, motions=Xm, weights=W, n_points=P, **KW).sum().backward())
                t = {k: [] for k in ops}
                for _ in range(args.rounds):
                    for k, fn in ops.items():
                        if k == "train":
                            t[k].append(_time(fn, args.warmup, args.iters))
                        else:
                            with torch.no_grad():
                                t[k].append(_time(fn, args.warmup, args.iters))
                ms = {k: float(np.median(v)) for k, v in t.items()}
                cell = 32 if dtype == torch.float32 else 16
                nbytes = B * K * H * H * 24 + B * H * H * 4 + inside[B] * cell
                res = dict(K=K, B=B, density=str(dtype).replace("torch.", ""), ms=ms, jac_over_fwd=ms["jac"] / ms["fwd"],
                           step_over_train=ms["step"] / ms["train"], samples_in_volume=inside[B], jac_model_bytes=nbytes,
                           jac_bytes_per_s=nbytes / (ms["jac"] * 1e-3), hbm_share_jac=nbytes / (ms["jac"] * 1e-3) / HBM_BYTES_PER_S)
                results.append(res)
                print(json.dumps(res), file=sys.stderr, flush=True)
            del drr
            torch.cuda.empty_cache()
    return results


def _about(w, t, centre):
    """x -> R (x - c) + c + t with R = exp(w^) (axis-angle w), per structure."""
    th = w.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    k = w / th
    Kx = torch.zeros(*w.shape[:-1], 3, 3, device=w.device, dtype=w.dtype)
    Kx[..., 0, 1], Kx[..., 0, 2], Kx[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    Kx = Kx - Kx.mT
    R = torch.eye(3, device=w.device, dtype=w.dtype) + th.sin()[..., None] * Kx + (1 - th.cos()[..., None]) * (Kx @ Kx)
    top = torch.cat([R, (centre + t - (R @ centre[..., None])[..., 0])[..., None]], dim=-1)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], device=w.device).expand(*w.shape[:-1], 1, 4)
    return torch.cat([top, bottom], dim=-2)


def _errors(X, X_true, centre):
    M = X.double() @ torch.linalg.inv(X_true.double())
    cos = ((M[..., 0, 0] + M[..., 1, 1] + M[..., 2, 2] - 1) / 2).clamp(-1, 1)
    c = torch.cat([centre.double(), torch.ones_like(centre[..., :1]).double()], -1)[..., None]
    disp = ((X.double() - X_true.double()) @ c)[..., :3, 0].norm(dim=-1)
    return float(torch.arccos(cos).max()), float(disp.max())


def registration(n, dev, lm_steps=40, adam_steps=500, rad=0.02, mm=2.0):
    s = n // 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    rng = np.random.default_rng(3)
    lab = np.zeros((n, n, n), np.float32)
    lab[30 * s:58 * s, 40 * s:70 * s, 36 * s:60 * s] = 1
    lab[70 * s:100 * s, 60 * s:86 * s, 66 * s:96 * s] = 2
    vol = (vol + (lab > 0) * (1.0 + 0.5 * rng.random((n, n, n), dtype=np.float32))).astype(np.float32)
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(96), renderer="trilinear").to(dev)
    del vol
    aff = torch.as_tensor(synthetic.make_affine(n), dtype=torch.float32)
    W = polyrigid_weights(drr.mask, (1, 2), grid=(32, 32, 32), sigma=6.0, spacing=tuple(float(aff[a, a]) for a in range(3)))
    centre = torch.stack([torch.as_tensor(np.argwhere(lab == k).mean(0), dtype=torch.float32) for k in (1, 2)])
    centre = (centre @ aff[:3, :3].T + aff[:3, 3]).to(dev)
    rot = torch.tensor([[0.0, 0.0, 0.0], [math.pi / 2, 0.0, 0.0], [0.0, math.pi / 2, 0.0]], device=dev)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=dev).expand(3, 3).contiguous()
    w_true = torch.tensor([[0.05, -0.03, 0.04], [-0.04, 0.05, 0.03]], device=dev)
    t_true = torch.tensor([[8.0, -6.0, 5.0], [-7.0, 9.0, -4.0]], device=dev)
    X_true = _about(w_true, t_true, centre)
    kw = dict(weights=W, n_points=250, **KW)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=X_true, **kw)
    out = dict(vol=n)
    # LM from the identity
    X = torch.eye(4, device=dev).expand(2, 4, 4).clone()
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=250, **KW)
    lm.step()   # warm-up: packs the lattice, loads the kernels
    X.copy_(torch.eye(4, device=dev).expand(2, 4, 4))
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=250, **KW)
    torch.cuda.synchronize()
    t0, hist = time.perf_counter(), []
    for k in range(1, lm_steps + 1):
        loss = float(lm.step())
        err = _errors(X, X_true, centre)
        hist.append((round(err[0], 5), round(err[1], 4), loss))
        if err[0] < rad and err[1] < mm:
            break
    out["lm"] = dict(steps=k, seconds=time.perf_counter() - t0, reached=err[0] < rad and err[1] < mm, rad=err[0], mm=err[1],
                     loss=loss, history=hist)
    # Adam from the identity
    w = torch.full((2, 3), 1e-4, device=dev, requires_grad=True)
    t = torch.zeros(2, 3, device=dev, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[w], lr=5e-3), dict(params=[t], lr=0.5)])
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.994)
    ncc = NormalizedCrossCorrelation2d()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(1, adam_steps + 1):
        opt.zero_grad()
        loss = -ncc(drr.render_polyrigid(rot, xyz, motions=_about(w, t, centre), **kw), target).mean()
        loss.backward()
        opt.step()
        sched.step()
        err = _errors(_about(w.detach(), t.detach(), centre), X_true, centre)
        if err[0] < rad and err[1] < mm:
            break
    out["adam"] = dict(steps=k, seconds=time.perf_counter() - t0, reached=err[0] < rad and err[1] < mm, rad=err[0], mm=err[1],
                       loss=1.0 + float(loss))
    print(json.dumps(out), file=sys.stderr, flush=True)
    return out


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
    ap.add_argument("--registration", type=int, nargs="*", default=[128, 512], help="volume sizes of the registration runs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("polyrigid_lm_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"gpu: {smi.stdout.strip()}", file=sys.stderr, flush=True)
    results = kernels(args, dev) if args.structures else []
    reg = [registration(n, dev) for n in args.registration]
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=args.vol, det=args.det, n_points=args.n_points, lattice=args.lattice,
                          results=results, registration=reg)))


if __name__ == "__main__":
    main()
