#!/usr/bin/env python
"""log_euclidean_lm_bench.py -- the log-Euclidean blended-rigid motion Jacobian and its Levenberg-Marquardt (DESIGN.md 6p) on the GPU.

Costs: 512^3 density (U[0,1) noise), 256^2 detector, n_points = 500, a 64^3 weight lattice of K smooth bumps, K in --ks, B in
--batches, shared motions (Bm = 1) and, with --per-pose, per-pose motions (Bm = B), fp32 and bf16 densities, steps = 10.
  fused:   DRR.polyrigid_jacobian(blend="log_euclidean"), split into `chain` (the velocity, its 6K tangents and the primal and
           tangent squarings) and `march` (b200drr_deform_jac alone);
  compose: the same Jacobian column by column from existing pieces, 6K x (10 b200drr_svf_square_jvp + 1 b200drr_deform_jvp);
  step:    one PolyrigidLevenbergMarquardt(blend="log_euclidean").step(); fwd / fwd_bwd: render_polyrigid(blend="log_euclidean")
           and its backward to the motions.
Byte model (compulsory traffic only; corner re-reads, mostly L2 hits, not counted): a tangent squaring reads the level and the P
tangents and writes P tangents, Bm g^3 (16 + 32 P) B; the march writes J and the image, B H W (24 K + 4) B, and reads the density
once, 4 or 2 B per voxel.  gbs_* are those bytes over the measured times.

Convergence (--convergence): test_gpu_log_euclidean_lm's two-structure scene (128^3, three views at 96^2, 32^3 lattice, target
rendered by the log-Euclidean blend, n_points = 250).  Adam (test_gpu_svf.test_registration_recovers_two_structures' schedule) and
the LM step from the identity until both errors are below 0.02 rad and 2 mm (host-side check after every step, inside the timed
window; Adam at most 500 steps, LM at most 40).  Wall times are host clocks around synchronised work.

CUDA events, medians of --rounds alternated rounds.  Prints one JSON line with the card's name and power limit; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, PolyrigidLevenbergMarquardt, polyrigid_weights, svf, synthetic  # noqa: E402
from diffdrr_b200 import polyrigid as pr  # noqa: E402
from diffdrr_b200.deform import _marches, field_jvp  # noqa: E402
from diffdrr_b200.structures import se3_exp, twist_matrix  # noqa: E402

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


def _alternate(fns, args):
    t = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            t[k].append(_time(fn, args.warmup, args.iters))
    return {k: float(np.median(v)) for k, v in t.items()}


def _weights(K, g, dev, seed=0):
    rng = np.random.default_rng(seed)
    x = np.stack(np.meshgrid(*[(np.arange(g) + 0.5) / g] * 3, indexing="ij"), -1)
    w = np.stack([np.exp(-((x - rng.uniform(0.2, 0.8, 3)) ** 2).sum(-1) / 0.02) for _ in range(K)])
    w[w < 1e-3] = 0.0
    return torch.from_numpy((w / np.maximum(w.sum(0), 1.0)).astype(np.float32)).to(dev)


def costs(args, dev):
    vol = torch.from_numpy(synthetic.make_volume(args.vol, "rand", seed=0))
    results = []
    for dtype in (torch.float32, torch.bfloat16):
        drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(args.det), renderer="trilinear").to(dev)
        drr.density = drr.density.to(dtype)
        dims = tuple(drr.density.shape)
        for K in args.ks:
            W = _weights(K, args.lattice, dev)
            pivots = pr.polyrigid_pivots(drr, W)
            for B in args.batches:
                for per_pose in ((False, True) if args.per_pose else (False,)):
                    rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
                    g = torch.Generator().manual_seed(K)
                    xi = ((torch.rand(*((B,) if per_pose else ()), K, 6, generator=g) * 2 - 1) *
                          torch.tensor([0.08] * 3 + [8.0] * 3)).to(dev)
                    X = se3_exp(xi).float()
                    kw = dict(motions=X, weights=W, n_points=args.n_points, blend="log_euclidean", steps=args.steps, **KW)
                    with torch.no_grad():
                        target = drr.render_polyrigid(rot, xyz, **{**kw, "motions": se3_exp(0.5 * xi).float()})
                    source, [(tgt, lens, arange, grid)] = _marches(drr, (rot, xyz), B, KW["parameterization"], KW["convention"],
                                                                   False, None, None, None)
                    packed = drr.renderer._packed_volume(drr.density)
                    state = {}

                    def chain():
                        with torch.no_grad():
                            levels, U = svf.square_chain(svf.polyrigid_velocity(drr, X, W), args.steps, dims)
                            T = svf.square_chain_tangents(levels, svf.velocity_tangents(drr, X, W, pivots), dims)
                        state.update(U=U, T=T)

                    chain()
                    Bm = state["U"].shape[0]
                    img = torch.empty(B, args.det ** 2, device=dev)
                    J = torch.empty(B, K, args.det ** 2, 6, device=dev)
                    rects = torch.empty(B, K, 4, dtype=torch.int32, device=dev)
                    fn, head, name, (src, tg, rl), _ = pr._launch_args("b200drr_deform_jac", drr.density, packed, source, tgt, lens,
                                                                       grid)

                    def march():
                        U, T = state["U"], state["T"]
                        pr._lib.check(fn(*head, *dims, pr._ptr(src), pr._ptr(tg), pr._ptr(rl), pr._ptr(U), Bm, *U.shape[1:4],
                                         pr._ptr(T), 6 * K, K, pr._ptr(img), pr._ptr(J), pr._ptr(rects), B, args.det, args.det, 0.5,
                                         1e-8, args.n_points, pr._ptr(arange), pr._stream()), name)

                    def fused():
                        drr.polyrigid_jacobian(rot, xyz, **kw)

                    def compose():
                        with torch.no_grad():
                            v = svf.polyrigid_velocity(drr, X, W)
                            T0 = svf.velocity_tangents(drr, X, W, pivots)
                            for p in range(6 * K):
                                U, Tp = svf.square_chain_jvp([v], T0[..., p, :].contiguous(), dims, steps=args.steps)
                                field_jvp(drr, packed, source, tgt, lens, U, Tp, arange, args.n_points, grid)

                    Xp = X.clone()
                    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, Xp, W, target, n_points=args.n_points, blend="log_euclidean",
                                                     steps=args.steps, **KW)

                    def step():
                        Xp.copy_(X)
                        lm.step()

                    def fwd():
                        with torch.no_grad():
                            drr.render_polyrigid(rot, xyz, **kw)

                    Xg = X.clone().requires_grad_(True)

                    def fwd_bwd():
                        drr.render_polyrigid(rot, xyz, **{**kw, "motions": Xg}).sum().backward()

                    fns = dict(chain=chain, march=march, fused=fused, step=step, fwd=fwd, fwd_bwd=fwd_bwd)
                    if not args.no_compose:
                        fns["compose"] = compose
                    ms = _alternate(fns, args)
                    P = 6 * K
                    chain_bytes = args.steps * Bm * args.lattice ** 3 * (16 + 32 * P)
                    march_bytes = B * args.det ** 2 * (24 * K + 4) + drr.density.numel() * drr.density.element_size()
                    res = dict(dtype=str(dtype).split(".")[-1], K=K, B=B, Bm=Bm, ms=ms,
                               tangent_level_mb=Bm * args.lattice ** 3 * P * 16 / 1e6,
                               compose_over_fused=(ms["compose"] / ms["fused"]) if "compose" in ms else None,
                               gbs_chain=chain_bytes / (ms["chain"] * 1e-3) / 1e9, gbs_march=march_bytes / (ms["march"] * 1e-3) / 1e9)
                    results.append(res)
                    print(json.dumps(res), file=sys.stderr, flush=True)
                    del state, J, lm
                    torch.cuda.empty_cache()
    return results


def _about(w, t, centre):
    R = torch.linalg.matrix_exp(twist_matrix(torch.cat([w, torch.zeros_like(w)], -1)))[..., :3, :3]
    top = torch.cat([R, (centre + t - (R @ centre[..., None])[..., 0])[..., None]], dim=-1)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], device=w.device).expand(*w.shape[:-1], 1, 4)
    return torch.cat([top, bottom], dim=-2)


def _errors(X, X_true, centre):
    M = X.double() @ torch.linalg.inv(X_true.double())
    cos = ((M[..., 0, 0] + M[..., 1, 1] + M[..., 2, 2] - 1) / 2).clamp(-1, 1)
    c = torch.cat([centre.double(), torch.ones_like(centre[..., :1]).double()], -1)[..., None]
    return float(torch.arccos(cos).max()), float(((X.double() - X_true.double()) @ c)[..., :3, 0].norm(dim=-1).max())


def convergence(dev):
    n = 128
    vol = synthetic.make_volume(n, "phantom", seed=11)
    rng = np.random.default_rng(3)
    lab = np.zeros((n, n, n), np.float32)
    lab[30:58, 40:70, 36:60] = 1
    lab[70:100, 60:86, 66:96] = 2
    vol = (vol + (lab > 0) * (1.0 + 0.5 * rng.random((n, n, n)))).astype(np.float32)
    drr = DRR(synthetic.make_subject(vol, mask=torch.from_numpy(lab)), **synthetic.detector_kwargs(96), renderer="trilinear").to(dev)
    aff = torch.as_tensor(synthetic.make_affine(n), dtype=torch.float32)
    W = polyrigid_weights(drr.mask, (1, 2), grid=(32, 32, 32), sigma=6.0, spacing=tuple(float(aff[a, a]) for a in range(3)))
    centre = torch.stack([torch.as_tensor(np.argwhere(lab == k).mean(0), dtype=torch.float32) for k in (1, 2)])
    centre = (centre @ aff[:3, :3].T + aff[:3, 3]).to(dev)
    rot = torch.tensor([[0.0, 0.0, 0.0], [math.pi / 2, 0.0, 0.0], [0.0, math.pi / 2, 0.0]], device=dev)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=dev).expand(3, 3).contiguous()
    w_true = torch.tensor([[0.05, -0.03, 0.04], [-0.04, 0.05, 0.03]], device=dev)
    t_true = torch.tensor([[8.0, -6.0, 5.0], [-7.0, 9.0, -4.0]], device=dev)
    X_true = _about(w_true, t_true, centre)
    kw = dict(weights=W, n_points=250, blend="log_euclidean", **KW)
    with torch.no_grad():
        target = drr.render_polyrigid(rot, xyz, motions=X_true, **kw)
    out = {}
    # Adam
    w = torch.full((2, 3), 1e-4, device=dev, requires_grad=True)
    t = torch.zeros(2, 3, device=dev, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[w], lr=5e-3), dict(params=[t], lr=0.5)])
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.994)
    ncc = NormalizedCrossCorrelation2d()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    k = 0
    for k in range(1, 501):
        opt.zero_grad()
        (-ncc(drr.render_polyrigid(rot, xyz, motions=_about(w, t, centre), **kw), target).mean()).backward()
        opt.step()
        sched.step()
        er, et = _errors(_about(w.detach(), t.detach(), centre), X_true, centre)
        if er < 0.02 and et < 2.0:
            break
    torch.cuda.synchronize()
    out["adam"] = dict(steps=k, seconds=time.perf_counter() - t0, rad=er, mm=et)
    # LM
    X = torch.eye(4, device=dev).expand(2, 4, 4).clone()
    lm = PolyrigidLevenbergMarquardt(drr, rot, xyz, X, W, target, n_points=250, blend="log_euclidean", steps=10, **KW)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(1, 41):
        lm.step()
        er, et = _errors(X, X_true, centre)
        if er < 0.02 and et < 2.0:
            break
    torch.cuda.synchronize()
    out["lm"] = dict(steps=k, seconds=time.perf_counter() - t0, rad=er, mm=et)
    print(json.dumps(out), file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--n-points", type=int, default=500)
    ap.add_argument("--lattice", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--ks", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--per-pose", action="store_true", help="also per-pose motions (Bm = B)")
    ap.add_argument("--no-compose", action="store_true", help="skip the column-by-column composition")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--convergence", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = dict(card=smi.stdout.strip(), costs=costs(args, dev))
    if args.convergence:
        out["convergence"] = convergence(dev)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
