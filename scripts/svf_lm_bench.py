#!/usr/bin/env python
"""svf_lm_bench.py -- the tangent of a squaring step and diffeomorphic Levenberg-Marquardt (DESIGN.md 6n) on the GPU.

Tangent step: b200drr_svf_square_jvp against b200drr_svf_square on g^3 lattices, g in --step-lattices, Bf in --step-batches, a
smooth velocity of ~g/8 voxels.  svf_bench.py's byte model: node reads and writes counted, the 8-corner reads (mostly L2 hits)
not: 32 B per node for the step, 48 B for the tangent without out, 64 B with it; `gbs_*` are those bytes over the time.

Costs: 512^3 density (U[0,1) noise), 256^2 detector, n_points = 500, a smooth ~5 mm world-mm velocity on a 32^3 and a 64^3 lattice
(shared by the poses), B in {1, 16}: one Gauss-Newton product and one step() at --cg-iters of DiffeomorphicLevenbergMarquardt,
and the same for DeformableLevenbergMarquardt on the same rays with the same field as a displacement.

Convergence (--convergence): test_gpu_svf.test_diffeomorphic_registration_lowers_ncc_and_stays_invertible's scene (phantom, four
views at 96^2, 8^3 velocity from zero towards a target rendered from a smooth 6 mm field, smoothness 1e-3, n_points = 250) at
128^3 and 512^3.  Adam (lr 0.3) on the velocity takes 200 steps; its E = mean(1 - NCC) + smoothness R(V) after them is the bar.
The velocity LM (steps = 10, cg_iters = 10) steps until its E is at or below the bar (a host-side check after every step, inside
the timed window), at most 40 steps.  Then both LMs run 20 steps from zero, on that target and on one rendered from twice the field,
and min det grad phi over the interior nodes is recorded for each (not asserted).  Wall times are host clocks around synchronised
work.

CUDA events, medians of --rounds alternated rounds.  Prints one JSON line with the card's name and power limit; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import svf_oracle as so  # noqa: E402
from deform_cases import smooth_field  # noqa: E402
from diffdrr_b200 import (DRR, DeformableLevenbergMarquardt, DiffeomorphicLevenbergMarquardt,  # noqa: E402
                          NormalizedCrossCorrelation2d, _lib, exp_velocity, synthetic)
from diffdrr_b200.registration import field_smoothness  # noqa: E402
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


def _alternate(fns, args, warmup=None, iters=None):
    t = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            t[k].append(_time(fn, args.warmup if warmup is None else warmup, args.iters if iters is None else iters))
    return {k: float(np.median(v)) for k, v in t.items()}


def tangent_step(args, dev):
    lib = _lib.load()
    results = []
    for g in args.step_lattices:
        for Bf in args.step_batches:
            u = torch.from_numpy(smooth_field(np.random.default_rng(g), Bf, (g, g, g), g / 8.0)).to(dev)
            t = torch.from_numpy(smooth_field(np.random.default_rng(g + 1), Bf, (g, g, g), 1.0)).to(dev)
            field = torch.nn.functional.pad(u.permute(0, 2, 3, 4, 1), (0, 1)).contiguous()
            tan = torch.nn.functional.pad(t.permute(0, 2, 3, 4, 1), (0, 1)).contiguous()
            out, tout, out2 = (torch.empty_like(field) for _ in range(3))
            dims = (4 * g, 4 * g, 4 * g)

            def step():
                lib.b200drr_svf_square(_ptr(field), _ptr(out), Bf, g, g, g, *dims, 1.0, _stream())

            def jvp(with_out):
                lib.b200drr_svf_square_jvp(_ptr(field), _ptr(tan), _ptr(tout), _ptr(out2) if with_out else None, Bf, g, g, g, *dims,
                                           1.0, _stream())

            step()
            jvp(True)
            torch.cuda.synchronize()
            ms = _alternate(dict(step=step, jvp=lambda: jvp(False), jvp_out=lambda: jvp(True)), args)
            nodes = Bf * g ** 3
            res = dict(lattice=g, Bf=Bf, ms=ms, out_equals_step=bool(torch.equal(out, out2)),
                       gbs_step=32.0 * nodes / (ms["step"] * 1e-3) / 1e9, gbs_jvp=48.0 * nodes / (ms["jvp"] * 1e-3) / 1e9,
                       gbs_jvp_out=64.0 * nodes / (ms["jvp_out"] * 1e-3) / 1e9)
            results.append(res)
            print(json.dumps(res), file=sys.stderr, flush=True)
            del field, tan, out, tout, out2
            torch.cuda.empty_cache()
    return results


def costs(args, dev):
    D, H, P = args.vol, args.det, args.n_points
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
    results = []
    for g in args.lattices:
        field = torch.from_numpy(smooth_field(np.random.default_rng(g), 1, (g, g, g), 5.0)[0]).to(dev)
        tan = torch.from_numpy(smooth_field(np.random.default_rng(g + 1), 1, (g, g, g), 1.0)[0]).to(dev)
        for B in args.batches:
            rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
            with torch.no_grad():
                target = drr.render_deformed(rot, xyz, field=torch.zeros_like(field), n_points=P, **KW)
            lms, prods = {}, {}
            for name, cls in (("svf", DiffeomorphicLevenbergMarquardt), ("disp", DeformableLevenbergMarquardt)):
                x = field.clone()
                lm = cls(drr, rot, xyz, x, target, cg_iters=args.cg_iters, n_points=P, **KW)
                lm.step()   # first image, damping (and the velocity's levels)
                _, Hprod = lm._model(lm._systems(x), lm._img)
                lms[name], prods[name] = lm, Hprod
            Ts = tan[None]

            def product(name):
                with torch.no_grad():
                    prods[name](Ts)

            ms = _alternate(dict(svf_product=lambda: product("svf"), disp_product=lambda: product("disp")), args)
            ms.update(_alternate(dict(svf_step=lms["svf"].step, disp_step=lms["disp"].step), args, warmup=1,
                                 iters=max(2, args.iters // 2)))
            res = dict(lattice=g, B=B, ms=ms, product_ratio=ms["svf_product"] / ms["disp_product"],
                       step_ratio=ms["svf_step"] / ms["disp_step"])
            results.append(res)
            print(json.dumps(res), file=sys.stderr, flush=True)
            del lms, prods
            torch.cuda.empty_cache()
    return results


def convergence(n, dev, adam_steps=200, max_lm=40, fixed=20):
    vol = synthetic.make_volume(n, "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(96), renderer="trilinear").to(dev)
    rot = torch.tensor([[0.0, 0.0, 0.0], [torch.pi / 2, 0.0, 0.0], [0.0, torch.pi / 2, 0.0], [torch.pi / 4, torch.pi / 4, 0.0]],
                       device=dev)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=dev).expand(4, 3).contiguous()
    grid = (8, 8, 8)
    U_true = torch.from_numpy(smooth_field(np.random.default_rng(21), 1, grid, 6.0)[0]).to(dev)
    kw = dict(n_points=250, **KW)
    ncc = NormalizedCrossCorrelation2d()
    lin = drr._affine_inverse.reshape(4, 4)[:3, :3].double()

    def target_of(U):
        with torch.no_grad():
            return drr.render_deformed(rot, xyz, field=U, **kw)

    def objective(V, target):
        with torch.no_grad():
            img = drr.render_deformed(rot, xyz, field=exp_velocity(drr, V), **kw)
            return float((1 - ncc(img, target)).mean() + 1e-3 * field_smoothness(V[None])[0])

    def min_det(u):
        return float(so.jacobian_det(torch.einsum("ij,jxyz->xyzi", lin, u.double())[None].cpu(), (n, n, n)).min())

    target = target_of(U_true)
    E0 = objective(torch.zeros_like(U_true), target)
    # warm both paths on a throw-away velocity
    v = torch.zeros_like(U_true, requires_grad=True)
    (1 - ncc(drr.render_deformed(rot, xyz, field=exp_velocity(drr, v), **kw), target)).mean().backward()
    DiffeomorphicLevenbergMarquardt(drr, rot, xyz, torch.zeros_like(U_true), target, smoothness=1e-3, cg_iters=10, **kw).step()
    torch.cuda.synchronize()

    V = torch.zeros_like(U_true, requires_grad=True)
    opt = torch.optim.Adam([V], lr=0.3)
    t0 = time.perf_counter()
    for _ in range(adam_steps):
        opt.zero_grad()
        loss = (1 - ncc(drr.render_deformed(rot, xyz, field=exp_velocity(drr, V), **kw), target)).mean()
        (loss + 1e-3 * field_smoothness(V[None]).sum()).backward()
        opt.step()
    torch.cuda.synchronize()
    adam_s = time.perf_counter() - t0
    bar = objective(V.detach(), target)

    W = torch.zeros_like(U_true)
    lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, W, target, steps=10, smoothness=1e-3, cg_iters=10, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    steps, lm_s, E = None, None, []
    for k in range(1, max_lm + 1):
        E.append(float(lm.step()))
        if E[-1] <= bar:
            steps, lm_s = k, time.perf_counter() - t0
            break
    res = dict(vol=n, E0=E0, adam_steps=adam_steps, adam_s=adam_s, adam_E=bar, adam_min_det=min_det(exp_velocity(drr, V.detach())),
               lm_steps=steps, lm_s=lm_s, lm_E=E)
    for scale in (1.0, 2.0):   # both LMs, `fixed` steps from zero
        tgt = target_of(scale * U_true)
        Vs, Us = torch.zeros_like(U_true), torch.zeros_like(U_true)
        svf_lm = DiffeomorphicLevenbergMarquardt(drr, rot, xyz, Vs, tgt, steps=10, smoothness=1e-3, cg_iters=10, **kw)
        disp_lm = DeformableLevenbergMarquardt(drr, rot, xyz, Us, tgt, smoothness=1e-3, cg_iters=10, **kw)
        for _ in range(fixed):
            svf_lm.step()
            disp_lm.step()
        with torch.no_grad():
            u = exp_velocity(drr, Vs)
            ncc_svf = float((1 - ncc(drr.render_deformed(rot, xyz, field=u, **kw), tgt)).mean())
            ncc_disp = float((1 - ncc(drr.render_deformed(rot, xyz, field=Us, **kw), tgt)).mean())
            ncc0 = float((1 - ncc(drr.render_deformed(rot, xyz, field=torch.zeros_like(Us), **kw), tgt)).mean())
        res[f"x{scale:g}"] = dict(ncc0=ncc0, svf_ncc=ncc_svf, disp_ncc=ncc_disp, svf_min_det=min_det(u), disp_min_det=min_det(Us),
                                  true_min_det=min_det(scale * U_true))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--step-lattices", type=int, nargs="+", default=[32, 64, 128])
    ap.add_argument("--step-batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--vol", type=int, default=512)
    ap.add_argument("--det", type=int, default=256)
    ap.add_argument("--n-points", type=int, default=500)
    ap.add_argument("--lattices", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--cg-iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--convergence", type=int, nargs="*", default=[128, 512])
    ap.add_argument("--no-costs", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("svf_lm_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    step = tangent_step(args, dev)
    results = [] if args.no_costs else costs(args, dev)
    conv = []
    for n in args.convergence:
        conv.append(convergence(n, dev))
        print(json.dumps(conv[-1]), file=sys.stderr, flush=True)
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=args.vol, det=args.det, n_points=args.n_points, cg_iters=args.cg_iters,
                          tangent_step=step, results=results, convergence=conv)))


if __name__ == "__main__":
    main()
