#!/usr/bin/env python
"""deform_lm_bench.py -- the field-tangent march and deformable Levenberg-Marquardt (DESIGN.md 6k) on the GPU.

Costs: 512^3 density (U[0,1) noise), 256^2 detector, n_points = 500, a smooth ~5 mm world-mm field on a 32^3 and a 64^3 lattice
(shared by the poses), B in {1, 16}, fp32 and bf16 densities.  Per configuration, alternated for --rounds rounds, median of
CUDA-event-timed calls after warm-up:
  fwd        b200drr_deform_fwd on the module's rays (the forward of render_deformed, rays precomputed);
  jvp        b200drr_deform_jvp on the same rays with the image (both outputs); jvp_only without it (img = NULL);
  gn_product one Gauss-Newton product H v of DeformableLevenbergMarquardt: a tangent march, the NCC Jacobian twice, a field
             scatter (b200drr_deform_bwd with only g_field) and the smoothness term;
  lm_step    one DeformableLevenbergMarquardt.step() at --cg-iters: a scatter for g, cg_iters products, one trial render_deformed;
  adam_step  one Adam step: render_deformed forward + backward to the field (camera fixed) + the optimizer update.
Byte model of the tangent march: 32 B (16 B for a 16-bit density) per sample whose pulled-back point lies in the zero-padded volume
(one packed-corner cell; counted with deform_bench.py's torch composition), the field and the tangent lattices once, jv and img
written; `hbm_share_jvp` is those bytes over the jvp time over the H100 SXM data sheet's 3.35 TB/s -- a statement about that byte
bound, not achieved DRAM bandwidth.

Convergence (--convergence): test_gpu_deform.test_registration_lowers_ncc_and_field_error's scene (phantom, four views at 96^2,
8^3 field from zero towards a target rendered from a smooth 6 mm field, smoothness 1e-3, n_points = 250) at 128^3 and 512^3.
Adam (lr 0.3) takes 300 steps; its objective E = mean(1 - NCC) + smoothness R after them is the bar.  LM (cg_iters = 10) steps
until its E is at or below the bar (a host-side check after every step, inside the timed window), at most 40 steps.  Wall times
are host clocks around synchronised work.

Prints one JSON line with the card's name and power limit; writes nothing.
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from deform_bench import torch_composition  # noqa: E402
from deform_cases import smooth_field  # noqa: E402
from diffdrr_b200 import DRR, DeformableLevenbergMarquardt, NormalizedCrossCorrelation2d, synthetic  # noqa: E402
from diffdrr_b200 import deform as dm  # noqa: E402
from diffdrr_b200.registration import field_smoothness  # noqa: E402

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


def costs(args, dev):
    D, H, P = args.vol, args.det, args.n_points
    vol = torch.from_numpy(synthetic.make_volume(D, "rand", seed=0))
    results = []
    for g in args.lattices:
        field = torch.from_numpy(smooth_field(np.random.default_rng(g), 1, (g, g, g), 5.0)[0]).to(dev)
        tan = torch.from_numpy(smooth_field(np.random.default_rng(g + 1), 1, (g, g, g), 1.0)[0]).to(dev)
        for dtype in (torch.float32, torch.bfloat16):
            drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(H), renderer="trilinear").to(dev)
            if dtype != torch.float32:
                drr.density = drr.density.to(dtype)
            r = drr.renderer
            for B in args.batches:
                rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=0))
                with torch.no_grad():
                    source, marches = dm._marches(drr, (rot, xyz), B, "euler_angles", "ZXY", False, None, None, None)
                    tgt, lens, arange, grid = marches[0]
                    U, T = dm.voxel_field(drr, field), dm.voxel_field(drr, tan)
                    packed = r._packed_volume(drr.density)
                    target = drr.render_deformed(rot, xyz, field=torch.zeros_like(field), n_points=P, **KW)
                img = torch.empty(B, H * H, device=dev)

                def fwd():
                    with torch.no_grad():
                        dm._DeformFunction.apply(drr.density, packed, source, tgt, lens, U, arange, float(r.voxel_shift),
                                                 float(r.eps), P, grid)

                def jvp(with_img=True):
                    return dm.field_jvp(drr, packed, source, tgt, lens, U, T, arange, P, grid, img=img if with_img else None)

                lm_field = field.clone()
                lm = DeformableLevenbergMarquardt(drr, rot, xyz, lm_field, target, cg_iters=args.cg_iters, n_points=P, **KW)
                lm.step()   # first image and damping
                _, Hprod = lm._model(lm._systems(lm_field), lm._img)
                Ts = tan[None]

                u_adam = field.clone().requires_grad_(True)
                opt = torch.optim.Adam([u_adam], lr=0.1)
                ncc = NormalizedCrossCorrelation2d()

                def adam():
                    opt.zero_grad()
                    loss = (1 - ncc(drr.render_deformed(rot, xyz, field=u_adam, n_points=P, **KW), target)).mean()
                    (loss + 1e-3 * field_smoothness(u_adam[None]).sum()).backward()
                    opt.step()

                res = dict(lattice=g, B=B, density=str(dtype).replace("torch.", ""))
                with torch.no_grad():
                    out = torch.empty(B, H * H, device=dev)
                    want = dm._DeformFunction.apply(drr.density, packed, source, tgt, lens, U, arange, float(r.voxel_shift),
                                                    float(r.eps), P, grid).reshape(B, -1)
                    jvp()
                    res["img_equals_fwd"] = bool(torch.equal(img, want))
                    _, inside = torch_composition(drr, rot, xyz, field, P)
                    del out
                t = {k: [] for k in ("fwd", "jvp", "jvp_only", "gn_product", "lm_step", "adam_step")}
                for _ in range(args.rounds):
                    t["fwd"].append(_time(fwd, args.warmup, args.iters))
                    t["jvp"].append(_time(jvp, args.warmup, args.iters))
                    t["jvp_only"].append(_time(lambda: jvp(False), args.warmup, args.iters))
                    with torch.no_grad():
                        t["gn_product"].append(_time(lambda: Hprod(Ts), args.warmup, args.iters))
                    t["lm_step"].append(_time(lm.step, 1, max(2, args.iters // 2)))
                    t["adam_step"].append(_time(adam, args.warmup, args.iters))
                res["ms"] = {k: float(np.median(v)) for k, v in t.items()}
                res["jvp_over_fwd"] = res["ms"]["jvp"] / res["ms"]["fwd"]
                cell = 32 if dtype == torch.float32 else 16
                res["samples_in_volume"] = inside
                res["model_bytes_jvp"] = inside * cell + 2 * g ** 3 * 16 + 2 * B * H * H * 4
                res["hbm_share_jvp"] = res["model_bytes_jvp"] / (res["ms"]["jvp"] * 1e-3) / HBM_BYTES_PER_S
                results.append(res)
                print(json.dumps(res), file=sys.stderr, flush=True)
                del lm, opt, u_adam, Hprod
            del drr
            torch.cuda.empty_cache()
    return results


def convergence(n, dev, adam_steps=300, max_lm=40):
    vol = synthetic.make_volume(n, "phantom", seed=11)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(96), renderer="trilinear").to(dev)
    rot = torch.tensor([[0.0, 0.0, 0.0], [torch.pi / 2, 0.0, 0.0], [0.0, torch.pi / 2, 0.0], [torch.pi / 4, torch.pi / 4, 0.0]],
                       device=dev)
    xyz = torch.tensor([[0.0, 850.0, 0.0]], device=dev).expand(4, 3).contiguous()
    grid = (8, 8, 8)
    U_true = torch.from_numpy(smooth_field(np.random.default_rng(21), 1, grid, 6.0)[0]).to(dev)
    kw = dict(n_points=250, **KW)
    ncc = NormalizedCrossCorrelation2d()
    with torch.no_grad():
        target = drr.render_deformed(rot, xyz, field=U_true, **kw)
    idx = [((np.arange(g) + 0.5) * n / g - 0.5).round().astype(int) for g in grid]
    body = torch.from_numpy(vol[np.ix_(*idx)] > 0.1 * vol.max()).to(dev)

    def objective(U):
        with torch.no_grad():
            return float((1 - ncc(drr.render_deformed(rot, xyz, field=U, **kw), target)).mean() + 1e-3 * field_smoothness(U[None])[0])

    def rms(U):
        return float(((U - U_true) ** 2).sum(0)[body].mean().sqrt())

    E0 = objective(torch.zeros_like(U_true))
    # warm both paths on a throw-away field
    u = torch.zeros_like(U_true, requires_grad=True)
    (1 - ncc(drr.render_deformed(rot, xyz, field=u, **kw), target)).mean().backward()
    DeformableLevenbergMarquardt(drr, rot, xyz, torch.zeros_like(U_true), target, smoothness=1e-3, cg_iters=10, **kw).step()
    torch.cuda.synchronize()

    U = torch.zeros_like(U_true, requires_grad=True)
    opt = torch.optim.Adam([U], lr=0.3)
    t0 = time.perf_counter()
    for _ in range(adam_steps):
        opt.zero_grad()
        loss = (1 - ncc(drr.render_deformed(rot, xyz, field=U, **kw), target)).mean()
        (loss + 1e-3 * field_smoothness(U[None]).sum()).backward()
        opt.step()
    torch.cuda.synchronize()
    adam_s = time.perf_counter() - t0
    bar, adam_rms = objective(U.detach()), rms(U.detach())

    V = torch.zeros_like(U_true)
    lm = DeformableLevenbergMarquardt(drr, rot, xyz, V, target, smoothness=1e-3, cg_iters=10, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    steps, lm_s, E = None, None, []
    for k in range(1, max_lm + 1):
        E.append(float(lm.step()))
        if E[-1] <= bar:
            steps, lm_s = k, time.perf_counter() - t0
            break
    return dict(vol=n, E0=E0, adam_steps=adam_steps, adam_s=adam_s, adam_E=bar, adam_rms_mm=adam_rms, lm_steps=steps, lm_s=lm_s,
                lm_E=E, lm_rms_mm=rms(V), rms0_mm=rms(torch.zeros_like(U_true)))


def main():
    ap = argparse.ArgumentParser()
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
        raise SystemExit("deform_lm_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    results = [] if args.no_costs else costs(args, dev)
    conv = []
    for n in args.convergence:
        conv.append(convergence(n, dev))
        print(json.dumps(conv[-1]), file=sys.stderr, flush=True)
    print(json.dumps(dict(gpu=smi.stdout.strip(), vol=args.vol, det=args.det, n_points=args.n_points, cg_iters=args.cg_iters,
                          results=results, convergence=conv)))


if __name__ == "__main__":
    main()
