#!/usr/bin/env python
"""Batches of one or two poses (registration loop, single-DRR inference), 512^3 (VOL) -> 256^2 (DET): the Siddon forward and
forward-with-sensitivities kernels with every ray cut into K pieces along its own major axis (variants 100+K of
b200drr_siddon_fwd_grid / b200drr_siddon_fwd_sens_grid) against the un-cut kernels, parity against each other.  `--loop` runs
the registration loop of BASELINE config 5 (bench.py's set-up) with the fused NCC kernels and torch's fused Adam, one CUDA graph
per step."""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from diffdrr_b200 import DRR, NormalizedCrossCorrelation2d, Registration, _lib, synthetic  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream, siddon_visits  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--loop", action="store_true")
ap.add_argument("--big", action="store_true", help="batches of 8 / 16 poses: major-axis pieces against the slab-major and brick kernels")
ap.add_argument("--trace", action="store_true", help="with --loop: kernel names x counts of one eager step (torch.profiler)")
ap.add_argument("--pieces", default="1,2,3,4,6,8,12,16,24,32")
ap.add_argument("--batches", default="1,2,3,4")
args = ap.parse_args()
D, H = int(os.environ.get("VOL", 512)), int(os.environ.get("DET", 256))
dev = torch.device("cuda:0")
lib = _lib.load()
peak = bench.hbm_peak()[0]


def kernels():
    vol = torch.as_tensor(synthetic.make_volume(D, "rand", seed=0)).to(dev)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H)).to(dev)
    N = H * H
    for B in [int(b) for b in args.batches.split(",")]:
        rot, xyz = synthetic.make_poses(max(B, 2), seed=0)
        s, t, l = bench._device_rays(drr, rot[:B], xyz[:B], dev)
        visits = int(siddon_visits((D, D, D), s, t).sum().item())
        out, sens = torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev)
        ref_out, ref_sens = torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev)

        def fwd(variant, o=out):
            _lib.check(lib.b200drr_siddon_fwd_grid(_ptr(vol), D, D, D, _ptr(s), _ptr(t), _ptr(l), _ptr(o), B, H, H, 0.5, 1e-8,
                                                   variant, _stream()), "fwd_grid")

        def sns(variant, o=out, q=sens):
            _lib.check(lib.b200drr_siddon_fwd_sens_grid(_ptr(vol), D, D, D, _ptr(s), _ptr(t), _ptr(l), _ptr(o), _ptr(q), B, H, H,
                                                        0.5, 1e-8, variant, _stream()), "fwd_sens_grid")

        fwd(15, ref_out)      # 32-plane slabs
        t_f0 = float(np.median(bench._time_events(lambda: fwd(15), 7, warmup=2)))
        sns(34, ref_out, ref_sens)   # one thread per ray (a single 512-plane slab): the pre-existing choice for B <= 2
        t_s0 = float(np.median(bench._time_events(lambda: sns(34), 7, warmup=2)))
        t_s48 = float(np.median(bench._time_events(lambda: sns(35), 7, warmup=2)))
        print(f"{D}^3 -> {H}^2 x {B} poses ({visits / (B * N):.0f} visits/ray): forward 32-plane slabs {t_f0 * 1e3:7.1f} us | "
              f"sens one thread per ray {t_s0 * 1e3:7.1f} us | sens 96-plane slabs {t_s48 * 1e3:7.1f} us", flush=True)
        for K in [int(k) for k in args.pieces.split(",")]:
            fwd(100 + K)
            ef = float((out - ref_out).abs().max() / ref_out.abs().max())
            tf = float(np.median(bench._time_events(lambda: fwd(100 + K), 7, warmup=2)))
            sns(100 + K)
            es = float((out - ref_out).abs().max() / ref_out.abs().max())
            eq = float((sens - ref_sens).abs().max() / ref_sens.abs().max())
            ts = float(np.median(bench._time_events(lambda: sns(100 + K), 7, warmup=2)))
            print(f"  K = {K:2d}: forward {tf * 1e3:7.1f} us ({4 * visits / tf * 1e-6 / peak * 100:4.1f} %) | "
                  f"sens {ts * 1e3:7.1f} us ({4 * visits / ts * 1e-6 / peak * 100:4.1f} % of HBM peak on visited voxels)   "
                  f"maxdiff/max fwd {ef:.1e} sens-img {es:.1e} sens {eq:.1e}", flush=True)
        fwd(0)
        sns(0)
        t_fd = float(np.median(bench._time_events(lambda: fwd(0), 7, warmup=2)))
        t_sd = float(np.median(bench._time_events(lambda: sns(0), 7, warmup=2)))
        print(f"  default (variant 0): forward {t_fd * 1e3:7.1f} us | sens {t_sd * 1e3:7.1f} us", flush=True)


def loop():
    x = torch.linspace(-1, 1, D, device=dev)
    X, Y, Z = x[:, None, None], x[None, :, None], x[None, None, :]
    smooth = torch.exp(-((X - 0.2) ** 2 + (Y + 0.1) ** 2 + (Z - 0.05) ** 2) / 0.18)
    smooth += 0.6 * torch.exp(-((X + 0.35) ** 2 + (Y - 0.3) ** 2 + (Z + 0.25) ** 2) / 0.05)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H), renderer="siddon", stop_gradients_through_grid_sample=True).to(dev)
    drr.density = smooth.contiguous()
    true_rot, true_xyz = torch.tensor([[0.0, 0.0, 0.0]], device=dev), torch.tensor([[0.0, 850.0, 0.0]], device=dev)
    with torch.no_grad():
        target = drr(true_rot, true_xyz, parameterization="euler_angles", convention="ZXY")
    for fused_ncc in (True, False):
        for fused_adam in (True, False):
            reg = Registration(drr, (true_rot + torch.tensor([[0.15, -0.1, 0.08]], device=dev)).clone(),
                               (true_xyz + torch.tensor([[12.0, -25.0, 9.0]], device=dev)).clone(), "euler_angles", "ZXY").to(dev)
            ncc = NormalizedCrossCorrelation2d()
            if not fused_ncc:
                ncc.fused_ok = lambda a, b: False
            groups = [{"params": [reg.rotation], "lr": 5e-3}, {"params": [reg.translation], "lr": 5e-1}]
            opt = torch.optim.Adam(groups, capturable=True, fused=True) if fused_adam else torch.optim.Adam(groups, capturable=True)

            def step():
                opt.zero_grad(set_to_none=False)
                loss = 1.0 - ncc(target, reg()).mean()
                loss.backward()
                opt.step()
                return loss

            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(5):
                    step()
                if args.trace and fused_ncc and fused_adam:  # which kernels one eager step launches (names x count)
                    from torch.profiler import ProfilerActivity, profile
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(4):
                            step()
                        torch.cuda.synchronize()
                    rows = sorted(((e.key, e.count, e.device_time_total) for e in prof.key_averages()), key=lambda r: -r[2])
                    print(f"launches per step: {sum(r[1] for r in rows) / 4:.1f}")
                    for k, c, tt in rows:
                        print(f"   {c / 4:5.1f} x {tt / max(c, 1):8.1f} us  {k[:110]}")
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
            n_it = 1000
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n_it):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            with torch.no_grad():
                final = float(1.0 - ncc(target, reg()).mean())
            print(f"registration loop {D}^3 -> {H}^2, fused NCC {fused_ncc}, fused Adam {fused_adam}: "
                  f"{n_it / (ms * 1e-3):8.1f} it/s ({ms / n_it * 1e3:6.1f} us/it)  "
                  f"1-ncc {final:.2e} rot err {float((reg.rotation.detach() - true_rot).abs().max()):.4f} "
                  f"xyz err {float((reg.translation.detach() - true_xyz).abs().max()):.3f}", flush=True)


def big():
    import ctypes
    vol = torch.as_tensor(synthetic.make_volume(D, "rand", seed=0)).to(dev)
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H)).to(dev)
    N = H * H
    for B in [int(b) for b in args.batches.split(",")]:
        rot, xyz = synthetic.make_poses(max(B, 2), seed=0)
        s, t, l = bench._device_rays(drr, rot[:B], xyz[:B], dev)
        visits = int(siddon_visits((D, D, D), s, t).sum().item())
        out, sens = torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev)
        ref_out = torch.empty(B, N, device=dev)
        ws = torch.empty(int(lib.b200drr_siddon_brick_workspace_bytes(B, H, H)), dtype=torch.uint8, device=dev)

        def fwd(variant, o=out):
            _lib.check(lib.b200drr_siddon_fwd_grid(_ptr(vol), D, D, D, _ptr(s), _ptr(t), _ptr(l), _ptr(o), B, H, H, 0.5, 1e-8,
                                                   variant, _stream()), "fwd_grid")

        def brick():
            _lib.check(lib.b200drr_siddon_fwd_brick(_ptr(vol), D, D, D, _ptr(s), _ptr(t), _ptr(l), None, None, None, None, _ptr(out),
                                                    ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, H, H, 0.5, 1e-8, 0, _stream()), "brick")

        def sns(variant, o=out, q=sens):
            _lib.check(lib.b200drr_siddon_fwd_sens_grid(_ptr(vol), D, D, D, _ptr(s), _ptr(t), _ptr(l), _ptr(o), _ptr(q), B, H, H,
                                                        0.5, 1e-8, variant, _stream()), "fwd_sens_grid")

        def ms(fn):
            return float(np.median(bench._time_events(fn, 9, warmup=3)))

        fwd(15, ref_out)
        pct = lambda tt: 4 * visits / tt * 1e-6 / peak * 100  # noqa: E731
        t_slab, t_brick, t_sens = ms(lambda: fwd(15)), ms(brick), ms(lambda: sns(0))
        print(f"{D}^3 -> {H}^2 x {B} poses ({visits / (B * N):.0f} visits/ray): forward slab-major {t_slab * 1e3:7.1f} us ({pct(t_slab):4.1f} %) | "
              f"brick {t_brick * 1e3:7.1f} us ({pct(t_brick):4.1f} %) | sens default {t_sens * 1e3:7.1f} us ({pct(t_sens):4.1f} %)", flush=True)
        for K in [int(k) for k in args.pieces.split(",")]:
            fwd(100 + K)
            e = float((out - ref_out).abs().max() / ref_out.abs().max())
            tf = ms(lambda: fwd(100 + K))
            sns(100 + K)
            es = float((out - ref_out).abs().max() / ref_out.abs().max())
            ts = ms(lambda: sns(100 + K))
            print(f"  K = {K:2d}: forward {tf * 1e3:7.1f} ({pct(tf):4.1f} %, {e:.0e}) | sens {ts * 1e3:7.1f} ({pct(ts):4.1f} %, {es:.0e})",
                  flush=True)


if args.loop:
    loop()
elif args.big:
    big()
else:
    kernels()
