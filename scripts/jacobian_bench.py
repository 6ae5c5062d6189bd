#!/usr/bin/env python
"""DRR.jacobian on one GPU: its time against the fused training step (forward + backward) at 512^3 -> 256^2, B = 1 and 16, both
renderers; the J kernels' achieved bandwidth; and Levenberg-Marquardt against the Adam loop of scripts/registration_bench.py
(iterations and wall time to the registration test's bounds: 1 - NCC < 1e-3, rotation error < 0.02 rad, translation < 2 mm),
from the test's start (128^3 -> 96^2) and from the benchmark's (512^3 -> 256^2).  Prints one JSON line per measurement."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from diffdrr_b200 import DRR, LevenbergMarquardt, NormalizedCrossCorrelation2d, Registration, _lib, synthetic  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream  # noqa: E402

dev = torch.device("cuda:0")
HBM_PEAK = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3  # us


def step_vs_jacobian(vol, renderer, B):
    kw = dict(stop_gradients_through_grid_sample=True) if renderer == "siddon" else {}
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(256), renderer=renderer, **kw).to(dev)
    rot, xyz = (t.to(dev) for t in synthetic.make_poses(B, seed=4))
    r, x = rot.clone().requires_grad_(True), xyz.clone().requires_grad_(True)
    g = torch.rand(B, 1, 256, 256, device=dev)
    par = dict(parameterization="euler_angles", convention="ZXY")

    def train():
        img = drr(r, x, **par)
        torch.autograd.grad((g * img).sum(), (r, x))

    t_step = timed(train, 20)
    t_jac = timed(lambda: drr.jacobian(rot, xyz, **par), 20)
    # the J kernel alone, on saved sensitivities of the right layout
    N, P = 256 * 256, 6
    nv = 8 if renderer == "siddon" else 12
    sens = torch.rand(B, N, nv, device=dev)
    tan = [torch.rand(B, P, *s, device=dev) for s in ((3,), (3, 4), (3, 4))]
    Wd = torch.rand(B, 3, 4, device=dev) + 1.0
    rows, cols = torch.linspace(-100, 100, 256, device=dev), torch.linspace(-100, 100, 256, device=dev)
    J = torch.empty(B, N, P, device=dev)
    lib = _lib.load()
    if renderer == "siddon":
        call = lambda: lib.b200drr_siddon_jac_sens_pose(_ptr(sens), *map(_ptr, tan), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(J),  # noqa: E731
                                                        B, 256, 256, P, 1, _stream())
    else:
        drange = torch.rand(B, 2, P, device=dev)
        call = lambda: lib.b200drr_trilinear_jac_sens_pose(_ptr(sens), *map(_ptr, tan), _ptr(Wd), _ptr(rows), _ptr(cols),  # noqa: E731
                                                           _ptr(drange), _ptr(J), B, 256, 256, P, _stream())
    t_kernel = timed(call, 200, warmup=20)
    nbytes = B * N * (nv * 4 + 4 * P)
    return {"what": f"jacobian {renderer} 512^3 -> 256^2 B={B}", "fused_step_us": round(t_step, 1), "jacobian_us": round(t_jac, 1),
            "jac_kernel_us": round(t_kernel, 2), "jac_kernel_bytes": nbytes, "jac_kernel_GBps": round(nbytes / t_kernel * 1e-3, 1),
            "jac_kernel_share_of_hbm_peak": round(nbytes / t_kernel * 1e6 / HBM_PEAK, 3)}


def registration(vol_n, det, rot_off, xyz_off, method, max_steps):
    vol = synthetic.make_volume(vol_n, "smooth", seed=1)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(det), renderer="siddon",
              stop_gradients_through_grid_sample=True).to(dev)
    true_rot, true_xyz = torch.tensor([[0.0, 0.0, 0.0]], device=dev), torch.tensor([[0.0, 850.0, 0.0]], device=dev)
    with torch.no_grad():
        target = drr(true_rot, true_xyz, parameterization="euler_angles", convention="ZXY")
    ncc = NormalizedCrossCorrelation2d()

    def fresh():
        return Registration(drr, (true_rot + torch.tensor([rot_off], device=dev)).clone(),
                            (true_xyz + torch.tensor([xyz_off], device=dev)).clone(), "euler_angles", "ZXY").to(dev)

    def done(reg):
        with torch.no_grad():
            loss = float(1.0 - ncc(target, reg()).mean())
        return (loss < 1e-3 and float((reg.rotation.detach() - true_rot).abs().max()) < 0.02
                and float((reg.translation.detach() - true_xyz).abs().max()) < 2.0), loss

    def run(reg, check_every):
        if method == "lm":
            lm = LevenbergMarquardt(reg, target)
            step = lm.step
        else:
            opt = torch.optim.Adam([{"params": [reg.rotation], "lr": 5e-3}, {"params": [reg.translation], "lr": 5e-1}], fused=True)

            def step():
                opt.zero_grad(set_to_none=False)
                loss = 1.0 - ncc(target, reg()).mean()
                loss.backward()
                opt.step()
        n = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while n < max_steps:
            for _ in range(check_every):
                step()
            n += check_every
            torch.cuda.synchronize()
            ok, loss = done(reg)  # the check is inside the clock: it is what a caller pays to know it may stop
            if ok:
                break
        return n, time.perf_counter() - t0, ok, loss

    run(fresh(), 1 if method == "lm" else 10)  # warm-up: module loads, caches
    n, dt, ok, loss = run(fresh(), 1 if method == "lm" else 10)
    return {"what": f"registration {method} from {vol_n}^3 -> {det}^2 start", "steps": n, "ms": round(dt * 1e3, 1), "converged": ok,
            "final_1_minus_ncc": loss}


if __name__ == "__main__":
    print(json.dumps({"card": card(), "torch": torch.__version__}))
    vol = synthetic.make_volume(512, "smooth", seed=1)
    for renderer in ("siddon", "trilinear"):
        for B in (1, 16):
            print(json.dumps(step_vs_jacobian(vol, renderer, B)), flush=True)
    for method in ("lm", "adam"):
        print(json.dumps(registration(128, 96, [0.12, -0.08, 0.06], [10.0, -20.0, 8.0], method, 30 if method == "lm" else 2000)),
              flush=True)
        print(json.dumps(registration(512, 256, [0.15, -0.1, 0.08], [12.0, -25.0, 9.0], method, 30 if method == "lm" else 3000)),
              flush=True)
