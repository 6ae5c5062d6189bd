#!/usr/bin/env python
"""Levenberg-Marquardt on the patch, multiscale and gradient NCC, on one GPU: the normal-equation kernels (csrc/ncc_normal.cu)
at 256^2, B = 1 and 16, P = 6 and 9, for the global NCC, p = 13, the gradient NCC (sigma 1) and the gradient NCC with p = 9; the
same system through the float64 torch statement with an explicit per-window Jz where it fits in memory; the kernels' achieved
bytes/s on the byte model below; and LM against Adam on the same loss (steps and wall time to the registration bounds:
1 - score < 1e-3, rotation error < 0.02 rad, translation < 2 mm) from the registration test's start (128^3 -> 96^2) and from the
benchmark's (512^3 -> 256^2), scaled by the fraction the Adam tests use per loss.  Prints one JSON line per measurement.

Byte model of one b200drr_ncc_normal call (compulsory traffic, B C images of H W pixels, P parameters):
  global  x, t and J read once:                                  B C H W (8 + 4P)
  patch   x, t read once, J read by the window and pixel passes: B C H W (8 + 8P)
The Sobel of the image and of the P Jacobian planes (gradient NCC) is timed in `model_us`, not in `kernel_us`."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from diffdrr_b200 import (DRR, GradientNormalizedCrossCorrelation2d, LevenbergMarquardt,  # noqa: E402
                          MultiscaleNormalizedCrossCorrelation2d, NormalizedCrossCorrelation2d, Registration, synthetic)
from diffdrr_b200.registration import ncc_normal_equations  # noqa: E402

dev = torch.device("cuda:0")
HBM_PEAK = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, iters, warmup=3):
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


def torch_system(x, t, J, p, eps=1e-5):
    """The float64 torch statement: Jz per (window, pixel) explicitly.  x, t (B, C, H, W); J (B, C, H, W, P)."""
    B, C, H, W = x.shape
    x, t, J = x.double(), t.double(), J.double()
    if p is None:
        xw, tw, Jw = x.reshape(B, C, 1, H * W), t.reshape(B, C, 1, H * W), J.reshape(B, C, 1, H * W, -1)
    else:
        win = lambda a: a.unfold(2, p, 1).unfold(3, p, 1).reshape(B, C, -1, p * p)  # noqa: E731
        xw, tw = win(x), win(t)
        Jw = J.permute(0, 1, 4, 2, 3).unfold(3, p, 1).unfold(4, p, 1).reshape(B, C, J.shape[-1], -1, p * p).permute(0, 1, 3, 4, 2)

    def norm(a):
        mu = a.mean(-1, keepdim=True)
        s = (((a - mu) ** 2).mean(-1, keepdim=True) + eps).sqrt()
        return (a - mu) / s, s

    z, s = norm(xw)
    zt, _ = norm(tw)
    Jz = (Jw - Jw.mean(-2, keepdim=True) - z[..., None] * (z[..., None] * Jw).mean(-2, keepdim=True)) / s[..., None]
    return torch.einsum("bcwqk,bcwql->bkl", Jz, Jz), torch.einsum("bcwqk,bcwq->bk", Jz, z - zt)


CONFIGS = {"global": (None, None), "p13": (13, None), "gradient_s1": (None, 1.0), "gradient_s1_p9": (9, 1.0)}


def kernel_case(name, B, P):
    p, sigma = CONFIGS[name]
    H = W = 256
    gen = torch.Generator(device=dev).manual_seed(0)
    img = torch.rand(B, 1, H, W, device=dev, generator=gen) * 3.0
    tgt = 0.5 * img + torch.rand(B, 1, H, W, device=dev, generator=gen)
    J = torch.randn(B, 1, H, W, P, device=dev, generator=gen)
    if sigma is None:
        loss = NormalizedCrossCorrelation2d(patch_size=p)
        x, t, Jv, strides = img, tgt, J, (H * W * P, 0, 1, P)
    else:
        loss = GradientNormalizedCrossCorrelation2d(patch_size=p, sigma=sigma)
        x, t = loss.sobel(img), loss.sobel(tgt)
        Jv = loss.sobel(J.reshape(B, H * W, P).transpose(1, 2).reshape(B * P, 1, H, W))
        strides = (2 * P * H * W, H * W, 2 * H * W, 1)
    C = x.shape[1]
    A = torch.zeros(B, P, P, dtype=torch.float64, device=dev)
    g = torch.zeros(B, P, dtype=torch.float64, device=dev)
    t_kernel = timed(lambda: ncc_normal_equations(x, t, Jv, strides, p, 1e-5, 1.0, A, g), 50)

    def model():  # what LevenbergMarquardt.normal_equations runs per step: the Sobel of the image and of J, then the kernels
        if sigma is None:
            xm, Jm = img, J
        else:
            xm = loss.sobel(img)
            Jm = loss.sobel(J.reshape(B, H * W, P).transpose(1, 2).reshape(B * P, 1, H, W))
        A.zero_()
        g.zero_()
        ncc_normal_equations(xm, t, Jm, strides, p, 1e-5, 1.0, A, g)

    t_model = timed(model, 20)
    nbytes = B * C * H * W * (8 + (4 if p is None else 8) * P)
    out = {"what": f"ncc_normal {name} 256^2 B={B} P={P}", "kernel_us": round(t_kernel, 1), "model_us": round(t_model, 1),
           "bytes": nbytes, "GBps": round(nbytes / t_kernel * 1e-3, 1), "share_of_hbm_peak": round(nbytes / t_kernel * 1e6 / HBM_PEAK, 3)}
    Jt = Jv.view(B, P, C, H, W).permute(0, 2, 3, 4, 1) if sigma is not None else J.expand(B, C, H, W, P)
    try:
        t_torch = timed(lambda: torch_system(x, t, Jt, p), 3, warmup=1)
        out["torch_fp64_us"] = round(t_torch, 1)
    except torch.OutOfMemoryError:
        out["torch_fp64_us"] = "not measured (out of memory)"
    torch.cuda.empty_cache()
    return out


LOSSES = {"gradient": (lambda: GradientNormalizedCrossCorrelation2d(), 0.7),
          "multiscale": (lambda: MultiscaleNormalizedCrossCorrelation2d([None, 13], [0.5, 0.5]), 0.9)}


def registration(vol_n, det, rot_off, xyz_off, loss_name, method, max_steps):
    make, f = LOSSES[loss_name]
    vol = synthetic.make_volume(vol_n, "smooth", seed=1)
    drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(det), renderer="siddon",
              stop_gradients_through_grid_sample=True).to(dev)
    true_rot, true_xyz = torch.tensor([[0.0, 0.0, 0.0]], device=dev), torch.tensor([[0.0, 850.0, 0.0]], device=dev)
    with torch.no_grad():
        target = drr(true_rot, true_xyz, parameterization="euler_angles", convention="ZXY")
    loss_fn = make()

    def fresh():
        return Registration(drr, (true_rot + f * torch.tensor([rot_off], device=dev)).clone(),
                            (true_xyz + f * torch.tensor([xyz_off], device=dev)).clone(), "euler_angles", "ZXY").to(dev)

    def done(reg):
        with torch.no_grad():
            loss = float(1.0 - loss_fn(target, reg()).mean())
        rot_err = float((reg.rotation.detach() - true_rot).abs().max())
        xyz_err = float((reg.translation.detach() - true_xyz).abs().max())
        return (loss < 1e-3 and rot_err < 0.02 and xyz_err < 2.0), loss, rot_err, xyz_err

    def run(reg, check_every):
        if method == "lm":
            step = LevenbergMarquardt(reg, target, loss=loss_fn).step
        else:
            opt = torch.optim.Adam([{"params": [reg.rotation], "lr": 5e-3}, {"params": [reg.translation], "lr": 5e-1}], fused=True)

            def step():
                opt.zero_grad(set_to_none=False)
                loss = 1.0 - loss_fn(target, reg()).mean()
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
            res = done(reg)  # inside the clock: it is what a caller pays to know it may stop
            if res[0]:
                break
        return n, time.perf_counter() - t0, res

    run(fresh(), 1 if method == "lm" else 10)  # warm-up: module loads, caches
    n, dt, (ok, loss, rot_err, xyz_err) = run(fresh(), 1 if method == "lm" else 10)
    return {"what": f"registration {loss_name} {method} from {f} x the {vol_n}^3 -> {det}^2 start", "steps": n,
            "ms": round(dt * 1e3, 1), "converged": ok, "final_1_minus_score": loss, "rot_err_rad": rot_err, "xyz_err_mm": xyz_err}


if __name__ == "__main__":
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    for name in CONFIGS:
        for B in (1, 16):
            for P in (6, 9):
                print(json.dumps(kernel_case(name, B, P)), flush=True)
    for loss_name in LOSSES:
        for method in ("lm", "adam"):
            print(json.dumps(registration(128, 96, [0.12, -0.08, 0.06], [10.0, -20.0, 8.0], loss_name, method,
                                          30 if method == "lm" else 2000)), flush=True)
            print(json.dumps(registration(512, 256, [0.15, -0.1, 0.08], [12.0, -25.0, 9.0], loss_name, method,
                                          30 if method == "lm" else 3000)), flush=True)
