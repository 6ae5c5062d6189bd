#!/usr/bin/env python
"""Kernel launches and peak memory of one forward + backward of each registration loss (B = 1, 256^2 by default), through the
CUDA kernels and through the reference's torch formula of the same loss on the same GPU.  Mirrors the registration step:
loss(target, image) with only the image needing a gradient.  Launches are counted with torch.profiler's CUDA activities
(kernels only; memsets and copies are listed separately).  Prints one JSON line per loss."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from diffdrr_b200 import (GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d,  # noqa: E402
                          NormalizedCrossCorrelation2d)

ap = argparse.ArgumentParser()
ap.add_argument("--det", type=int, default=256)
args = ap.parse_args()
dev = torch.device("cuda:0")
LOSSES = {
    "ncc": lambda: NormalizedCrossCorrelation2d(),
    "patch13": lambda: NormalizedCrossCorrelation2d(patch_size=13),
    "multiscale[None,13]": lambda: MultiscaleNormalizedCrossCorrelation2d([None, 13], [0.5, 0.5]),
    "gradient_s1": lambda: GradientNormalizedCrossCorrelation2d(sigma=1.0),
    "gradient_s1_p9": lambda: GradientNormalizedCrossCorrelation2d(patch_size=9, sigma=1.0),
}


def torch_formula(loss):
    """Route every part of `loss` to the reference's torch formula (the fallback CPU / fp64 inputs take)."""
    for m in loss.modules():
        if isinstance(m, NormalizedCrossCorrelation2d):
            m.fused_ok = m.local_ok = lambda a, b: False
        if hasattr(m, "kernel_ok"):
            m.kernel_ok = lambda img: False
    for m in getattr(loss, "nccs", []):
        m.fused_ok = m.local_ok = lambda a, b: False
    return loss


def step(loss, target, img):
    img.grad = None
    (1.0 - loss(target, img).mean()).backward()


def measure(loss):
    gen = torch.Generator().manual_seed(0)
    target = torch.rand(1, 1, args.det, args.det, generator=gen).to(dev)
    img = (0.5 * target + torch.rand(1, 1, args.det, args.det, generator=gen).to(dev)).requires_grad_(True)
    for _ in range(3):
        step(loss, target, img)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(loss, target, img)
        torch.cuda.synchronize()
    kernels = other = 0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            if "memset" in e.name.lower() or "memcpy" in e.name.lower():
                other += 1
            else:
                kernels += 1
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step(loss, target, img)
    torch.cuda.synchronize()
    return kernels, other, (torch.cuda.max_memory_allocated() - base) / 2**20


for name, make in LOSSES.items():
    k, o, mem = measure(make())
    kt, ot, memt = measure(torch_formula(make()))
    print(json.dumps({"loss": name, "image": f"1x1x{args.det}x{args.det}", "kernels": k, "memset_memcpy": o, "peak_mib": round(mem, 2),
                      "torch_formula_kernels": kt, "torch_formula_memset_memcpy": ot, "torch_formula_peak_mib": round(memt, 2),
                      "device": torch.cuda.get_device_name(dev)}))
