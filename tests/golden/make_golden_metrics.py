#!/usr/bin/env python
"""Records MultiscaleNormalizedCrossCorrelation2d and GradientNormalizedCrossCorrelation2d values + gradients from the UNMODIFIED
reference (diffdrr/metrics.py:47-104; torchvision's gaussian_blur for the blur).  metrics.py also imports kornia for
MutualInformation; it is stubbed here (never in the product).  Run in the build container:
python tests/golden/make_golden_metrics.py"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "_refshim"))
sys.path.insert(0, "/root/reference")
for name in ("kornia", "kornia.enhance", "kornia.enhance.histogram"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["kornia.enhance.histogram"].marginal_pdf = sys.modules["kornia.enhance.histogram"].joint_pdf = None
from diffdrr.metrics import (GradientNormalizedCrossCorrelation2d,  # noqa: E402  (the reference's own classes)
                             MultiscaleNormalizedCrossCorrelation2d)

g = torch.Generator().manual_seed(0)
x1 = torch.rand(3, 1, 24, 20, generator=g)
x2 = (0.6 * x1 + 0.4 * torch.rand(3, 1, 24, 20, generator=g)).contiguous()
s1 = torch.rand(2, 1, 9, 11, generator=g)
s2 = (0.5 * s1 + 0.5 * torch.rand(2, 1, 9, 11, generator=g)).contiguous()
rec = {"x1": x1.numpy(), "x2": x2.numpy(), "small_x1": s1.numpy(), "small_x2": s2.numpy()}
cases = (
    ("grad_s1", lambda: GradientNormalizedCrossCorrelation2d(sigma=1.0), "x"),
    ("grad_s1_p5", lambda: GradientNormalizedCrossCorrelation2d(patch_size=5, sigma=1.0), "x"),
    ("grad_s0", lambda: GradientNormalizedCrossCorrelation2d(sigma=0.0), "x"),
    ("multiscale", lambda: MultiscaleNormalizedCrossCorrelation2d([None, 5], [0.5, 0.5]), "x"),
    ("grad_s1_small", lambda: GradientNormalizedCrossCorrelation2d(sigma=1.0), "small_x"),
)
for tag, make, src in cases:
    a0, b0 = torch.as_tensor(rec[src + "1"]), torch.as_tensor(rec[src + "2"])
    for dt, suf in ((torch.float32, "f32"), (torch.float64, "f64")):
        loss = make().to(dt)  # .to(float64) converts the Sobel Conv2d's weights along with the images
        a = a0.to(dt)
        b = b0.to(dt).clone().detach().requires_grad_(True)
        score = loss(a, b)
        w = torch.tensor([1.0, -2.0, 0.5][: a.shape[0]], dtype=dt)
        (score * w).sum().backward()
        rec[f"{tag}_score_{suf}"] = score.detach().numpy()
        rec[f"{tag}_grad_x2_{suf}"] = b.grad.numpy()
np.savez_compressed(os.path.join(HERE, "metrics_reference.npz"), **rec)
print({k: v.shape for k, v in rec.items()})
