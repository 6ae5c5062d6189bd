#!/usr/bin/env python
"""BASELINE config 5: 2D/3D registration loop, 512^3 CT, 256^2 target DRR, gradient steps on one H100.

Mirrors the loop of notebooks/tutorials/registration.ipynb cell 10: Registration(drr, rot, xyz) -> NCC vs a fixed
target -> backward -> optimizer step.  Prints it/s and the final pose error.  --loss picks the image loss: global NCC (the
default), multiscale NCC ([None, 13] patch sizes, weights [0.5, 0.5]) or gradient NCC (sigma = 1)."""
import argparse, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from diffdrr_b200 import (DRR, GradientNormalizedCrossCorrelation2d, MultiscaleNormalizedCrossCorrelation2d,
                          NormalizedCrossCorrelation2d, Registration, synthetic)

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=1000)
ap.add_argument("--vol", type=int, default=512)
ap.add_argument("--det", type=int, default=256)
ap.add_argument("--renderer", default="siddon")
ap.add_argument("--graph", action="store_true", help="capture one optimisation step in a CUDA graph")
ap.add_argument("--loss", choices=("ncc", "multiscale", "gradient"), default="ncc")
args = ap.parse_args()
dev = torch.device("cuda:0")
vol = torch.from_numpy(synthetic.make_volume(args.vol, "smooth", seed=1))
kw = dict(stop_gradients_through_grid_sample=True) if args.renderer == "siddon" else {}
drr = DRR(synthetic.make_subject(vol), **synthetic.detector_kwargs(args.det), renderer=args.renderer, **kw).to(dev)
true_rot, true_xyz = torch.tensor([[0.0, 0.0, 0.0]], device=dev), torch.tensor([[0.0, 850.0, 0.0]], device=dev)
with torch.no_grad():
    target = drr(true_rot, true_xyz, parameterization="euler_angles", convention="ZXY")
rot0 = true_rot + torch.tensor([[0.15, -0.1, 0.08]], device=dev)
xyz0 = true_xyz + torch.tensor([[12.0, -25.0, 9.0]], device=dev)
reg = Registration(drr, rot0.clone(), xyz0.clone(), "euler_angles", "ZXY").to(dev)
ncc = {"ncc": lambda: NormalizedCrossCorrelation2d(),
       "multiscale": lambda: MultiscaleNormalizedCrossCorrelation2d([None, 13], [0.5, 0.5]),
       "gradient": lambda: GradientNormalizedCrossCorrelation2d(sigma=1.0)}[args.loss]()
opt = torch.optim.SGD([{"params": [reg.rotation], "lr": 5e-2}, {"params": [reg.translation], "lr": 3e2}], momentum=0.9,
                      capturable=False) if False else torch.optim.Adam(
    [{"params": [reg.rotation], "lr": 5e-3}, {"params": [reg.translation], "lr": 5e-1}], capturable=args.graph, fused=True)


def step():
    opt.zero_grad(set_to_none=False)
    loss = 1.0 - ncc(target, reg()).mean()
    loss.backward()
    opt.step()
    return loss


side = torch.cuda.Stream()
side.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(side):  # warm up on a side stream (the documented recipe for whole-step graph capture)
    for _ in range(5):
        loss = step()
torch.cuda.current_stream().wait_stream(side)
torch.cuda.synchronize()
if args.graph:
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static_loss = step()
    run = g.replay
else:
    run = step
t0 = time.perf_counter()
for _ in range(args.steps):
    run()
torch.cuda.synchronize()
dt = time.perf_counter() - t0
with torch.no_grad():
    final = float(1.0 - ncc(target, reg()).mean())
loss_tag = "" if args.loss == "ncc" else f", loss {args.loss}"
print(json.dumps({"config": f"registration loop {args.vol}^3 CT, {args.det}^2 target, {args.renderer}, B=1{loss_tag}", "steps": args.steps,
                  "it_per_s": args.steps / dt, "ms_per_it": 1e3 * dt / args.steps, "cuda_graph": args.graph, "final_1_minus_ncc": final,
                  "rot_err": (reg.rotation.detach() - true_rot).abs().max().item(),
                  "xyz_err": (reg.translation.detach() - true_xyz).abs().max().item()}))
