#!/usr/bin/env python
"""Times the brick-major (TMA) Siddon forward variants on the bench workload and checks them against the slab-major kernel.

  BVARIANTS=0,1,...   brick variants (siddon_brick.cu; ids other than 0 need B200DRR_BUILD_EXPERIMENTS=1)   B=16  poses   D=512  H=256
  SMALL=1             also run small / odd-shaped correctness cases first
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from diffdrr_b200 import DRR, _lib, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream, siddon_visits  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
PEAK = 6570.9


def rays(dims, H, W, B, seed=0):
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(dims)
    drr = DRR(subj, **synthetic.detector_kwargs(H, W)).to(dev)
    rot, xyz = synthetic.make_poses(B, seed=seed)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot.to(dev), xyz.to(dev), parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
        src = drr.affine_inverse(src).reshape(B, 3).contiguous()
        tgt = drr.affine_inverse(tgt).contiguous()
    return src, tgt, raylen


def timeit(fn, iters=5):
    fn(); fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def brick_call(vol, dims, src, tgt, raylen, out, ws, B, H, W, v):
    _lib.check(lib.b200drr_siddon_fwd_brick(_ptr(vol), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), None, None, None, None,
                                            _ptr(out), ws.data_ptr(), ws.numel(), B, H, W, 0.5, 1e-8, v, _stream()), "brick")


def grid_call(vol, dims, src, tgt, raylen, out, B, H, W, v=0):
    _lib.check(lib.b200drr_siddon_fwd_grid(_ptr(vol), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, H, W, 0.5, 1e-8, v,
                                           _stream()), "grid")


variants = [int(v) for v in os.environ.get("BVARIANTS", "0").split(",")]

if os.environ.get("SMALL", "1") == "1":
    for dims, H, W, B in (((40, 48, 56), 32, 32, 2), ((100, 72, 64), 48, 40, 5), ((64, 64, 64), 64, 64, 1), ((130, 96, 160), 96, 96, 35)):
        vol = torch.rand(*dims, device=dev)
        src, tgt, raylen = rays(dims, H, W, B, seed=3)
        N = H * W
        ref = torch.empty(B, N, device=dev)
        _lib.check(lib.b200drr_siddon_fwd(_ptr(vol), *dims, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(ref), B, N, 0.5, 1e-8, 0, 0, _stream()), "fwd")
        ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(B, H, W), dtype=torch.uint8, device=dev)
        for v in variants:
            out = torch.full((B, N), float("nan"), device=dev)
            brick_call(vol, dims, src, tgt, raylen, out, ws, B, H, W, v)
            torch.cuda.synchronize()
            err = float((out - ref).abs().max() / ref.abs().max())
            print(f"small {dims} {H}x{W} B={B} brick variant {v}: maxdiff vs plain {err:.2e}", flush=True)

D, H, B = int(os.environ.get("D", 512)), int(os.environ.get("H", 256)), int(os.environ.get("B", 16))
dims = (D, D, D)
vol = torch.rand(*dims, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
src, tgt, raylen = rays(dims, H, H, B)
N = H * H
visits = int(siddon_visits(dims, src, tgt).sum())
gbytes = (4 * visits + 20 * B * N) / 1e9
print("dims", dims, "det", H, "B", B, "visits/ray", visits / (B * N), "alg GB", gbytes, flush=True)
ref = torch.empty(B, N, device=dev)
ms = timeit(lambda: grid_call(vol, dims, src, tgt, raylen, ref, B, H, H))
print(f"slab-major (variant 0)  : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {gbytes / ms * 1e3:8.1f} GB/s  {gbytes / ms * 1e3 / PEAK * 100:5.1f}% of HBM peak", flush=True)
ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(B, H, H), dtype=torch.uint8, device=dev)
for v in variants:
    out = torch.zeros(B, N, device=dev)
    try:
        ms = timeit(lambda: brick_call(vol, dims, src, tgt, raylen, out, ws, B, H, H, v))
    except Exception as e:
        print(f"brick variant {v}: {e}", flush=True)
        continue
    err = float((out - ref).abs().max() / ref.abs().max())
    print(f"brick variant {v:2d}        : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {gbytes / ms * 1e3:8.1f} GB/s  {gbytes / ms * 1e3 / PEAK * 100:5.1f}% of HBM peak   maxdiff vs slab {err:.1e}", flush=True)

# ---- batch sweep: where does the brick kernel overtake the slab-major one? (BSWEEP=1,2,4,8,32) -------------------------
if os.environ.get("BSWEEP"):
    for Bs in [int(x) for x in os.environ["BSWEEP"].split(",")]:
        src, tgt, raylen = rays(dims, H, H, Bs)
        ref = torch.empty(Bs, N, device=dev)
        out = torch.zeros(Bs, N, device=dev)
        ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(Bs, H, H), dtype=torch.uint8, device=dev)
        t_slab = timeit(lambda: grid_call(vol, dims, src, tgt, raylen, ref, Bs, H, H))
        t_brick = timeit(lambda: brick_call(vol, dims, src, tgt, raylen, out, ws, Bs, H, H, 0))
        err = float((out - ref).abs().max() / ref.abs().max())
        print(f"B={Bs:3d}: slab-major {t_slab:8.3f} ms ({Bs / t_slab * 1e3:8.1f} DRR/s)   brick {t_brick:8.3f} ms ({Bs / t_brick * 1e3:8.1f} DRR/s)   maxdiff {err:.1e}", flush=True)
