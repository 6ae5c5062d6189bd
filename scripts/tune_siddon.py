#!/usr/bin/env python
"""Times Siddon-forward kernel variants on the bench workload and checks them against the plain kernel."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from diffdrr_b200 import DRR, _lib, synthetic  # noqa: E402
from diffdrr_b200.pose import convert  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream, siddon_visits  # noqa: E402

D, H, B = 512, 256, int(os.environ.get("B", 16))
D1, D2 = int(os.environ.get("D1", D)), int(os.environ.get("D2", D))  # non-power-of-two pitches (bank-conflict experiment)
dev = torch.device("cuda:0")
lib = _lib.load()
vol = torch.rand(D, D1, D2, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
subj.volume.affine = synthetic.make_affine(D)
drr = DRR(subj, **synthetic.detector_kwargs(H)).to(dev)
rot, xyz = synthetic.make_poses(B, seed=0)
with torch.no_grad():
    src, tgt = drr.detector(convert(rot.to(dev), xyz.to(dev), parameterization="euler_angles", convention="ZXY"), None)
    raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
    src = drr.affine_inverse(src).reshape(B, 3).contiguous()
    tgt = drr.affine_inverse(tgt).contiguous()
N = H * H
visits = int(siddon_visits((D, D1, D2), src, tgt).sum())
print("dims", (D, D1, D2), "visits/ray", visits / (B * N))
gbytes = (4 * visits + 20 * B * N) / 1e9
peak = 6570.9


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


ref = torch.empty(B, N, device=dev)
def base():
    _lib.check(lib.b200drr_siddon_fwd(_ptr(vol), D, D1, D2, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(ref), B, N, 0.5, 1e-8, 0, 0, _stream()), "fwd")
ms = timeit(base)
print(f"baseline linear       : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {gbytes / ms * 1e3:8.1f} GB/s  {gbytes / ms * 1e3 / peak * 100:5.1f}% of HBM peak")
variants = [int(v) for v in os.environ.get("VARIANTS", "0,15").split(",")]
for v in variants:
    out = torch.zeros(B, N, device=dev)
    def run():
        _lib.check(lib.b200drr_siddon_fwd_grid(_ptr(vol), D, D1, D2, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, H, H, 0.5, 1e-8, v, _stream()), "grid")
    try:
        ms = timeit(run)
    except Exception as e:  # unknown variant
        print(f"variant {v}: {e}")
        continue
    err = float((out - ref).abs().max() / ref.abs().max())
    print(f"grid variant {v:2d}       : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {gbytes / ms * 1e3:8.1f} GB/s  {gbytes / ms * 1e3 / peak * 100:5.1f}% of HBM peak   maxdiff vs plain {err:.1e}")

# ---- EXPERIMENT: chunk-reuse forward over a major-axis-fastest copy (b200drr_x_*), XVARIANTS=0,1,... [XAXIS=1] ------------
if os.environ.get("XVARIANTS"):
    axis = int(os.environ.get("XAXIS", 1))  # the bench poses travel along volume axis 1
    volT = torch.empty(D * D1 * D2 + 4, device=dev)
    t_ms = timeit(lambda: _lib.check(lib.b200drr_x_transpose_volume(_ptr(vol), D, D1, D2, axis, _ptr(volT), _stream()), "transpose"), 2)
    print(f"transpose to axis-{axis}-fastest: {t_ms:.3f} ms")
    for v in [int(x) for x in os.environ["XVARIANTS"].split(",")]:
        out = torch.zeros(B, N, device=dev)
        def run():
            _lib.check(lib.b200drr_x_siddon_fwd_chunk(_ptr(volT), D, D1, D2, axis, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, H, H, 0.5, 1e-8, v, _stream()), "chunk")
        try:
            ms = timeit(run)
        except Exception as e:
            print(f"chunk variant {v}: {e}")
            continue
        err = float((out - ref).abs().max() / ref.abs().max())
        print(f"chunk variant {v:2d}      : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {gbytes / ms * 1e3:8.1f} GB/s  {gbytes / ms * 1e3 / peak * 100:5.1f}% of HBM peak   maxdiff vs plain {err:.1e}")

    for v in [int(x) for x in os.environ.get("XSVARIANTS", "").split(",") if x]:
        out, sens = torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev)
        def run():
            _lib.check(lib.b200drr_x_siddon_sens_chunk(_ptr(volT), D, D1, D2, axis, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens), B, H, H, 0.5, 1e-8, v, _stream()), "sens chunk")
        try:
            ms = timeit(run)
        except Exception as e:
            print(f"sens chunk variant {v}: {e}")
            continue
        err = float((out - ref).abs().max() / ref.abs().max())
        print(f"sens chunk variant {v:2d} : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {(gbytes + 32e-9 * B * N) / ms * 1e3 / peak * 100:5.1f}% of HBM peak   maxdiff img vs plain {err:.1e}")

# ---- forward + sensitivities (training-step fast path) variants ----------------------------------------------------
if os.environ.get("SVARIANTS"):
    gout_s = torch.rand(B, N, device=dev)
    g_src0, g_tgt0, g_len0 = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev)
    _lib.check(lib.b200drr_siddon_bwd(_ptr(vol), D, D1, D2, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout_s), _ptr(g_src0), _ptr(g_tgt0), _ptr(g_len0), None, B, N, 0.5, 1e-8, 0, 0, _stream()), "bwd")
    sbytes = (4 * visits + 52 * B * N) / 1e9
    for v in [int(x) for x in os.environ["SVARIANTS"].split(",")]:
        out, sens = torch.empty(B, N, device=dev), torch.empty(B, N, 8, device=dev)
        g_src, g_tgt, g_len = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev)
        def run():
            _lib.check(lib.b200drr_siddon_fwd_sens_grid(_ptr(vol), D, D1, D2, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens), B, H, H, 0.5, 1e-8, v, _stream()), "sens")
        try:
            ms = timeit(run)
        except Exception as e:
            print(f"sens variant {v}: {e}")
            continue
        _lib.check(lib.b200drr_siddon_bwd_sens(_ptr(sens), _ptr(gout_s), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), B, N, 0, _stream()), "bwd_sens")
        e = [float((a - b).abs().max() / b.abs().max()) for a, b in ((out, ref), (g_src, g_src0), (g_tgt, g_tgt0), (g_len, g_len0))]
        print(f"sens variant {v:2d}       : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {sbytes / ms * 1e3:8.1f} GB/s  {sbytes / ms * 1e3 / peak * 100:5.1f}% of HBM peak   maxdiff img/src/tgt/len {e[0]:.1e} {e[1]:.1e} {e[2]:.1e} {e[3]:.1e}")
    if os.environ.get("SENS_ONLY"):
        sys.exit(0)

# ---- backward variants ----------------------------------------------------------------------------------------
gout = torch.rand(B, N, device=dev)
g_src0, g_tgt0, g_len0 = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev)
def bbase():
    _lib.check(lib.b200drr_siddon_bwd(_ptr(vol), D, D1, D2, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), _ptr(g_src0), _ptr(g_tgt0), _ptr(g_len0), None, B, N, 0.5, 1e-8, 0, 0, _stream()), "bwd")
bbytes = (4 * visits + 36 * B * N) / 1e9
ms = timeit(bbase, 3)
print(f"bwd baseline linear   : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {bbytes / ms * 1e3:8.1f} GB/s  {bbytes / ms * 1e3 / peak * 100:5.1f}% of HBM peak")
for v in [int(x) for x in os.environ.get("BVARIANTS", "0").split(",")]:
    g_src, g_tgt, g_len = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev)
    def run():
        _lib.check(lib.b200drr_siddon_bwd_grid(_ptr(vol), D, D1, D2, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), None, B, H, H, 0.5, 1e-8, 0, v, _stream()), "bwd_grid")
    ms = timeit(run)
    e = [float((a - b).abs().max() / b.abs().max()) for a, b in ((g_src, g_src0), (g_tgt, g_tgt0), (g_len, g_len0))]
    print(f"bwd grid variant {v:2d}   : {ms:8.3f} ms  {B / ms * 1e3:9.1f} DRR/s  {bbytes / ms * 1e3:8.1f} GB/s  {bbytes / ms * 1e3 / peak * 100:5.1f}% of HBM peak   maxdiff src/tgt/len {e[0]:.1e} {e[1]:.1e} {e[2]:.1e}")
