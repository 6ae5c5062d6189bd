#!/usr/bin/env python
"""Times the trilinear kernels on BASELINE config 3's shape (512^3 -> 512^2, n_points=500) at a reduced batch.

  VARIANTS=-1,1,10,...   -1 = one thread per ray (b200drr_trilinear_fwd / _bwd), 1 = the full-grid kernels
                         (b200drr_trilinear_fwd_grid / _bwd_grid, 16x16 tiles), 10 + S = the packed-corner kernels with
                         S-plane slabs (0 = whole rays)
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from diffdrr_b200 import DRR, _lib, synthetic
from diffdrr_b200.pose import convert
from diffdrr_b200.renderers import _ptr, _stream, _get_alpha_minmax

D, H, B, P = 512, int(os.environ.get("H", 512)), int(os.environ.get("B", 4)), 500
dev = torch.device("cuda:0")
lib = _lib.load()
vol = torch.rand(D, D, D, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1)); subj.volume.affine = synthetic.make_affine(D)
drr = DRR(subj, **synthetic.detector_kwargs(H)).to(dev)
rot, xyz = synthetic.make_poses(B, seed=0)
with torch.no_grad():
    src, tgt = drr.detector(convert(rot.to(dev), xyz.to(dev), parameterization="euler_angles", convention="ZXY"), None)
    raylen = (tgt - src).norm(dim=-1).reshape(B, -1).contiguous()
    src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt).contiguous()
    amin, amax = _get_alpha_minmax(src, tgt, torch.tensor([D, D, D], device=dev, dtype=torch.float32), 0.5, 1e-8)
    ar = torch.stack([amin.min(), amax.max()]).contiguous()
    src = src.reshape(B, 3).contiguous()
N = H * H
# in-volume samples (>= 1 corner in bounds) for the algorithmic byte count: 32 B per such sample (SURVEY 8d)
with torch.no_grad():
    lin = torch.linspace(0, 1, P, device=dev) * (ar[1] - ar[0]) + ar[0]
    cnt = 0
    for b in range(B):
        for c in range(0, N, 65536):
            pts = src[b][None, None, :] + lin[None, :, None] * (tgt[b, c:c + 65536][:, None, :] - src[b][None, None, :])
            pix = pts  # shift 0.5 -> pix = x
            cnt += int(((pix > -1) & (pix < D)).all(-1).sum())
gb = cnt * 32 / 1e9
print(f"in-volume samples {cnt / (B * N * P):.3f} of all; algorithmic {gb:.2f} GB fwd")
out = torch.empty(B, N, device=dev)
gout = torch.rand(B, N, device=dev)
g_src, g_tgt, g_len, g_ar = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev), torch.zeros(2, device=dev)
def timeit(fn, iters=3):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters
packed = None
def get_packed():
    """(D+1)^3 x 8 packed-corner volume (b200drr_pack_corners)."""
    global packed
    if packed is None:
        packed = torch.empty(int(lib.b200drr_packed_volume_floats(D, D, D)), device=dev)
        t = timeit(lambda: _lib.check(lib.b200drr_pack_corners(_ptr(vol), D, D, D, _ptr(packed), _stream()), "pack"), 2)
        print(f"pack_corners: {t:.3f} ms for {packed.numel() * 4 / 1e9:.2f} GB")
    return packed
for variant in [int(v) for v in os.environ.get("VARIANTS", "-1").split(",")]:
    def fwd():
        if variant < 0:
            _lib.check(lib.b200drr_trilinear_fwd(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, N, 0.5, 1e-8, P, _ptr(ar), 0, 0, _stream()), "tri fwd")
        elif variant >= 10:
            _lib.check(lib.b200drr_trilinear_fwd_packed(_ptr(get_packed()), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, H, H, 0.5, 1e-8, P, _ptr(ar), max(0, variant - 10), _stream()), "tri fwd packed")
        else:
            _lib.check(lib.b200drr_trilinear_fwd_grid(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, H, H, 0.5, 1e-8, P, _ptr(ar), variant, _stream()), "tri fwd grid")
    def bwd():
        if variant >= 10:
            _lib.check(lib.b200drr_trilinear_bwd_packed(_ptr(get_packed()), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_ar), B, H, H, 0.5, 1e-8, P, _ptr(ar), max(0, variant - 10), _stream()), "tri bwd packed")
            return
        if variant < 0:
            _lib.check(lib.b200drr_trilinear_bwd(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), None, _ptr(g_ar), B, N, 0.5, 1e-8, P, _ptr(ar), 0, _stream()), "tri bwd")
        else:
            _lib.check(lib.b200drr_trilinear_bwd_grid(_ptr(vol), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), None, _ptr(g_ar), B, H, H, 0.5, 1e-8, P, _ptr(ar), variant, _stream()), "tri bwd grid")
    f = timeit(fwd)
    if "ref" not in globals():
        ref = out.clone()  # the first variant in the list is the reference for maxdiff
    err = float((out - ref).abs().max() / ref.abs().max())
    b_ = timeit(bwd) if not os.environ.get("FWD_ONLY") else float("nan")
    print(f"variant {variant:2d}: fwd {f:8.3f} ms {B / f * 1e3:8.1f} DRR/s {gb / f * 1e3:7.1f} GB/s ({gb / f * 1e3 / 65.709:5.1f}%)   bwd {b_:8.3f} ms   fwd+bwd {B / (f + b_) * 1e3:7.1f} DRR/s  {2 * gb / (f + b_) * 1e3:7.1f} GB/s   maxdiff {err:.1e}")

# ---- forward + sensitivities (one march) + elementwise backward: the training-step fast path ------------------------
for slab in [int(v) for v in os.environ.get("SENS_SLABS", "").split(",") if v]:
    sens = torch.empty(B, N, 12, device=dev)
    out2 = torch.empty(B, N, device=dev)
    h_src, h_tgt, h_len, h_ar = torch.empty(B, 3, device=dev), torch.empty(B, N, 3, device=dev), torch.empty(B, N, device=dev), torch.zeros(2, device=dev)
    def sens_fwd():
        _lib.check(lib.b200drr_trilinear_fwd_sens_packed(_ptr(get_packed()), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out2), _ptr(sens), B, H, H, 0.5, 1e-8, P, _ptr(ar), slab, _stream()), "tri sens")
    def sens_bwd():
        h_ar.zero_()
        _lib.check(lib.b200drr_trilinear_bwd_sens(_ptr(sens), _ptr(gout), _ptr(h_src), _ptr(h_tgt), _ptr(h_len), _ptr(h_ar), B, N, _stream()), "tri bwd sens")
    f, b_ = timeit(sens_fwd), timeit(sens_bwd)
    # reference gradients from the two-march packed backward
    g_ar.zero_()
    _lib.check(lib.b200drr_trilinear_bwd_packed(_ptr(get_packed()), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_ar), B, H, H, 0.5, 1e-8, P, _ptr(ar), 0, _stream()), "tri bwd packed")
    _lib.check(lib.b200drr_trilinear_fwd_packed(_ptr(get_packed()), D, D, D, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, H, H, 0.5, 1e-8, P, _ptr(ar), 0, _stream()), "tri fwd packed")
    sens_bwd()
    e = [float((a - b).abs().max() / b.abs().max()) for a, b in ((out2, out), (h_src, g_src), (h_tgt, g_tgt), (h_len, g_len), (h_ar, g_ar))]
    print(f"sens slab {slab:3d}: march {f:8.3f} ms ({gb / f * 1e3 / 65.709:5.1f}% of peak on fwd bytes)  bwd {b_:6.3f} ms   fwd+bwd {B / (f + b_) * 1e3:7.1f} DRR/s   maxdiff img/src/tgt/len/ar " + " ".join(f"{x:.1e}" for x in e))
