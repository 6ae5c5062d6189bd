"""`Siddon` and `Trilinear` renderer modules backed by hand-written sm_90a CUDA kernels.

Drop-in for the reference's renderer slot (`DRR.renderer`, reference drr.py:94-101,210): same constructor and
`forward` signatures as reference renderers.py:14-42 (Siddon) and 189-216 (Trilinear), same `(B, 1, N)` result.
The whole `(B, N, M)`-shaped tensor algebra of the reference (plane alphas, sort, midpoints, grid_sample, diff,
sum) is ONE kernel launch per direction through the C ABI of include/b200drr.h; backward is a closed-form
kernel (no saved activations: `checkpoint_gradients` is a no-op by construction).  When only ray / pose gradients are
needed the forward kernel also writes each ray's end-point sensitivities (32-48 B per ray) and the backward is elementwise.

There is no CPU / PyTorch fallback: tensors must be CUDA fp32 (tuned kernels) or CUDA fp64 (reference-literal kernels of
csrc/literal.cu, which also serve a callable `reducefn`), otherwise the call raises.  The volume may also be STORED in fp16 or
bf16 with fp32 rays (DESIGN.md 4.5): the same kernels read it through a widening load; options outside that contract raise.
"""
from __future__ import annotations

import ctypes
import weakref
from typing import Callable

import torch
from torch.autograd.function import once_differentiable

from . import _lib

_REDUCE = {"sum": 0, "max": 1}
# Slab-major scheduling of the packed trilinear FORWARD (include/b200drr.h): 16 base-voxel planes per slab once the batch
# has >= 8 poses to share the slab through L2.  The backward stays one-CTA-per-ray-tile: its per-slab reductions cost more
# than the L2 sharing returns.  (These thresholds have not been re-measured on the H100.)
_PACKED_SLAB_FWD = 16
_PACKED_SLAB_SENS = 0   # forward+sensitivities march: unslabbed (its registers and per-slab set-up outweigh the L2 sharing)
_PACKED_SLAB_MIN_BATCH = 8


# 16-bit volume storage (include/b200drr.h: B200DRR_VOL_F16 / B200DRR_VOL_BF16; DESIGN.md 4.5)
_VOL16 = {torch.float16: 1, torch.bfloat16: 2}


def _check_inputs(volume, source, target, img, dtype=torch.float32, vol16=False):
    for name, t in (("volume", volume), ("source", source), ("target", target), ("img", img)):
        if not t.is_cuda:
            raise _lib.B200DRRError(
                f"diffdrr_b200 renderers run on CUDA devices only ({name} is on {t.device}); there is no CPU fallback")
        if t.dtype != dtype and not (vol16 and t is volume and t.dtype in _VOL16):
            raise NotImplementedError(
                f"diffdrr_b200 kernels take fp32 tensors, or fp64 tensors throughout ({name} is {t.dtype}, volume is {volume.dtype})")
    if volume.dim() != 3:
        raise ValueError(f"volume must be (D0, D1, D2), got {tuple(volume.shape)}")
    B, N = target.shape[0], target.shape[1]
    if target.dim() != 3 or target.shape[2] != 3 or source.numel() != B * 3 or img.numel() != B * N:
        raise ValueError(
            f"expected source (B,1,3), target (B,N,3), img (B,1,N); got {tuple(source.shape)}, {tuple(target.shape)}, "
            f"{tuple(img.shape)}")
    return B, N


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _vol_entry(lib, name, vol, data=None):
    """(entry point, its leading volume arguments, its name): the fp32 entry point `name`, or for a 16-bit volume its twin
    `name`_v16, which takes the voxel type after the pointer (include/b200drr.h).  `data` (default: the volume) is the array
    passed, e.g. the volume's packed-corner copy."""
    data = vol if data is None else data
    code = _VOL16.get(vol.dtype)
    if code is None:
        return getattr(lib, name), (_ptr(data),), name
    return getattr(lib, name + "_v16"), (_ptr(data), code), name + "_v16"


def _check_vol16(volume, source, target=None):
    """A 16-bit volume is a STATIC density read by the default-option kernels; refuse the rest before any launch."""
    if volume.requires_grad:
        raise NotImplementedError(
            f"a {volume.dtype} volume cannot require grad: 16-bit volumes are static densities (ray and pose gradients are "
            "supported; optimise an fp32 volume for volume gradients)")
    for name, t in (("source", source), ("target", target)):
        if t is not None and t.dtype != torch.float32:
            raise NotImplementedError(
                f"a {volume.dtype} volume is rendered with fp32 rays and poses ({name} is {t.dtype}): convert only the density, "
                "e.g. drr.density = drr.density.to(torch.bfloat16), not the whole module")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# Brick-major forward (include/b200drr.h: b200drr_siddon_fwd_brick; csrc/siddon_brick.cu): TMA-staged voxel bricks in
# shared memory, every staged voxel serves all poses of the batch.  The per-(ray, brick) set-up only pays off once a few
# poses share each staged brick, hence the batch threshold (B200DRR_BRICK_MIN_BATCH).
import os as _os

_BRICK_MIN_BATCH = int(_os.environ.get("B200DRR_BRICK_MIN_BATCH", "2"))
_brick_ws: dict = {}


_BRICK_MIN_BRICKS = int(_os.environ.get("B200DRR_BRICK_MIN_BRICKS", "2048"))
_BRICK_MAX_RAY_DENSITY = float(_os.environ.get("B200DRR_BRICK_MAX_RAY_DENSITY", "0.5"))


def _brick_ok(vol, B, H, W, check_density: bool = True) -> bool:
    # 24 x 32 x 32-voxel bricks over 2 x 132 resident CTAs: below ~7 bricks per CTA the tail of the dynamic brick queue
    # costs more than the staging returns (256^3 = 704 bricks, 512^3 = 5632 bricks)
    n_bricks = -(-vol.shape[0] // 24) * -(-vol.shape[1] // 32) * -(-vol.shape[2] // 32)
    # ... and only for SPARSE ray sets (detector pixels fewer than ~half the voxels of a volume cross-section, i.e. rays
    # >= ~1.4 voxels apart): dense rays share 32-byte sectors in L1 and the slab-major gather wins (at 512^3 -> 1024^2;
    # at 512^3 -> 256^2 the other way round)
    sparse = (not check_density) or H * W <= _BRICK_MAX_RAY_DENSITY * float(vol.numel()) ** (2.0 / 3.0)
    # the TMA map needs 16-byte row strides: D2 % 4 == 0 for fp32 voxels, D2 % 8 == 0 for 16-bit ones
    aligned = vol.shape[2] % (16 // vol.element_size()) == 0
    return (B >= _BRICK_MIN_BATCH and n_bricks >= _BRICK_MIN_BRICKS and sparse and aligned and 2 <= H <= 2048
            and 2 <= W <= 2048 and B * H * W < 2**31 and vol.data_ptr() % 16 == 0 and vol.numel() < 2**31 - 1)


# Full detector grids: at a load of 1 (B * H * W in units of 256^2 rays) the library's own forward kernel, which cuts every ray
# into pieces along its major axis (csrc/siddon.cu small_batch_pieces), beats the brick kernel; from 2 poses on the brick kernel
# is faster.  H100 (scripts/tune_thresholds.py, 512^3 -> 256^2, us per launch, pieces / brick): 1 pose 124 / 240, 2: 384 / 284,
# 4: 538 / 390, 16: 2479 / 1263.
_BRICK_FULL_GRID_MIN_LOAD = float(_os.environ.get("B200DRR_BRICK_MIN_LOAD", "1"))


def _brick_full_grid_ok(vol, B, H, W) -> bool:
    return B * H * W > _BRICK_FULL_GRID_MIN_LOAD * 65536.0 and _brick_ok(vol, B, H, W)


_BRICK_BWD = _os.environ.get("B200DRR_BRICK_BWD", "1") != "0"
_BRICK_BWD_MIN_BATCH = int(_os.environ.get("B200DRR_BRICK_BWD_MIN_BATCH", "1"))


def _brick_bwd_ok(vol, B, H, W) -> bool:
    """Volume gradient through the brick kernel's scatter mode (b200drr_siddon_bwd_vol_brick): shared-memory accumulation and one
    TMA store per brick instead of one global atomic per voxel visit."""
    return (_BRICK_BWD and B >= _BRICK_BWD_MIN_BATCH
            and _brick_ok(vol, max(B, _BRICK_MIN_BATCH), H, W))  # sparse rays only: at 512^3 -> 512^2 the CAS loops collide (1.08x)


def _brick_workspace(device, B, H, W):
    """Cached scratch for the brick kernel (ray table + per-pose geometry), grown on demand; one buffer per device and
    stream so concurrent streams never share it (the pointer is stable, so captured CUDA graphs stay valid)."""
    need = int(_lib.load().b200drr_siddon_brick_workspace_bytes(B, H, W))
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    ws = _brick_ws.get(key)
    if ws is None or ws.numel() < need:
        if torch.cuda.is_current_stream_capturing():
            raise _lib.B200DRRError("brick workspace must be allocated before CUDA-graph capture: run one eager step first")
        ws = torch.empty(need, dtype=torch.uint8, device=device)
        _brick_ws[key] = ws
    return ws


# Arbitrary ray sets (sub-sampled detectors, patches, user rays) reach the tiled, slab-major kernels through a LOCALITY
# ORDER: rays are sorted by the Morton code of their target points, so consecutive groups of 32 rays are spatial neighbours
# like the 8x4-pixel bundles of the detector-grid kernels (include/b200drr.h: b200drr_siddon_fwd_sorted / _fwd_sens_sorted).
_SORT_MIN_RAYS = int(_os.environ.get("B200DRR_SORT_MIN_RAYS", "1024"))


def _spread3(x: torch.Tensor) -> torch.Tensor:
    """10-bit integers -> bits 0, 3, 6, ... (one lane of a 30-bit 3-D Morton code)."""
    x = (x | (x << 16)) & 0x030000FF
    x = (x | (x << 8)) & 0x0300F00F
    x = (x | (x << 4)) & 0x030C30C3
    return (x | (x << 2)) & 0x09249249


def _locality_order(tgt: torch.Tensor) -> torch.Tensor:
    """(B, N, 3) target points -> (B, N) permutation that sorts every pose's rays along a Z-order curve of their targets."""
    with torch.no_grad():
        lo, hi = tgt.amin(dim=1, keepdim=True), tgt.amax(dim=1, keepdim=True)
        q = ((tgt - lo) / (hi - lo).clamp_min(1e-20) * 1023.0).to(torch.int64).clamp_(0, 1023)
        key = _spread3(q[..., 0]) | (_spread3(q[..., 1]) << 1) | (_spread3(q[..., 2]) << 2)
        return key.argsort(dim=1)


# Training-step fast path: when only the ray end points need gradients, the forward walk also accumulates the per-ray
# sensitivities and the backward pass is elementwise (one walk per step instead of two).  Module-level switch for A/B tests.
_FUSED_SENSITIVITIES = True


def _wants_sens(needs_input_grad, stop_grad) -> bool:
    """inputs 1..3 are the ray-defining tensors; input 0 is the volume (its gradient needs the backward walk)."""
    need_vol = needs_input_grad[0] and not stop_grad
    return any(needs_input_grad[1:4]) and not need_vol


def _ray_grads(ctx, B, N, dtype, device, stop_grad=False):
    """Gradient buffers of the ray inputs that need one -- inputs 1..3 (source, target, img) of every ray-tensor autograd
    function: g_src (B,3), g_tgt (B,N,3), g_len (B,N), or None; stop_grad drops the ray-length gradient."""
    _, need_src, need_tgt, need_len = ctx.needs_input_grad[:4]
    return (torch.empty(B, 3, dtype=dtype, device=device) if need_src else None,
            torch.empty(B, N, 3, dtype=dtype, device=device) if need_tgt else None,
            torch.empty(B, N, dtype=dtype, device=device) if (need_len and not stop_grad) else None)


def _ray_grads_back(ctx, g_src, g_tgt, g_len):
    """The buffers of _ray_grads viewed as the shapes forward received (ctx.ray_shapes)."""
    src_shape, img_shape = ctx.ray_shapes
    return None if g_src is None else g_src.view(src_shape), g_tgt, None if g_len is None else g_len.view(img_shape)


class _SiddonFunction(torch.autograd.Function):
    """out (B,1,N) = Siddon line integrals; backward = closed-form kernel (include/b200drr.h).  An fp64 volume takes the
    reference-literal kernels (csrc/literal.cu: b200drr_siddon_fwd_f64 / _bwd_f64, what `drr.to(torch.float64)` reaches in
    the reference, drr.py:75) and mode = 1 (Siddon(mode="bilinear"), reference renderers.py:18,66: trilinear sampling at the
    segment midpoints) the general walk (b200drr_siddon_fwd_general / _bwd_general); both run one thread per ray whatever the
    ray set, and their reducefn="max" is forward-only."""

    @staticmethod
    def forward(ctx, volume, source, target, img, voxel_shift, eps, reduce, align_corners, stop_grad, grid, subset=None,
                mode=0):
        fp64 = volume.dtype == torch.float64
        B, N = _check_inputs(volume, source, target, img, torch.float64 if fp64 else torch.float32, vol16=True)
        vol = volume.contiguous()
        src = source.reshape(B, 3).contiguous()
        tgt = target.contiguous()
        raylen = img.reshape(B, N).contiguous()
        out = torch.empty(B, N, dtype=torch.float64 if fp64 else torch.float32, device=vol.device)
        literal = fp64 or mode != 0
        # full detector grid + default options -> tiled, slab-major kernels (include/b200drr.h: *_grid)
        if grid is not None and (literal or grid[0] * grid[1] != N or reduce != 0 or align_corners
                                 or vol.numel() >= 2**31 - 1):
            grid = None
        lib = _lib.load()
        fast = not literal and reduce == 0 and not align_corners and vol.numel() < 2**31 - 1
        # Ray gradients wanted and no volume gradient: ONE walk yields the image and the 6 per-ray sensitivities, and the
        # backward is elementwise (include/b200drr.h: b200drr_siddon_fwd_sens_grid / _bwd_sens).
        sens = None
        if fast and _FUSED_SENSITIVITIES and _wants_sens(ctx.needs_input_grad, stop_grad):
            sens = torch.empty(B, N, 8, dtype=torch.float32, device=vol.device)
        if vol.dtype in _VOL16 and sens is None and any(ctx.needs_input_grad[1:4]):
            raise NotImplementedError(f"ray gradients from a {vol.dtype} volume come from the fused sensitivities walk only")
        with torch.cuda.device(vol.device):
            if literal:   # b200drr_siddon_fwd_f64 takes the arguments of b200drr_siddon_fwd; the general walk adds the mode
                name = "b200drr_siddon_fwd_f64" if fp64 else "b200drr_siddon_fwd_general"
                _lib.check(getattr(lib, name)(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, N,
                                              voxel_shift, eps, reduce, int(align_corners), *(() if fp64 else (mode,)),
                                              _stream()), name)
            elif (grid is None and fast and sens is None and subset is not None and subset[0].numel() == subset[2] * subset[3]
                    and N == subset[4] and _brick_ok(vol, B, subset[2], subset[3], check_density=False)):
                # inference on a sub-sampled detector: brick-major kernel with a pixel -> ray map (include/b200drr.h)
                pix, corners, Hs, Ws, _n = subset
                ws = _brick_workspace(vol.device, B, 1, N)
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_brick_subset", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), ctypes.c_void_p(pix.data_ptr()),
                              _ptr(corners.contiguous().float()), _ptr(out), ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, Hs, Ws,
                              N, voxel_shift, eps, 0, _stream()), name)
            elif grid is None and fast and N >= _SORT_MIN_RAYS:
                # arbitrary ray set, big enough to be worth ordering: sort for locality, walk slab-major, un-sort the results
                perm = _locality_order(tgt)
                tgt_s = torch.gather(tgt, 1, perm.unsqueeze(-1).expand(-1, -1, 3)).contiguous()
                len_s = torch.gather(raylen, 1, perm).contiguous()
                out_s = torch.empty_like(out)
                if sens is not None:
                    sens_s = torch.empty_like(sens)
                    fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_sens_sorted", vol)
                    _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt_s), _ptr(len_s), _ptr(out_s), _ptr(sens_s), B, N,
                                  voxel_shift, eps, _stream()), name)
                    sens.scatter_(1, perm.unsqueeze(-1).expand(-1, -1, 8), sens_s)
                else:
                    fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_sorted", vol)
                    _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt_s), _ptr(len_s), _ptr(out_s), B, N, voxel_shift, eps,
                                  _stream()), name)
                out.scatter_(1, perm, out_s)
            elif sens is not None and grid is None:   # small arbitrary ray set (one thread per ray)
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_sens", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens), B, N, voxel_shift,
                              eps, _stream()), name)
            elif sens is not None:
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_sens_grid", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens), B, grid[0], grid[1],
                              voxel_shift, eps, 0, _stream()), name)
            elif grid is not None and _brick_full_grid_ok(vol, B, grid[0], grid[1]):
                ws = _brick_workspace(vol.device, B, grid[0], grid[1])
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_brick", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), None, None, None, None, _ptr(out),
                              ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, grid[0], grid[1], voxel_shift, eps, 0, _stream()),
                           name)
            elif grid is not None:
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_grid", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, grid[0], grid[1], voxel_shift,
                              eps, 0, _stream()), name)
            else:
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, N, voxel_shift, eps, reduce,
                              int(align_corners), _stream()), name)
        if sens is not None:
            ctx.save_for_backward(sens)
        else:
            ctx.save_for_backward(vol, src, tgt, raylen)
        ctx.fused = sens is not None
        ctx.cfg = (voxel_shift, eps, reduce, align_corners, stop_grad, grid, mode)
        ctx.ray_shapes = (tuple(source.shape), tuple(img.shape))
        return out.view(B, 1, N)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        voxel_shift, eps, reduce, align_corners, stop_grad, grid, mode = ctx.cfg
        if ctx.fused:
            (sens,) = ctx.saved_tensors
            B, N = sens.shape[0], sens.shape[1]
            gout = gout.reshape(B, N).contiguous().float()
            g_src, g_tgt, g_len = _ray_grads(ctx, B, N, torch.float32, sens.device, stop_grad)
            with torch.cuda.device(sens.device):
                _lib.check(_lib.load().b200drr_siddon_bwd_sens(_ptr(sens), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len),
                                                               B, N, int(stop_grad), _stream()), "b200drr_siddon_bwd_sens")
            return (None, *_ray_grads_back(ctx, g_src, g_tgt, g_len), None, None, None, None, None, None, None, None)
        vol, src, tgt, raylen = ctx.saved_tensors
        fp64 = vol.dtype == torch.float64
        if fp64 and reduce != 0:
            raise NotImplementedError("fp64 Siddon: backward is implemented for reducefn='sum'")
        if mode != 0 and reduce != 0:
            raise NotImplementedError("backward through Siddon(mode='bilinear', reducefn='max') is not implemented")
        B, N = tgt.shape[0], tgt.shape[1]
        gout = gout.reshape(B, N).contiguous().to(torch.float64 if fp64 else torch.float32)
        g_src, g_tgt, g_len = _ray_grads(ctx, B, N, gout.dtype, vol.device, stop_grad)
        need_vol = ctx.needs_input_grad[0] and not stop_grad
        vol_by_brick = (need_vol and grid is not None and reduce == 0 and not align_corners
                        and _brick_bwd_ok(vol, B, grid[0], grid[1]))
        g_vol = (torch.empty_like(vol) if vol_by_brick else torch.zeros_like(vol)) if need_vol else None
        lib = _lib.load()
        with torch.cuda.device(vol.device):
            if fp64:   # b200drr_siddon_bwd_f64 takes the arguments of b200drr_siddon_bwd
                _lib.check(lib.b200drr_siddon_bwd_f64(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                      _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), B, N, voxel_shift, eps,
                                                      int(stop_grad), int(align_corners), _stream()), "b200drr_siddon_bwd_f64")
            elif reduce != 0 or align_corners or mode != 0:  # options outside the fast kernels: plane-by-plane general walk
                _lib.check(lib.b200drr_siddon_bwd_general(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                          _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), B, N, voxel_shift,
                                                          eps, int(stop_grad), reduce, int(align_corners), mode, _stream()),
                           "b200drr_siddon_bwd_general")
            elif vol_by_brick:
                # volume gradient by the brick kernel's scatter mode (no global atomics; g_vol overwritten), ray gradients --
                # when wanted at all -- by the slab-major walk without a volume gradient
                ws = _brick_workspace(vol.device, B, grid[0], grid[1])
                _lib.check(lib.b200drr_siddon_bwd_vol_brick(_ptr(gout), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), None, None,
                                                            None, None, _ptr(g_vol), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                                            B, grid[0], grid[1], voxel_shift, eps, _stream()),
                           "b200drr_siddon_bwd_vol_brick")
                if g_src is not None or g_tgt is not None or g_len is not None:
                    _lib.check(lib.b200drr_siddon_bwd_grid(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                           _ptr(g_src), _ptr(g_tgt), _ptr(g_len), None, B, grid[0], grid[1],
                                                           voxel_shift, eps, int(stop_grad), 0, _stream()),
                               "b200drr_siddon_bwd_grid")
            elif grid is not None:
                _lib.check(lib.b200drr_siddon_bwd_grid(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                       _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), B, grid[0], grid[1],
                                                       voxel_shift, eps, int(stop_grad), 0, _stream()),
                           "b200drr_siddon_bwd_grid")
            else:
                _lib.check(lib.b200drr_siddon_bwd(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                  _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), B, N, voxel_shift, eps,
                                                  int(stop_grad), int(align_corners), _stream()),
                           "b200drr_siddon_bwd")
        return (g_vol, *_ray_grads_back(ctx, g_src, g_tgt, g_len), None, None, None, None, None, None, None, None)


def _siddon_sens_pose(vol, src, G, Wd, rows, cols, voxel_shift, eps):
    """The sensitivities walk of the in-kernel rays of a full detector grid (include/b200drr.h: b200drr_siddon_fwd_sens_pose):
    -> (out (B, H*W), sens (B, H*W, 8)), the image and every ray's end-point sensitivities.  Inputs contiguous fp32."""
    B, H, W = G.shape[0], rows.numel(), cols.numel()
    out = torch.empty(B, H * W, dtype=torch.float32, device=vol.device)
    sens = torch.empty(B, H * W, 8, dtype=torch.float32, device=vol.device)
    fn, head, name = _vol_entry(_lib.load(), "b200drr_siddon_fwd_sens_pose", vol)
    with torch.cuda.device(vol.device):
        _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(G), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(out), _ptr(sens), B, H, W,
                      voxel_shift, eps, _stream()), name)
    return out, sens


class _SiddonPoseFunction(torch.autograd.Function):
    """Siddon line integrals of the full detector grid with the rays generated IN the kernel from per-pose 3x4 matrices
    (include/b200drr.h: b200drr_siddon_fwd_pose / _bwd_pose); gradients come back as matrices, no (B,N,3) tensors."""

    @staticmethod
    def forward(ctx, volume, src, G, Wd, rows, cols, voxel_shift, eps, stop_grad):
        vol = volume.contiguous()
        B, H, W = G.shape[0], rows.numel(), cols.numel()
        src, G, Wd = src.contiguous().float(), G.contiguous().float(), Wd.contiguous().float()
        rows, cols = rows.contiguous().float(), cols.contiguous().float()
        ctx.fused = _FUSED_SENSITIVITIES and _wants_sens(ctx.needs_input_grad, stop_grad)
        ctx.cfg = (voxel_shift, eps, stop_grad)
        if vol.dtype in _VOL16 and not ctx.fused and any(ctx.needs_input_grad[1:4]):
            raise NotImplementedError(f"pose gradients from a {vol.dtype} volume come from the fused sensitivities walk only")
        if ctx.fused:  # one walk: image + per-ray sensitivities; backward is elementwise
            out, sens = _siddon_sens_pose(vol, src, G, Wd, rows, cols, voxel_shift, eps)
            ctx.save_for_backward(sens, Wd, rows, cols)
            return out.view(B, 1, H * W)
        out = torch.empty(B, H * W, dtype=torch.float32, device=vol.device)
        lib = _lib.load()
        with torch.cuda.device(vol.device):
            if _brick_full_grid_ok(vol, B, H, W):
                ws = _brick_workspace(vol.device, B, H, W)
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_brick", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), None, None, _ptr(G), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(out),
                              ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, H, W, voxel_shift, eps, 0, _stream()), name)
            else:
                fn, head, name = _vol_entry(lib, "b200drr_siddon_fwd_pose", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(G), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(out), B, H, W,
                              voxel_shift, eps, _stream()), name)
        ctx.save_for_backward(vol, src, G, Wd, rows, cols)
        return out.view(B, 1, H * W)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        voxel_shift, eps, stop_grad = ctx.cfg
        if ctx.fused:
            sens, Wd, rows, cols = ctx.saved_tensors
            B, H, W = Wd.shape[0], rows.numel(), cols.numel()
            dev = sens.device
            gout = gout.reshape(B, H * W).contiguous().float()
            g_src = torch.empty(B, 3, dtype=torch.float32, device=dev)
            g_G = torch.empty(B, 3, 4, dtype=torch.float32, device=dev)
            g_Wd = torch.empty(B, 3, 4, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(_lib.load().b200drr_siddon_bwd_sens_pose(_ptr(sens), _ptr(gout), _ptr(Wd), _ptr(rows), _ptr(cols),
                                                                    _ptr(g_src), _ptr(g_G), _ptr(g_Wd), B, H, W,
                                                                    int(stop_grad), _stream()), "b200drr_siddon_bwd_sens_pose")
            return None, g_src, g_G, g_Wd, None, None, None, None, None
        vol, src, G, Wd, rows, cols = ctx.saved_tensors
        B, H, W = G.shape[0], rows.numel(), cols.numel()
        dev = vol.device
        gout = gout.reshape(B, H * W).contiguous().float()
        want_vol = ctx.needs_input_grad[0] and not stop_grad
        want_pose = any(ctx.needs_input_grad[1:4])
        g_vol = None
        if want_vol and _brick_bwd_ok(vol, B, H, W):
            # volume gradient by the brick kernel's scatter mode (rays generated in-kernel, no global atomics, g_vol overwritten)
            g_vol = torch.empty_like(vol)
            ws = _brick_workspace(dev, B, H, W)
            with torch.cuda.device(dev):
                _lib.check(_lib.load().b200drr_siddon_bwd_vol_brick(_ptr(gout), *vol.shape, _ptr(src), None, None, _ptr(G), _ptr(Wd),
                                                                    _ptr(rows), _ptr(cols), _ptr(g_vol),
                                                                    ctypes.c_void_p(ws.data_ptr()), ws.numel(), B, H, W,
                                                                    voxel_shift, eps, _stream()), "b200drr_siddon_bwd_vol_brick")
            if not want_pose:  # reconstruction: fixed poses, only the volume is optimised
                return g_vol, None, None, None, None, None, None, None, None
            want_vol = False
        g_src = torch.empty(B, 3, dtype=torch.float32, device=dev)
        g_G = torch.empty(B, 3, 4, dtype=torch.float32, device=dev)
        g_Wd = torch.empty(B, 3, 4, dtype=torch.float32, device=dev)
        ws_tgt = torch.empty(B, H * W, 3, dtype=torch.float32, device=dev)
        ws_len = torch.empty(B, H * W, dtype=torch.float32, device=dev)
        if want_vol:
            g_vol = torch.zeros_like(vol)
        g_vol_walk = g_vol if want_vol else None
        with torch.cuda.device(dev):
            _lib.check(_lib.load().b200drr_siddon_bwd_pose(_ptr(vol), *vol.shape, _ptr(src), _ptr(G), _ptr(Wd), _ptr(rows),
                                                           _ptr(cols), _ptr(gout), _ptr(g_src), _ptr(g_G), _ptr(g_Wd),
                                                           _ptr(g_vol_walk), _ptr(ws_tgt), _ptr(ws_len), B, H, W, voxel_shift,
                                                           eps, int(stop_grad), _stream()), "b200drr_siddon_bwd_pose")
        return g_vol, g_src, g_G, g_Wd, None, None, None, None, None


class _TrilinearFunction(torch.autograd.Function):
    """out (B,1,N) = fixed-step trilinear line integrals for the range alpha_range = [alphamin, alphamax].  An fp64 volume
    takes the reference-literal kernels (b200drr_trilinear_fwd_f64 / _bwd_f64; alpha_range fp64, reducefn="max" forward-only)
    whatever the ray set."""

    @staticmethod
    def forward(ctx, volume, source, target, img, alpha_range, voxel_shift, eps, n_points, reduce, align_corners, grid,
                packed):
        fp64 = volume.dtype == torch.float64
        B, N = _check_inputs(volume, source, target, img, torch.float64 if fp64 else torch.float32, vol16=True)
        if grid is not None and (fp64 or grid[0] * grid[1] != N or reduce != 0 or align_corners):
            grid = None
        if grid is None:
            packed = None
        vol = volume.contiguous()
        src = source.reshape(B, 3).contiguous()
        tgt = target.contiguous()
        raylen = img.reshape(B, N).contiguous()
        dtype = torch.float64 if fp64 else torch.float32
        arange = alpha_range.detach().to(device=vol.device, dtype=dtype).contiguous()
        out = torch.empty(B, N, dtype=dtype, device=vol.device)
        lib = _lib.load()
        # training-step fast path (twin of the Siddon one): ray gradients wanted, static (packed) volume -> one march
        # yields the image and the per-ray sensitivities; backward is elementwise (b200drr_trilinear_bwd_sens)
        sens = None
        if (not fp64 and _FUSED_SENSITIVITIES and reduce == 0 and any(ctx.needs_input_grad[1:5])
                and not ctx.needs_input_grad[0]):
            sens = torch.empty(B, N, 12, dtype=torch.float32, device=vol.device)
        if vol.dtype in _VOL16 and sens is None and any(ctx.needs_input_grad[1:5]):
            raise NotImplementedError(f"ray gradients from a {vol.dtype} volume come from the fused sensitivities march only")
        with torch.cuda.device(vol.device):
            if fp64:   # b200drr_trilinear_fwd_f64 takes the arguments of b200drr_trilinear_fwd
                _lib.check(lib.b200drr_trilinear_fwd_f64(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B,
                                                         N, voxel_shift, eps, n_points, _ptr(arange), reduce,
                                                         int(align_corners), _stream()), "b200drr_trilinear_fwd_f64")
            elif sens is not None and packed is None:   # plain volume: arbitrary ray sets, or the grid without a packed copy
                h, w_ = grid if grid is not None else (0, 0)
                fn, head, name = _vol_entry(lib, "b200drr_trilinear_fwd_sens", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens), B, N, h, w_,
                              voxel_shift, eps, n_points, _ptr(arange), int(align_corners), _stream()), name)
            elif sens is not None:
                fn, head, name = _vol_entry(lib, "b200drr_trilinear_fwd_sens_packed", vol, packed)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), _ptr(sens), B, grid[0], grid[1],
                              voxel_shift, eps, n_points, _ptr(arange),
                              _PACKED_SLAB_SENS if B >= _PACKED_SLAB_MIN_BATCH else 0, _stream()), name)
            elif packed is not None:
                fn, head, name = _vol_entry(lib, "b200drr_trilinear_fwd_packed", vol, packed)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, grid[0], grid[1], voxel_shift,
                              eps, n_points, _ptr(arange), _PACKED_SLAB_FWD if B >= _PACKED_SLAB_MIN_BATCH else 0, _stream()),
                           name)
            elif grid is not None:
                fn, head, name = _vol_entry(lib, "b200drr_trilinear_fwd_grid", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, grid[0], grid[1], voxel_shift,
                              eps, n_points, _ptr(arange), 1, _stream()), name)
            else:
                fn, head, name = _vol_entry(lib, "b200drr_trilinear_fwd", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(out), B, N, voxel_shift, eps, n_points,
                              _ptr(arange), reduce, int(align_corners), _stream()), name)
        ctx.fused = sens is not None
        if ctx.fused:
            ctx.save_for_backward(sens)
        else:
            ctx.save_for_backward(vol, src, tgt, raylen, arange)
        ctx.packed = None if ctx.fused else packed
        ctx.cfg = (voxel_shift, eps, n_points, reduce, align_corners, grid)
        ctx.ray_shapes = (tuple(source.shape), tuple(img.shape))
        return out.view(B, 1, N)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        voxel_shift, eps, n_points, reduce, align_corners, grid = ctx.cfg
        need_ar = ctx.needs_input_grad[4]
        if ctx.fused:
            (sens,) = ctx.saved_tensors
            B, N = sens.shape[0], sens.shape[1]
            dev = sens.device
            gout = gout.reshape(B, N).contiguous().float()
            g_src, g_tgt, g_len = _ray_grads(ctx, B, N, torch.float32, dev)
            g_ar = torch.zeros(2, dtype=torch.float32, device=dev) if need_ar else None
            with torch.cuda.device(dev):
                _lib.check(_lib.load().b200drr_trilinear_bwd_sens(_ptr(sens), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len),
                                                                  _ptr(g_ar), B, N, _stream()), "b200drr_trilinear_bwd_sens")
            return (None, *_ray_grads_back(ctx, g_src, g_tgt, g_len), g_ar, None, None, None, None, None, None, None)
        vol, src, tgt, raylen, arange = ctx.saved_tensors
        fp64 = vol.dtype == torch.float64
        if fp64 and reduce != 0:
            raise NotImplementedError("fp64 trilinear: backward is implemented for reducefn='sum'")
        B, N = tgt.shape[0], tgt.shape[1]
        gout = gout.reshape(B, N).contiguous().to(torch.float64 if fp64 else torch.float32)
        dev = vol.device
        g_src, g_tgt, g_len = _ray_grads(ctx, B, N, gout.dtype, dev)
        g_vol = torch.zeros_like(vol) if ctx.needs_input_grad[0] else None
        g_ar = torch.zeros(2, dtype=gout.dtype, device=dev) if need_ar else None
        lib = _lib.load()
        with torch.cuda.device(dev):
            if fp64:   # b200drr_trilinear_bwd_f64 takes the arguments of b200drr_trilinear_bwd
                _lib.check(lib.b200drr_trilinear_bwd_f64(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                         _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), _ptr(g_ar), B, N,
                                                         voxel_shift, eps, n_points, _ptr(arange), int(align_corners),
                                                         _stream()), "b200drr_trilinear_bwd_f64")
            elif reduce != 0:  # reducefn="max": the first maximal sample carries the gradient
                _lib.check(lib.b200drr_trilinear_bwd_max(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                         _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), _ptr(g_ar), B, N,
                                                         voxel_shift, eps, n_points, _ptr(arange), int(align_corners),
                                                         _stream()), "b200drr_trilinear_bwd_max")
            elif ctx.packed is not None and g_vol is None:
                _lib.check(lib.b200drr_trilinear_bwd_packed(_ptr(ctx.packed), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                            _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_ar), B,
                                                            grid[0], grid[1], voxel_shift, eps, n_points, _ptr(arange),
                                                            0, _stream()), "b200drr_trilinear_bwd_packed")
            elif grid is not None:
                _lib.check(lib.b200drr_trilinear_bwd_grid(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                          _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol),
                                                          _ptr(g_ar), B, grid[0], grid[1], voxel_shift, eps, n_points,
                                                          _ptr(arange), 1, _stream()), "b200drr_trilinear_bwd_grid")
            else:
                _lib.check(lib.b200drr_trilinear_bwd(_ptr(vol), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen), _ptr(gout),
                                                     _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), _ptr(g_ar), B, N,
                                                     voxel_shift, eps, n_points, _ptr(arange), int(align_corners), _stream()),
                           "b200drr_trilinear_bwd")
        return (g_vol, *_ray_grads_back(ctx, g_src, g_tgt, g_len), g_ar, None, None, None, None, None, None, None)


def _trilinear_sens_pose(volume, packed, src, G, Wd, rows, cols, voxel_shift, eps, n_points, arange):
    """The sensitivities march of the in-kernel rays of a full detector grid through the packed-corner copy of `volume`
    (include/b200drr.h: b200drr_trilinear_fwd_sens_pose): -> (out (B, H*W), sens (B, H*W, 12)), the image and every ray's
    end-point and range sensitivities.  Inputs contiguous fp32."""
    B, H, W = G.shape[0], rows.numel(), cols.numel()
    out = torch.empty(B, H * W, dtype=torch.float32, device=packed.device)
    sens = torch.empty(B, H * W, 12, dtype=torch.float32, device=packed.device)
    fn, head, name = _vol_entry(_lib.load(), "b200drr_trilinear_fwd_sens_pose", volume, packed)
    with torch.cuda.device(packed.device):
        _lib.check(fn(*head, *volume.shape, _ptr(src), _ptr(G), _ptr(Wd), _ptr(rows), _ptr(cols), _ptr(out), _ptr(sens), B, H,
                      W, voxel_shift, eps, n_points, _ptr(arange), _PACKED_SLAB_SENS if B >= _PACKED_SLAB_MIN_BATCH else 0,
                      _stream()), name)
    return out, sens


class _TrilinearPoseFunction(torch.autograd.Function):
    """Trilinear line integrals of the full detector grid with the rays generated IN the kernel from per-pose 3x4 matrices
    (include/b200drr.h: b200drr_trilinear_fwd_sens_pose / _bwd_sens_pose): the training-step path of a STATIC (packed) volume;
    gradients come back as matrices + the two range partials, no (B,N,3) tensors exist."""

    @staticmethod
    def forward(ctx, volume, packed, src, G, Wd, rows, cols, alpha_range, voxel_shift, eps, n_points):
        B, H, W = G.shape[0], rows.numel(), cols.numel()
        src, G, Wd = src.contiguous().float(), G.contiguous().float(), Wd.contiguous().float()
        rows, cols = rows.contiguous().float(), cols.contiguous().float()
        arange = alpha_range.detach().to(device=packed.device, dtype=torch.float32).contiguous()
        out, sens = _trilinear_sens_pose(volume, packed, src, G, Wd, rows, cols, voxel_shift, eps, n_points, arange)
        ctx.save_for_backward(sens, Wd, rows, cols)
        return out.view(B, 1, H * W)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        sens, Wd, rows, cols = ctx.saved_tensors
        B, H, W = Wd.shape[0], rows.numel(), cols.numel()
        dev = sens.device
        gout = gout.reshape(B, H * W).contiguous().float()
        g_src = torch.empty(B, 3, dtype=torch.float32, device=dev)
        g_G = torch.empty(B, 3, 4, dtype=torch.float32, device=dev)
        g_Wd = torch.empty(B, 3, 4, dtype=torch.float32, device=dev)
        g_ar = torch.zeros(2, dtype=torch.float32, device=dev) if ctx.needs_input_grad[7] else None
        with torch.cuda.device(dev):
            _lib.check(_lib.load().b200drr_trilinear_bwd_sens_pose(_ptr(sens), _ptr(gout), _ptr(Wd), _ptr(rows), _ptr(cols),
                                                                   _ptr(g_src), _ptr(g_G), _ptr(g_Wd), _ptr(g_ar), B, H, W,
                                                                   _stream()), "b200drr_trilinear_bwd_sens_pose")
        return None, None, g_src, g_G, g_Wd, None, None, g_ar, None, None, None


def trilinear_pose_render(renderer, volume, packed, src, G, Wd, rows, cols, n_points):
    """Fused pose-in rendering for a `Trilinear` module with default options and a packed static volume (used by DRR.forward
    when pose gradients are wanted); -> (B, 1, H*W).  The batch-global sampling range (reference renderers.py:217-222) is found
    by a reduction kernel over the in-kernel rays, then rebuilt differentiably in torch from the TWO rays that attain it."""
    if volume.dtype in _VOL16:
        _check_vol16(volume, src, G)
    alpha_range, _ = pose_alpha_range(renderer, volume, src, G, Wd, rows, cols)
    return _TrilinearPoseFunction.apply(volume, packed, src, G, Wd, rows, cols, alpha_range, float(renderer.voxel_shift),
                                        float(renderer.eps), int(n_points))


def pose_alpha_range(renderer, volume, src, G, Wd, rows, cols):
    """(alpha_range [2], arg [2]): the batch-global sampling range of the in-kernel rays, differentiable in (src, G), and the
    linear ray index b*H*W + h*W + w of the ray attaining each end (see trilinear_pose_render)."""
    B, H, W = G.shape[0], rows.numel(), cols.numel()
    dev = volume.device
    src_c, G_c, Wd_c = src.detach().contiguous().float(), G.detach().contiguous().float(), Wd.detach().contiguous().float()
    rows_c, cols_c = rows.contiguous().float(), cols.contiguous().float()
    rng = torch.empty(2, dtype=torch.float32, device=dev)
    arg = torch.empty(2, dtype=torch.int64, device=dev)
    scratch = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200drr_trilinear_alpha_range_pose(*volume.shape, _ptr(src_c), _ptr(G_c), _ptr(Wd_c), _ptr(rows_c),
                                                                  _ptr(cols_c), _ptr(rng), _ptr(arg), _ptr(scratch), B, H, W,
                                                                  float(renderer.voxel_shift), float(renderer.eps), _stream()),
                   "b200drr_trilinear_alpha_range_pose")
    # the two extremal rays, rebuilt with torch ops so that autograd reaches the pose through the range as the reference's
    # `.min()` / `.max()` do (the gradient goes to the arg-min / arg-max ray); no host sync: indices stay on the device
    b, n = arg // (H * W), arg % (H * W)
    p = torch.stack([cols_c[n % W], rows_c[n // W], torch.ones(2, device=dev), torch.ones(2, device=dev)], dim=-1)  # (2, 4)
    tgt2 = torch.einsum("kij,kj->ki", G[b].float(), p).unsqueeze(1)            # (2, 1, 3)
    src2 = src[b].float().unsqueeze(1)                                           # (2, 1, 3)
    dims = _dims_tensor(volume.shape, dev, torch.float32)
    amin, amax = _get_alpha_minmax(src2, tgt2, dims, renderer.voxel_shift, renderer.eps)
    return torch.stack([amin[0, 0, 0], amax[1, 0, 0]]), arg


class _SegmentsFunction(torch.autograd.Function):
    """Un-reduced render for a CALLABLE `reducefn` (reference renderers.py:175-183 hands it the per-segment tensor):
    kind 0 = Siddon -> (B, N, D0+D1+D2+2) segments in the reference's sorted order, kind 1 = trilinear -> (B, N, n_points).
    include/b200drr.h: b200drr_segments_fwd / _bwd (reference-literal kernels, fp32 or fp64 after the volume's dtype)."""

    @staticmethod
    def forward(ctx, volume, source, target, img, alpha_range, kind, voxel_shift, eps, n_points, align_corners, stop_grad):
        dtype = volume.dtype
        B, N = _check_inputs(volume, source, target, img, dtype)
        vol, src = volume.contiguous(), source.reshape(B, 3).contiguous()
        tgt, raylen = target.contiguous(), img.reshape(B, N).contiguous()
        arange = None if alpha_range is None else alpha_range.detach().to(device=vol.device, dtype=dtype).contiguous()
        M = sum(vol.shape) + 2 if kind == 0 else int(n_points)
        out = torch.empty(B, N, M, dtype=dtype, device=vol.device)
        with torch.cuda.device(vol.device):
            _lib.check(_lib.load().b200drr_segments_fwd(kind, int(dtype == torch.float64), _ptr(vol), *vol.shape, _ptr(src), _ptr(tgt),
                                                        _ptr(raylen), _ptr(out), B, N, voxel_shift, eps, int(n_points),
                                                        _ptr(arange), int(align_corners), _stream()), "b200drr_segments_fwd")
        ctx.save_for_backward(vol, src, tgt, raylen, arange)
        ctx.cfg = (kind, voxel_shift, eps, int(n_points), align_corners, stop_grad)
        ctx.ray_shapes = (tuple(source.shape), tuple(img.shape))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gseg):
        kind, voxel_shift, eps, n_points, align_corners, stop_grad = ctx.cfg
        vol, src, tgt, raylen, arange = ctx.saved_tensors
        B, N = tgt.shape[0], tgt.shape[1]
        dev, dtype = vol.device, vol.dtype
        gseg = gseg.to(dtype).contiguous()
        g_src, g_tgt, g_len = _ray_grads(ctx, B, N, dtype, dev, stop_grad)
        g_vol = torch.zeros_like(vol) if (ctx.needs_input_grad[0] and not stop_grad) else None
        g_ar = torch.zeros(2, dtype=dtype, device=dev) if (ctx.needs_input_grad[4] and kind == 1) else None
        with torch.cuda.device(dev):
            _lib.check(_lib.load().b200drr_segments_bwd(kind, int(dtype == torch.float64), _ptr(vol), *vol.shape, _ptr(src), _ptr(tgt),
                                                        _ptr(raylen), _ptr(gseg), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol),
                                                        _ptr(g_ar), B, N, voxel_shift, eps, n_points, _ptr(arange), int(stop_grad),
                                                        int(align_corners), _stream()), "b200drr_segments_bwd")
        return (g_vol, *_ray_grads_back(ctx, g_src, g_tgt, g_len), g_ar, None, None, None, None, None, None)


def _mask_channels(mask: torch.Tensor) -> int:
    """Number of label channels, as the reference computes it (renderers.py:81; one host sync per call)."""
    return int(mask.max().item() + 1)


class _MaskFunction(torch.autograd.Function):
    """mask_to_channels rendering (B, C, N) through b200drr_*_fwd_mask; backward = b200drr_*_bwd_mask (the per-segment /
    per-sample upstream gradient is the gradient of the channel the label routed it to)."""

    @staticmethod
    def forward(ctx, volume, source, target, img, alpha_range, mask, kind, voxel_shift, eps, n_points, align_corners,
                stop_grad, C, grid=None):
        B, N = _check_inputs(volume, source, target, img)
        if grid is not None and grid[0] * grid[1] != N:
            grid = None
        vol, msk = volume.contiguous(), mask
        src, tgt, raylen = source.reshape(B, 3).contiguous(), target.contiguous(), img.reshape(B, N).contiguous()
        out = torch.empty(B, C, N, dtype=torch.float32, device=vol.device)
        lib = _lib.load()
        ar = None
        with torch.cuda.device(vol.device):
            if kind == "siddon" and grid is not None:   # full detector grid: tile-ordered threads (same per-ray results)
                _lib.check(lib.b200drr_siddon_fwd_mask_grid(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                            _ptr(out), B, grid[0], grid[1], C, voxel_shift, eps, _stream()),
                           "b200drr_siddon_fwd_mask_grid")
            elif kind == "siddon":
                _lib.check(lib.b200drr_siddon_fwd_mask(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                       _ptr(out), B, N, C, voxel_shift, eps, _stream()),
                           "b200drr_siddon_fwd_mask")
            elif grid is not None:
                ar = alpha_range.detach().to(device=vol.device, dtype=torch.float32).contiguous()
                _lib.check(lib.b200drr_trilinear_fwd_mask_grid(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt),
                                                               _ptr(raylen), _ptr(out), B, grid[0], grid[1], C, voxel_shift, eps,
                                                               int(n_points), _ptr(ar), int(align_corners), _stream()),
                           "b200drr_trilinear_fwd_mask_grid")
            else:
                ar = alpha_range.detach().to(device=vol.device, dtype=torch.float32).contiguous()
                _lib.check(lib.b200drr_trilinear_fwd_mask(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt),
                                                          _ptr(raylen), _ptr(out), B, N, C, voxel_shift, eps, int(n_points),
                                                          _ptr(ar), int(align_corners), _stream()),
                           "b200drr_trilinear_fwd_mask")
        ctx.save_for_backward(vol, msk, src, tgt, raylen, ar)
        ctx.cfg = (kind, voxel_shift, eps, n_points, align_corners, stop_grad, C, grid)
        ctx.ray_shapes = (tuple(source.shape), tuple(img.shape))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        vol, msk, src, tgt, raylen, ar = ctx.saved_tensors
        kind, voxel_shift, eps, n_points, align_corners, stop_grad, C, grid = ctx.cfg
        B, N = tgt.shape[0], tgt.shape[1]
        need_ar = ctx.needs_input_grad[4]
        dev = vol.device
        gout = gout.reshape(B, C, N).contiguous().float()
        g_src, g_tgt, g_len = _ray_grads(ctx, B, N, torch.float32, dev, stop_grad)
        g_vol = torch.zeros_like(vol) if (ctx.needs_input_grad[0] and not stop_grad) else None
        g_ar = None
        lib = _lib.load()
        with torch.cuda.device(dev):
            if kind == "siddon" and grid is not None:
                _lib.check(lib.b200drr_siddon_bwd_mask_grid(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                            _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), B,
                                                            grid[0], grid[1], C, voxel_shift, eps, int(stop_grad), _stream()),
                           "b200drr_siddon_bwd_mask_grid")
            elif kind == "siddon":
                _lib.check(lib.b200drr_siddon_bwd_mask(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt), _ptr(raylen),
                                                       _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len), _ptr(g_vol), B, N, C,
                                                       voxel_shift, eps, int(stop_grad), _stream()), "b200drr_siddon_bwd_mask")
            elif grid is not None:
                g_ar = torch.zeros(2, dtype=torch.float32, device=dev) if need_ar else None
                _lib.check(lib.b200drr_trilinear_bwd_mask_grid(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt),
                                                               _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len),
                                                               _ptr(g_vol), _ptr(g_ar), B, grid[0], grid[1], C, voxel_shift, eps,
                                                               int(n_points), _ptr(ar), int(align_corners), _stream()),
                           "b200drr_trilinear_bwd_mask_grid")
            else:
                g_ar = torch.zeros(2, dtype=torch.float32, device=dev) if need_ar else None
                _lib.check(lib.b200drr_trilinear_bwd_mask(_ptr(vol), _ptr(msk), *vol.shape, _ptr(src), _ptr(tgt),
                                                          _ptr(raylen), _ptr(gout), _ptr(g_src), _ptr(g_tgt), _ptr(g_len),
                                                          _ptr(g_vol), _ptr(g_ar), B, N, C, voxel_shift, eps, int(n_points),
                                                          _ptr(ar), int(align_corners), _stream()),
                           "b200drr_trilinear_bwd_mask")
        return (g_vol, *_ray_grads_back(ctx, g_src, g_tgt, g_len), g_ar, None, None, None, None, None, None, None, None, None)


def _render_mask(kind, volume, mask, source, target, img, voxel_shift, eps, n_points=None, alpha_range=None,
                 align_corners=False, stop_grad=False, grid=None):
    """mask_to_channels rendering -> (B, C, N), differentiable w.r.t. volume, rays, ray lengths (and the trilinear
    sampling range)."""
    if not mask.is_cuda or mask.shape != volume.shape:
        raise ValueError("mask must be a CUDA label volume with the shape of the density volume")
    msk = mask.detach().contiguous().float()
    if alpha_range is None:
        alpha_range = torch.zeros(2, dtype=torch.float32, device=volume.device)
    return _MaskFunction.apply(volume, source, target, img, alpha_range, msk, kind, float(voxel_shift), float(eps),
                               0 if n_points is None else int(n_points), bool(align_corners), bool(stop_grad),
                               _mask_channels(msk), grid)


_DIMS_CACHE: dict = {}


def _dims_tensor(shape, device, dtype) -> torch.Tensor:
    """Volume shape as a device tensor, built once per (shape, device, dtype): a host->device copy per call would be a
    sync point and cannot be captured in a CUDA graph."""
    key = (tuple(shape), str(device), dtype)
    t = _DIMS_CACHE.get(key)
    if t is None:
        t = _DIMS_CACHE[key] = torch.tensor(tuple(shape), dtype=dtype).to(device)
    return t


def _reduce_code(reducefn):
    if isinstance(reducefn, str) and reducefn in _REDUCE:
        return _REDUCE[reducefn]
    if isinstance(reducefn, Callable):
        return 2  # un-reduced render (_SegmentsFunction), then reducefn(img) as in reference renderers.py:175-183
    raise ValueError(f"Only supports reducefn 'sum' or 'max', not {reducefn}")


class Siddon(torch.nn.Module):
    """Differentiable X-ray renderer, Siddon's exact ray tracing -- fused sm_90a kernel (reference renderers.py:11-91)."""

    def __init__(self, voxel_shift: float = 0.5, mode: str = "nearest", stop_gradients_through_grid_sample: bool = False,
                 filter_intersections_outside_volume: bool = False, reducefn: str = "sum", eps: float = 1e-8):
        super().__init__()
        self.mode = mode
        self.stop_gradients_through_grid_sample = stop_gradients_through_grid_sample
        self.filter_intersections_outside_volume = filter_intersections_outside_volume
        self.reducefn = reducefn
        self.voxel_shift = voxel_shift
        self.eps = eps
        # (H, W) when the rays handed to forward() are the full row-major detector grid (set by DRR.render);
        # enables the tiled slab-major kernels.  None = arbitrary ray set (sub-sampled / patched / user rays).
        self.detector_shape = None
        # (pix_index (H*W,) int32, corners (B,3,3) voxel space, H, W, n_rays) when the rays are a SUB-SAMPLE of the detector grid
        # (one-shot hint set by DRR.forward): inference batches then take the brick-major kernel
        self.ray_subset = None

    def dims(self, volume):
        return _dims_tensor(volume.shape, volume.device, volume.dtype)

    def forward(self, volume, source, target, img, align_corners=False, mask=None):
        if self.mode not in ("nearest", "bilinear"):
            raise ValueError(f"mode must be 'nearest' or 'bilinear', not {self.mode!r}")
        if self.filter_intersections_outside_volume:
            # the reference crashes on this flag (renderers.py:118 calls _get_alpha_minmax with too few arguments)
            raise NotImplementedError("filter_intersections_outside_volume=True is broken in the reference and "
                                      "unnecessary here: the fused walk already clips to the volume")
        if volume.dtype in _VOL16:  # 16-bit volume storage (DESIGN.md 4.5): default options only
            if (mask is not None or self.mode != "nearest" or not isinstance(self.reducefn, str) or self.reducefn != "sum"
                    or align_corners):
                raise NotImplementedError(
                    f"a {volume.dtype} volume is rendered with the default Siddon options only (mode='nearest', reducefn='sum', "
                    "align_corners=False, no mask_to_channels); use an fp32 volume for the others")
            _check_vol16(volume, source, target)
        if _reduce_code(self.reducefn) == 2:  # callable: it receives the (B, N, M-1) segment tensor (renderers.py:175-183)
            if mask is not None or self.mode != "nearest":
                raise NotImplementedError("a callable reducefn is implemented for mode='nearest' without mask_to_channels")
            seg = _SegmentsFunction.apply(volume, source, target, img, None, 0, float(self.voxel_shift), float(self.eps), 0,
                                          bool(align_corners), bool(self.stop_gradients_through_grid_sample))
            return self.reducefn(seg).unsqueeze(1)
        if volume.dtype == torch.float64:  # `drr.to(torch.float64)` (reference drr.py:75): the reference-literal fp64 kernels
            if mask is not None or self.mode != "nearest":
                raise NotImplementedError("fp64 Siddon is implemented for mode='nearest' without mask_to_channels")
        elif mask is not None:
            if align_corners or _reduce_code(self.reducefn) != 0:
                raise NotImplementedError("mask_to_channels is implemented for reducefn='sum', align_corners=False")
            if self.mode != "nearest":
                raise NotImplementedError("mask_to_channels is implemented for mode='nearest'")
            return _render_mask("siddon", volume, mask, source, target, img, float(self.voxel_shift), float(self.eps),
                                stop_grad=self.stop_gradients_through_grid_sample, grid=self.detector_shape)
        # mode="bilinear" (trilinear sampling at the segment midpoints) is the general walk's mode 1
        return _SiddonFunction.apply(volume, source, target, img, float(self.voxel_shift), float(self.eps),
                                     _reduce_code(self.reducefn), bool(align_corners),
                                     bool(self.stop_gradients_through_grid_sample), self.detector_shape, self.ray_subset,
                                     int(self.mode == "bilinear"))


def siddon_pose_render(renderer, volume, src, G, Wd, rows, cols):
    """Fused pose-in rendering for a `Siddon` module with default options (used by DRR.forward); -> (B, 1, H*W)."""
    if volume.dtype in _VOL16:
        _check_vol16(volume, src, G)
    return _SiddonPoseFunction.apply(volume, src, G, Wd, rows, cols, float(renderer.voxel_shift), float(renderer.eps),
                                     bool(renderer.stop_gradients_through_grid_sample))


def _get_alpha_minmax(source, target, dims, voxel_shift, eps):
    """Per-ray entry/exit alphas of the slab test of reference renderers.py:124-140 (far plane dims + 1: quirk Q4)."""
    direction = target - source + eps
    lo_plane = -voxel_shift
    hi_plane = dims.to(source) + (1.0 - voxel_shift)
    a0 = (lo_plane - source) / direction
    a1 = (hi_plane - source) / direction
    alphamin = torch.minimum(a0, a1).amax(dim=-1, keepdim=True)
    alphamax = torch.maximum(a0, a1).amin(dim=-1, keepdim=True)
    return alphamin.clamp_min(0.0), alphamax.clamp_max(1.0)


class Trilinear(torch.nn.Module):
    """Differentiable X-ray renderer, trilinear ray marching -- fused sm_90a kernel (reference renderers.py:186-254)."""

    def __init__(self, voxel_shift: float = 0.5, mode: str = "bilinear", reducefn: str = "sum", eps: float = 1e-8):
        super().__init__()
        self.mode = mode
        self.reducefn = reducefn
        self.voxel_shift = voxel_shift
        self.eps = eps
        self.detector_shape = None  # (H, W) when the rays are the full row-major detector grid (set by DRR.render)
        # Packed-corner copy of a STATIC volume (8x its size, include/b200drr.h: b200drr_pack_corners): one 32-byte read
        # per sample instead of 8 gathers.  Built lazily, re-built when the volume tensor changes, skipped when the
        # volume is being optimised (requires_grad) or the copy would exceed `pack_corners_max_bytes`.
        self.pack_corners = True
        self.pack_corners_max_bytes = 24 * 2**30
        self._packed = None
        self._packed_key = None
        self._packed_src = None

    def dims(self, volume):
        return _dims_tensor(volume.shape, volume.device, volume.dtype)

    def invalidate_packed(self):
        """Drop the cached packed-corner copy (needed only after writes that bypass autograd's version counter)."""
        self._packed, self._packed_key, self._packed_src = None, None, None

    def _packed_volume(self, volume):
        if (not self.pack_corners or volume.requires_grad or not volume.is_cuda or volume.dim() != 3
                or volume.dtype not in (torch.float32, *_VOL16)):
            return None
        lib = _lib.load()
        n = int(lib.b200drr_packed_volume_floats(*volume.shape))   # 8 corners per cell, in the volume's own type
        if n * volume.element_size() > self.pack_corners_max_bytes:
            return None
        # The cache is tied to the tensor OBJECT (weak reference) and its in-place version counter: a temporary volume that
        # the caching allocator re-creates at the same address must not find a stale packed copy (ADVICE r1).  Writes
        # through `.data` bypass the version counter -- call `invalidate_packed()` after those.
        key = (volume._version, tuple(volume.shape), volume.device, volume.dtype)
        src = self._packed_src() if self._packed_src is not None else None
        if self._packed is None or src is not volume or self._packed_key != key:
            vol = volume.contiguous()
            try:
                # fp32: 32 B per cell; 16-bit: the corners stay 16-bit, 16 B per cell (include/b200drr.h: _v16 twins)
                packed = torch.empty(n * volume.element_size() // 4, dtype=torch.float32, device=vol.device)
            except torch.cuda.OutOfMemoryError:
                self._packed, self._packed_key, self._packed_src = None, None, None
                return None  # no room for the 8x copy: the gather kernels read the volume as stored
            with torch.cuda.device(vol.device):
                fn, head, name = _vol_entry(lib, "b200drr_pack_corners", vol)
                _lib.check(fn(*head, *vol.shape, _ptr(packed), _stream()), name)
            self._packed, self._packed_key, self._packed_src = packed, key, weakref.ref(volume)
        return self._packed

    def forward(self, volume, source, target, img, n_points=500, align_corners=False, mask=None, alphamin=None,
                alphamax=None):
        if self.mode != "bilinear":
            raise NotImplementedError("Trilinear kernels implement mode='bilinear' (the reference default) only")
        if volume.dtype in _VOL16:  # 16-bit volume storage (DESIGN.md 4.5): default options only
            if mask is not None or not isinstance(self.reducefn, str) or self.reducefn != "sum" or align_corners:
                raise NotImplementedError(
                    f"a {volume.dtype} volume is rendered with the default Trilinear options only (reducefn='sum', "
                    "align_corners=False, no mask_to_channels); use an fp32 volume for the others")
            _check_vol16(volume, source, target)
        if mask is not None and _reduce_code(self.reducefn) != 0:
            raise NotImplementedError("mask_to_channels is implemented for reducefn='sum'")
        if alphamin is None or alphamax is None:
            # batch-global sampling range over whatever rays are in this call (quirk Q3), differentiable torch ops
            dims = _dims_tensor(volume.shape, source.device, source.dtype)
            amin, amax = _get_alpha_minmax(source, target, dims, self.voxel_shift, self.eps)
            alphamin, alphamax = amin.min(), amax.max()
        if _reduce_code(self.reducefn) == 2:  # callable: it receives the (B, N, n_points) sample tensor
            if mask is not None:
                raise NotImplementedError("a callable reducefn is implemented without mask_to_channels")
            alpha_range = torch.stack([torch.as_tensor(alphamin, dtype=volume.dtype, device=volume.device),
                                       torch.as_tensor(alphamax, dtype=volume.dtype, device=volume.device)])
            smp = _SegmentsFunction.apply(volume, source, target, img, alpha_range, 1, float(self.voxel_shift), float(self.eps),
                                          int(n_points), bool(align_corners), False)
            return self.reducefn(smp).unsqueeze(1)
        fp64 = volume.dtype == torch.float64  # `drr.to(torch.float64)`: reference-literal fp64 kernels
        if fp64 and mask is not None:
            raise NotImplementedError("fp64 trilinear is implemented without mask_to_channels")
        dtype = torch.float64 if fp64 else torch.float32
        alpha_range = torch.stack([torch.as_tensor(alphamin, dtype=dtype, device=volume.device),
                                   torch.as_tensor(alphamax, dtype=dtype, device=volume.device)])
        if mask is not None:
            return _render_mask("trilinear", volume, mask, source, target, img, float(self.voxel_shift), float(self.eps),
                                n_points=n_points, alpha_range=alpha_range, align_corners=align_corners,
                                grid=self.detector_shape)
        return _TrilinearFunction.apply(volume, source, target, img, alpha_range, float(self.voxel_shift), float(self.eps),
                                        int(n_points), _reduce_code(self.reducefn), bool(align_corners),
                                        self.detector_shape,
                                        self._packed_volume(volume) if self.detector_shape is not None else None)


def siddon_visits(volume_shape, source, target, voxel_shift: float = 0.5, eps: float = 1e-8) -> torch.Tensor:
    """Voxels crossed per ray (B, N) int32 -- the unit of the algorithmic byte count (SURVEY.md 8d)."""
    B, N = target.shape[0], target.shape[1]
    src = source.reshape(B, 3).contiguous().float()
    tgt = target.contiguous().float()
    out = torch.empty(B, N, dtype=torch.int32, device=tgt.device)
    with torch.cuda.device(tgt.device):
        _lib.check(_lib.load().b200drr_siddon_visits(*volume_shape, _ptr(src), _ptr(tgt), _ptr(out), B, N, voxel_shift, eps,
                                                     _stream()), "b200drr_siddon_visits")
    return out
