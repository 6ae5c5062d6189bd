"""ctypes binding of libb200drr.so -- the C ABI declared in include/b200drr.h.

There is NO fallback: if the CUDA library is missing or an entry point fails, this raises.  Tensors are
passed as raw device pointers (`tensor.data_ptr()`), the stream as `torch.cuda.current_stream().cuda_stream`.
"""
from __future__ import annotations

import ctypes
import os

from . import build as _build

_c_float_p = ctypes.c_void_p
_SIGNATURES = {
    "b200drr_version": (ctypes.c_int, []),
    "b200drr_error_string": (ctypes.c_char_p, [ctypes.c_int]),
    "b200drr_device_sm_count": (ctypes.c_int, []),
    "b200drr_device_cc": (ctypes.c_int, []),
    "b200drr_siddon_fwd": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_grid": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_grid": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
        ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_fwd": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_bwd": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float,
        ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_grid": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_trilinear_bwd_grid": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
        ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_pose": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_siddon_bwd_pose": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int,
        ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_sens": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_siddon_fwd_sens_grid": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_sens": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_siddon_fwd_sens_pose": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_siddon_bwd_sens_pose": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_sens": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p,
        ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_sens_packed": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_trilinear_bwd_sens": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64,
        ctypes.c_void_p]),
    "b200drr_trilinear_alpha_range_pose": (ctypes.c_int, [
        ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_sens_pose": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int,
        _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_bwd_sens_pose": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_euler_pose_fwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, _c_float_p, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_euler_pose_bwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_void_p]),
    "b200drr_pose_rays_fwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_pose_rays_bwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_mask": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_mask": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_siddon_fwd_mask_grid": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_mask_grid": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p,
        ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_general": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_int,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_general": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int,
        ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_bwd_max": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float,
        ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_mask": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_float,
        ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_bwd_mask": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int,
        ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_mask_grid": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
        ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_bwd_mask_grid": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
        ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_packed_volume_floats": (ctypes.c_int64, [ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "b200drr_pack_corners": (ctypes.c_int, [_c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_packed": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_trilinear_bwd_packed": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
        ctypes.c_float, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_f64": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int,
        ctypes.c_int64, ctypes.c_double, ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_f64": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double, ctypes.c_double, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]),
    "b200drr_trilinear_fwd_f64": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int,
        ctypes.c_int64, ctypes.c_double, ctypes.c_double, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_trilinear_bwd_f64": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double,
        ctypes.c_double, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_segments_fwd": (ctypes.c_int, [
        ctypes.c_int, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double, ctypes.c_double, ctypes.c_int, _c_float_p, ctypes.c_int,
        ctypes.c_void_p]),
    "b200drr_segments_bwd": (ctypes.c_int, [
        ctypes.c_int, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double,
        ctypes.c_double, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_fwd_sorted": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int,
        ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_siddon_fwd_sens_sorted": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_siddon_brick_workspace_bytes": (ctypes.c_int64, [ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "b200drr_siddon_fwd_brick": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
        ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_bwd_vol_brick": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
        ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_siddon_fwd_brick_subset": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, _c_float_p,
        _c_float_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_float,
        ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_siddon_visits": (ctypes.c_int, [
        ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int,
        ctypes.c_int64, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b200drr_ncc_workspace_bytes": (ctypes.c_int64, [ctypes.c_int, ctypes.c_int, ctypes.c_int64]),
    "b200drr_ncc_fwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, _c_float_p,
        _c_float_p, ctypes.c_void_p]),
    "b200drr_ncc_bwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64,
        ctypes.c_void_p]),
    "b200drr_local_ncc_workspace_bytes": (ctypes.c_int64, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "b200drr_local_ncc_fwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
        ctypes.c_void_p, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "b200drr_local_ncc_bwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "b200drr_sobel_workspace_bytes": (ctypes.c_int64, [ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "b200drr_sobel_fwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_sobel_bwd": (ctypes.c_int, [
        _c_float_p, _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, ctypes.c_int, ctypes.c_void_p,
        ctypes.c_void_p]),
}

# entry points of rejected experiments (include/b200drr_experimental.h): bound only when the experimental build is loaded
_EXPERIMENTAL_SIGNATURES = {
    "b200drr_x_transpose_volume": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, ctypes.c_void_p]),
    "b200drr_x_siddon_fwd_chunk": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
    "b200drr_x_siddon_sens_chunk": (ctypes.c_int, [
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
        _c_float_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]),
}

_lib = None


class B200DRRError(RuntimeError):
    pass


def lib_path() -> str:
    # B200DRR_LIB: an alternative build of the same C ABI (kernel A/B experiments from scripts/); default = the in-tree build
    return os.environ.get("B200DRR_LIB") or _build.LIB_PATH


def load():
    """Load (once) and return the ctypes handle; raises if the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.exists(path):
            raise B200DRRError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). diffdrr_b200 has no CPU or PyTorch fallback.")
        handle = ctypes.CDLL(path)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the ABI and the header drift apart
            fn.restype = restype
            fn.argtypes = argtypes
        for name, (restype, argtypes) in _EXPERIMENTAL_SIGNATURES.items():
            if hasattr(handle, name):
                fn = getattr(handle, name)
                fn.restype = restype
                fn.argtypes = argtypes
        _lib = handle
    return _lib


def check(code: int, what: str) -> None:
    if code != 0:
        msg = load().b200drr_error_string(code)
        raise B200DRRError(f"{what} failed with code {code}: {msg.decode() if msg else '?'}")


def exported_symbols():
    return sorted(_SIGNATURES)
