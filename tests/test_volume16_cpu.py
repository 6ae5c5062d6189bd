"""16-bit volumes on the CPU (DESIGN.md 4.5): the kernels' fp16 / bf16 -> fp32 conversion against numpy for every bit pattern, the
Siddon walks reading a 16-bit volume through the templated header code against the fp32 walks on the up-cast volume (bit for bit),
the argument checks of the _v16 entry points, and the accuracy of 16-bit storage against the fp32 goldens of the reference."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden, relerr
from hostemu import emu_volume16
from oracle import oracle

ALL_BITS = np.arange(65536, dtype=np.uint32).astype(np.uint16)


def _same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def test_fp16_conversion_equals_numpy_for_every_bit_pattern():
    """subnormals, +-0, +-inf and NaN payloads included: the host decoder is bit-exact to numpy's float16 -> float32."""
    ours = emu_volume16.vox16_to_f32(ALL_BITS, bf16=False)
    ref = ALL_BITS.view(np.float16).astype(np.float32)
    assert _same_bits(ours, ref)
    assert np.isnan(ours[0x7e00]) and ours[0x7c00] == np.inf and ours[0xfc00] == -np.inf and ours[0x0001] == 2.0 ** -24


def test_bf16_conversion_is_the_top_half_of_an_fp32_for_every_bit_pattern():
    ours = emu_volume16.vox16_to_f32(ALL_BITS, bf16=True)
    ref = (ALL_BITS.astype(np.uint32) << 16).view(np.float32)
    assert _same_bits(ours, ref)
    # and torch's bfloat16 agrees (the storage the module hands to the kernels)
    t = torch.from_numpy(ALL_BITS.astype(np.int16)).view(torch.bfloat16).float().numpy()
    assert _same_bits(ours, t)


def _bits(vol, dtype):
    return torch.from_numpy(vol).to(dtype).view(torch.int16).numpy().view(np.uint16)


def _upcast(vol, dtype):
    return torch.from_numpy(vol).to(dtype).float().numpy()


@pytest.mark.parametrize("dtype,name", [(torch.float16, "float16"), (torch.bfloat16, "bfloat16")])
@pytest.mark.parametrize("seed", [0, 1])
def test_16bit_walks_equal_the_fp32_walks_on_the_upcast_volume(dtype, name, seed):
    """Dyadic ray geometry (exact ties through voxel and brick edges) over a volume with values across the 16-bit range: the lean
    walk, the sensitivities walk and the brick-pair decomposition of both give the same floats, in the same order, from the 16-bit
    storage as from its fp32 up-cast."""
    rng = np.random.default_rng(seed)
    dims = tuple(int(x) for x in rng.integers(10, 30, 3))
    vol = (rng.standard_normal(dims) * np.exp(rng.uniform(-12, 8, dims))).astype(np.float32)
    vol[rng.random(dims) < 0.1] = 0.0
    if name == "float16":
        vol = np.clip(vol, -60000, 60000)
    n = 200
    d = rng.choice([32.0, 64.0, 128.0], size=(n, 3)) * rng.choice([-1.0, 1.0], size=(n, 3))
    through = np.stack([rng.integers(0, dims[a] + 1, n).astype(np.float64) for a in range(3)], 1) - 0.5
    through += rng.uniform(0, 1, size=(n, 3)) * rng.choice([0.0, 1.0], size=(n, 1))
    src = through - d * 0.5
    s, t = src.astype(np.float32).reshape(n, 1, 3), (src + 2.0 * d).astype(np.float32).reshape(n, 1, 3)  # one ray per "pose"
    ref = emu_volume16.siddon_walks(_upcast(vol, dtype), "float32", s, t, brick=(5, 4, 7))
    out = emu_volume16.siddon_walks(_bits(vol, dtype), name, s, t, brick=(5, 4, 7))
    assert np.abs(ref["lean"]).max() > 0
    for key in ("lean", "sens", "brick_fwd", "brick_sens"):
        assert _same_bits(out[key], ref[key]), key


def test_16bit_walks_at_the_production_brick_shape():
    """The production 24 x 32 x 32 bricks over a 48 x 40 x 72 volume (D2 % 8 == 0), rays of a detector-like fan."""
    rng = np.random.default_rng(3)
    dims = (48, 40, 72)
    vol = rng.random(dims, dtype=np.float32) * 2.0
    n = 256
    s = np.array([[[-60.0, 20.0, 36.0]]], np.float32)
    t = np.stack([np.full(n, 120.0), rng.uniform(-5, 45, n), rng.uniform(-5, 77, n)], -1).astype(np.float32)[None]
    for dtype, name in ((torch.float16, "float16"), (torch.bfloat16, "bfloat16")):
        ref = emu_volume16.siddon_walks(_upcast(vol, dtype), "float32", s, t)
        out = emu_volume16.siddon_walks(_bits(vol, dtype), name, s, t)
        for key in ("lean", "sens", "brick_fwd", "brick_sens"):
            assert _same_bits(out[key], ref[key]), (name, key)


def test_v16_entry_points_reject_bad_arguments_without_gpu():
    from diffdrr_b200 import _lib
    from diffdrr_b200 import build as b200build

    b200build.build()
    lib = _lib.load()
    n = None
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    for vt in (1, 2):  # all-NULL calls
        assert lib.b200drr_siddon_fwd_v16(n, vt, 4, 4, 4, n, n, n, n, 1, 1, 0.5, 1e-8, 0, 0, n) == -1
        assert lib.b200drr_siddon_fwd_sens_v16(n, vt, 4, 4, 4, n, n, n, n, n, 1, 1, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_sorted_v16(n, vt, 4, 4, 4, n, n, n, n, 1, 1, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_sens_sorted_v16(n, vt, 4, 4, 4, n, n, n, n, n, 1, 1, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_grid_v16(n, vt, 4, 4, 4, n, n, n, n, 1, 2, 2, 0.5, 1e-8, 0, n) == -1
        assert lib.b200drr_siddon_fwd_sens_grid_v16(n, vt, 4, 4, 4, n, n, n, n, n, 1, 2, 2, 0.5, 1e-8, 0, n) == -1
        assert lib.b200drr_siddon_fwd_brick_v16(n, vt, 4, 4, 8, n, n, n, n, n, n, n, n, n, 0, 1, 2, 2, 0.5, 1e-8, 0, n) == -1
        assert lib.b200drr_siddon_fwd_brick_subset_v16(n, vt, 4, 4, 8, n, n, n, n, n, n, n, 0, 1, 2, 2, 4, 0.5, 1e-8, 0, n) == -1
        assert lib.b200drr_siddon_fwd_pose_v16(n, vt, 4, 4, 4, n, n, n, n, n, n, 1, 2, 2, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_sens_pose_v16(n, vt, 4, 4, 4, n, n, n, n, n, n, n, 1, 2, 2, 0.5, 1e-8, n) == -1
    # valid-looking pointers: a bad voxel type, or an option outside the default kernels, is refused before any CUDA call
    for vt in (0, 3, -1):
        assert lib.b200drr_siddon_fwd_v16(p, vt, 4, 4, 4, p, p, p, p, 1, 1, 0.5, 1e-8, 0, 0, n) == -1
        assert lib.b200drr_siddon_fwd_sens_v16(p, vt, 4, 4, 4, p, p, p, p, p, 1, 1, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_sorted_v16(p, vt, 4, 4, 4, p, p, p, p, 1, 1, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_sens_sorted_v16(p, vt, 4, 4, 4, p, p, p, p, p, 1, 1, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_grid_v16(p, vt, 4, 4, 4, p, p, p, p, 1, 2, 2, 0.5, 1e-8, 0, n) == -1
        assert lib.b200drr_siddon_fwd_sens_grid_v16(p, vt, 4, 4, 4, p, p, p, p, p, 1, 2, 2, 0.5, 1e-8, 0, n) == -1
        assert lib.b200drr_siddon_fwd_brick_v16(p, vt, 4, 4, 8, p, p, p, n, n, n, n, p, p, 1 << 20, 1, 2, 2, 0.5, 1e-8, 0,
                                                n) == -1
        assert lib.b200drr_siddon_fwd_brick_subset_v16(p, vt, 4, 4, 8, p, p, p, p, p, p, p, 1 << 20, 1, 2, 2, 4, 0.5, 1e-8, 0,
                                                       n) == -1
        assert lib.b200drr_siddon_fwd_pose_v16(p, vt, 4, 4, 4, p, p, p, p, p, p, 1, 2, 2, 0.5, 1e-8, n) == -1
        assert lib.b200drr_siddon_fwd_sens_pose_v16(p, vt, 4, 4, 4, p, p, p, p, p, p, p, 1, 2, 2, 0.5, 1e-8, n) == -1
    assert lib.b200drr_siddon_fwd_v16(p, 1, 4, 4, 4, p, p, p, p, 1, 1, 0.5, 1e-8, 1, 0, n) == -1   # reducefn="max"
    assert lib.b200drr_siddon_fwd_v16(p, 2, 4, 4, 4, p, p, p, p, 1, 1, 0.5, 1e-8, 0, 1, n) == -1   # align_corners
    # the brick twins run the production shape only: a tuning variant is refused before any CUDA call
    assert lib.b200drr_siddon_fwd_brick_v16(p, 1, 96, 96, 96, p, p, p, n, n, n, n, p, p, 1 << 30, 1, 2, 2, 0.5, 1e-8, 7, n) == -2
    assert lib.b200drr_siddon_fwd_brick_subset_v16(p, 2, 96, 96, 96, p, p, p, p, p, p, p, 1 << 30, 1, 2, 2, 4, 0.5, 1e-8, 7,
                                                   n) == -2
    # Trilinear twins
    for vt in (1, 2):
        assert lib.b200drr_pack_corners_v16(n, vt, 4, 4, 4, n, n) == -1
        assert lib.b200drr_trilinear_fwd_v16(n, vt, 4, 4, 4, n, n, n, n, 1, 1, 0.5, 1e-8, 10, n, 0, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_grid_v16(n, vt, 4, 4, 4, n, n, n, n, 1, 2, 2, 0.5, 1e-8, 10, n, 1, n) == -1
        assert lib.b200drr_trilinear_fwd_sens_v16(n, vt, 4, 4, 4, n, n, n, n, n, 1, 4, 0, 0, 0.5, 1e-8, 10, n, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_packed_v16(n, vt, 4, 4, 4, n, n, n, n, 1, 2, 2, 0.5, 1e-8, 10, n, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_sens_packed_v16(n, vt, 4, 4, 4, n, n, n, n, n, 1, 2, 2, 0.5, 1e-8, 10, n, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_sens_pose_v16(n, vt, 4, 4, 4, n, n, n, n, n, n, n, 1, 2, 2, 0.5, 1e-8, 10, n, 0, n) == -1
    for vt in (0, 3):
        assert lib.b200drr_pack_corners_v16(p, vt, 4, 4, 4, p, n) == -1
        assert lib.b200drr_trilinear_fwd_v16(p, vt, 4, 4, 4, p, p, p, p, 1, 1, 0.5, 1e-8, 10, p, 0, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_grid_v16(p, vt, 4, 4, 4, p, p, p, p, 1, 2, 2, 0.5, 1e-8, 10, p, 1, n) == -1
        assert lib.b200drr_trilinear_fwd_sens_v16(p, vt, 4, 4, 4, p, p, p, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_packed_v16(p, vt, 4, 4, 4, p, p, p, p, 1, 2, 2, 0.5, 1e-8, 10, p, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_sens_packed_v16(p, vt, 4, 4, 4, p, p, p, p, p, 1, 2, 2, 0.5, 1e-8, 10, p, 0, n) == -1
        assert lib.b200drr_trilinear_fwd_sens_pose_v16(p, vt, 4, 4, 4, p, p, p, p, p, p, p, 1, 2, 2, 0.5, 1e-8, 10, p, 0, n) == -1
    assert lib.b200drr_trilinear_fwd_v16(p, 1, 4, 4, 4, p, p, p, p, 1, 1, 0.5, 1e-8, 10, p, 1, 0, n) == -1   # reducefn="max"
    assert lib.b200drr_trilinear_fwd_sens_v16(p, 2, 4, 4, 4, p, p, p, p, p, 1, 4, 0, 0, 0.5, 1e-8, 10, p, 1, n) == -1  # align_corners


# ---- accuracy of 16-bit storage ---------------------------------------------------------------------------------------------------
# The C oracle renders the golden volumes rounded to fp16 / bf16 (with fp32 geometry and sums, as the kernels do); its error against
# the reference's fp32 images is the cost of the storage alone.  Measured (max-abs error / max-abs of the fp32 golden image):
#   fp16: 0.73e-4 .. 1.62e-4      bf16: 4.4e-4 .. 7.6e-4
# so neither fits the 1e-4 budget of the fp32 kernels: fp16 exceeds it by up to 1.6x, bf16 by up to 7.6x.  The GPU tests
# (test_gpu_volume16.py) recompute this error per case and allow it plus ACCURACY_MARGIN (the fp32 kernels' own agreement with the
# oracle is far below that).
SIDDON_GOLDENS = [("siddon_nc_b4", {}), ("siddon_nc_b4_ragged", {}), ("siddon_nc_inside", {}), ("siddon_c1", {}),
                  ("siddon_nc_axis", {}), ("siddon_nc_b4_shift0", dict(voxel_shift=0.0))]
MEASURED_MAX = {torch.float16: 1.7e-4, torch.bfloat16: 8.0e-4}
ACCURACY_MARGIN = 2e-5


def storage_error(name, kw, dtype):
    g = load_golden(name)
    out = oracle.siddon_fwd(_upcast(g["volume"], dtype), g["source"], g["target"], g["raylen"], **kw)
    return relerr(out, g["img_f32"])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name,kw", SIDDON_GOLDENS)
def test_storage_error_against_the_fp32_goldens(name, kw, dtype):
    err = storage_error(name, kw, dtype)
    assert 0 < err < MEASURED_MAX[dtype], (name, dtype, err)
    if dtype == torch.bfloat16:
        assert err > 1e-4  # bf16 storage does NOT meet the fp32 budget: it is documented, not hidden


# Trilinear: the same storage error through the C oracle's trilinear march.  Measured (max-abs error / max-abs of the fp32 golden):
#   fp16: 0.54e-4 .. 1.25e-4      bf16: 1.6e-4 .. 4.9e-4
# (fp16 meets the 1e-4 budget on four of the five cases, bf16 on none); test_gpu_volume16.py recomputes it per case and allows it
# plus ACCURACY_MARGIN.
TRILINEAR_GOLDENS = [("trilinear_nc_b4", 160), ("trilinear_nc_b4_ragged", 77), ("trilinear_nc_inside", 150), ("trilinear_c1", 500),
                     ("trilinear_nc_axis", 200)]
TRILINEAR_MEASURED_MAX = {torch.float16: 1.3e-4, torch.bfloat16: 5.2e-4}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name,n_points", TRILINEAR_GOLDENS)
def test_trilinear_storage_error_against_the_fp32_goldens(name, n_points, dtype):
    g = load_golden(name)
    out = oracle.trilinear_fwd(_upcast(g["volume"], dtype), g["source"], g["target"], g["raylen"], n_points=n_points)
    err = relerr(out, g["img_f32"])
    assert 0 < err < TRILINEAR_MEASURED_MAX[dtype], (name, dtype, err)
