"""The side limit of the brick kernel's per-ray frame record (csrc/brick.cuh, kSensFrameMaxSide = 1024: the entry voxel index is
packed into 10 bits per axis).  A volume whose longest side is at the limit runs through the brick kernel and matches the
slab-major kernel; one voxel more is refused by the brick kernel and routed to the slab kernels by the library's default."""
import pytest
import torch

from conftest import relerr
from gpu_common import DEV
from test_gpu_brick_sens import SLAB, _rays, _same_as_slab, _sens

pytestmark = pytest.mark.gpu


def _volume(D0):
    from diffdrr_b200 import synthetic
    return synthetic.make_volume((D0, 256, 256), "smooth", seed=4)


def test_frame_record_at_the_side_limit():
    H, B = 64, 4
    vol_np = _volume(1024)
    src, tgt, raylen = _rays(vol_np, H, B, seed=4, cubic=False)
    out, _ = _same_as_slab(torch.as_tensor(vol_np).to(DEV), src, tgt, raylen, H, H)
    assert out.abs().max() > 0


def test_side_above_the_limit_takes_the_slab_kernels():
    H, B = 64, 4
    vol_np = _volume(1025)
    src, tgt, raylen = _rays(vol_np, H, B, seed=4, cubic=False)
    vol = torch.as_tensor(vol_np).to(DEV)
    with pytest.raises(RuntimeError):
        _sens(42, vol, src, tgt, raylen, H, H)  # the brick kernel refuses the shape
    torch.cuda.synchronize()
    out0, sens0 = _sens(0, vol, src, tgt, raylen, H, H)  # default: 1025 x 256 x 256 at 4 poses is a brick shape but for the side
    out_s, sens_s = _sens(SLAB, vol, src, tgt, raylen, H, H)
    assert out0.abs().max() > 0
    assert relerr(out0.cpu().numpy(), out_s.cpu().numpy()) < 5e-5
    s0, ss = sens0.cpu().numpy(), sens_s.cpu().numpy()
    for k in range(7):
        assert relerr(s0[..., k], ss[..., k]) < 1e-4, k
