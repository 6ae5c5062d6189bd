"""The training step's sensitivities walk cut into bricks (csrc/siddon_brick.cu, SENS mode) on the CPU: every (ray, brick) pair runs
the exact-frame walk of the slab kernels on a zero-filled copy of the brick, and the pairs must add up to the un-cut walk -- the
image, the ray-length gradient and, per axis, the end-point gradients (a crossing coefficient attributed to the wrong axis moves
gradient between the components of g_target without changing the image)."""
import numpy as np
import pytest

from conftest import relerr
from hostemu import emu
from hostemu import emu_brick_sens


@pytest.mark.parametrize("brick", [(3, 4, 4), (5, 2, 7)])
@pytest.mark.parametrize("seed", [0, 1])
def test_brick_pairs_equal_the_uncut_walk_on_exact_ties(brick, seed):
    """Dyadic geometry (as test_major_axis_pieces_equal_the_uncut_walk_on_exact_ties): every plane alpha is exact in fp32, so rays
    run through voxel edges and corners and, with bricks this small, through brick edges and corners -- cuts on two or three axes
    at one alpha."""
    rng = np.random.default_rng(seed)
    for _ in range(12):
        dims = tuple(int(x) for x in rng.integers(8, 40, 3))
        g = np.meshgrid(*[np.linspace(-1, 1, d) for d in dims], indexing="ij")
        vol = (np.exp(-(g[0] ** 2 + (g[1] - 0.2) ** 2 + g[2] ** 2) / 0.5) + 0.3 * rng.random(dims)).astype(np.float32)
        n = 300
        d = rng.choice([32.0, 64.0, 128.0], size=(n, 3)) * rng.choice([-1.0, 1.0], size=(n, 3))
        through = np.stack([rng.integers(0, dims[a] + 1, n).astype(np.float64) for a in range(3)], 1) - 0.5   # a lattice point
        through += rng.choice([0.0, 0.0, 0.25, 0.5], size=(n, 1)) * rng.choice([0.0, 1.0], size=(n, 3))
        src = through - d * rng.integers(1, 4, size=(n, 1)) * 0.25
        s, t = src.astype(np.float32).reshape(n, 1, 3), (src + 2.0 * d).astype(np.float32).reshape(n, 1, 3)   # one ray per "pose"
        l = np.linalg.norm(t - s, axis=-1).reshape(n, 1, 1).astype(np.float32)
        w = np.ones((n, 1, 1), np.float32)
        whole = emu.siddon_sens(vol, s, t, l, w, slab=0)
        cut = emu_brick_sens.siddon_sens_brick(vol, s, t, l, w, brick=brick)
        assert cut["pairs"] > n
        for key in ("img", "g_target", "g_source", "g_raylen"):
            assert relerr(cut[key], whole[key]) < 1e-5, (dims, brick, key)


def test_brick_pairs_equal_the_uncut_walk_on_the_bench_rays():
    """512^3 -> 256^2, pose 1 of the bench's pose set, detector rows 45-70 (rays through voxel edges on the cuts of the major-axis
    pieces, test_major_axis_pieces_keep_every_crossing_coefficient_on_its_axis) with the production 24 x 32 x 32 bricks."""
    import torch
    from diffdrr_b200 import DRR, synthetic
    from diffdrr_b200.pose import convert
    D, H = 512, 256
    x = torch.linspace(-1, 1, D)
    vol = torch.exp(-((x[:, None, None] - 0.1) ** 2 + (x[None, :, None] + 0.2) ** 2 + x[None, None, :] ** 2) / 0.3).numpy()
    subj = synthetic.make_subject(torch.zeros(1, 1, 1, 1))
    subj.volume.affine = synthetic.make_affine(D)
    drr = DRR(subj, **synthetic.detector_kwargs(H))
    rot, xyz = synthetic.make_poses(2, seed=0)
    with torch.no_grad():
        src, tgt = drr.detector(convert(rot[1:], xyz[1:], parameterization="euler_angles", convention="ZXY"), None)
        raylen = (tgt - src).norm(dim=-1).unsqueeze(1)
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
    rows = slice(45 * H, 71 * H)
    s, t, l = src.numpy(), tgt[:, rows].numpy(), raylen[:, :, rows].numpy()
    w = np.ones_like(l)
    whole = emu.siddon_sens(vol, s, t, l, w, slab=0)
    cut = emu_brick_sens.siddon_sens_brick(vol, s, t, l, w, brick=(24, 32, 32))
    for key in ("img", "g_target", "g_source", "g_raylen"):
        assert relerr(cut[key], whole[key]) < 1e-5, key
    # per component of every ray's end-point sensitivities, not only the maximum over the batch
    ref = whole["g_target"].reshape(-1, 3)
    err = np.abs(cut["g_target"].reshape(-1, 3) - ref).max(axis=1) / np.abs(ref).max()
    assert err.max() < 1e-5, (int(err.argmax()), float(err.max()))
