"""The host emulation of the brick kernel's sensitivities work lists (tests/hostemu/hostemu_brick_sens_refill.cpp), which DESIGN
§4.2b uses to weigh the chunk schedule of the walk against per-lane refill: the rounds it builds must hold every (ray, brick)
pair that passes the hit test exactly once, and the refill schedule must claim every item of every round exactly once."""
import numpy as np
import pytest

from hostemu import emu_brick_sens, emu_brick_sens_refill


def _bench_like_rays(D, H, B):
    from bench import make_host_rays
    src, tgt, raylen = make_host_rays(D, H, B, seed=0)
    return src.reshape(B, 3), tgt, raylen


@pytest.mark.parametrize("thresh", [1, 16])
def test_rounds_hold_every_pair_once_and_refill_claims_each_once(thresh):
    D, H, B = 64, 64, 4
    src, tgt, raylen = _bench_like_rays(D, H, B)
    vol = np.random.default_rng(0).random((D, D, D), dtype=np.float32)
    pairs = emu_brick_sens.siddon_sens_brick(vol, src, tgt, raylen, np.ones_like(raylen))["pairs"]
    r = emu_brick_sens_refill.schedule(src, tgt, H, H, (D, D, D), thresh=thresh)
    assert r["items"] == pairs > 0
    assert r["rounds_ok"] == r["rounds"] > 0
    assert r["lanesteps_ideal"] <= min(r["lanesteps_a"], r["lanesteps_b"])
    assert r["setups_a"] >= r["items"] / 32
