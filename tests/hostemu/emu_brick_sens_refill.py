"""ctypes front-end of tests/hostemu/libhostemu_brick_sens_refill.so: the brick kernel's sensitivities work lists rebuilt on the
CPU, scheduled as 32-item chunks (today's walk) and with per-lane refill (test infra).

    python tests/hostemu/emu_brick_sens_refill.py [--poses 16] [--brick-step 1]

prints the bench geometry's counts (512^3 -> 256^2, 24 x 32 x 32 bricks, U = 6) for several refill thresholds."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhostemu_brick_sens_refill.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None

# Warp instructions per piece of the fp32 SENS instantiation at U = 6 (cuobjdump -sass, major axis 0): the pair's set-up from
# its item to the first walk group (record and ray-table loads, start_walk_in_frame, lean_init), the chunk claim, one U-step
# group, and the exit tail with the flush.
SASS_COST = dict(setup=315, claim=30, group=185, tail=100)


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "hostemu_brick_sens_refill.cpp")] + [
            os.path.join(_ROOT, "diffdrr_b200", "csrc", f) for f in ("common.cuh", "ray_math.cuh", "brick.cuh")]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17",
                                   "-Wno-unknown-pragmas", "-o", _SO, srcs[0]])
        _lib = ctypes.CDLL(_SO)
        _lib.emu_brick_sens_schedule.restype = ctypes.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def schedule(src, tgt, H, W, dims, brick=(24, 32, 32), thresh=1, brick_step=1, cost=None, shift=0.5, eps=1e-8):
    """Counts of the two schedules over every round of every brick (every brick_step-th brick): dict with issue_a / issue_b
    (warp instructions from `cost`), lanesteps_a / lanesteps_b, setups_a / setups_b, items, rounds, rounds_ok (rounds whose
    items the refill schedule claimed exactly once each) mismatched (items whose walk's major axis is not their key's) and
    lanesteps_ideal (the steps of every pair's own groups: no lane ever idle)."""
    src, tgt = (np.ascontiguousarray(x, dtype=np.float32) for x in (src, tgt))
    cost = np.asarray([(cost or SASS_COST)[k] for k in ("setup", "claim", "group", "tail")], np.float32)
    out = np.zeros(11, np.float64)
    lib().emu_brick_sens_schedule(_p(src), _p(tgt), ctypes.c_int(tgt.shape[0]), ctypes.c_int(H), ctypes.c_int(W),
                                  *map(ctypes.c_int, dims), ctypes.c_float(shift), ctypes.c_float(eps), *map(ctypes.c_int, brick),
                                  _p(cost), ctypes.c_int(thresh), ctypes.c_int(brick_step), _p(out))
    keys = ("issue_a", "issue_b", "lanesteps_a", "lanesteps_b", "setups_a", "setups_b", "items", "rounds_ok", "rounds",
            "mismatched", "lanesteps_ideal")
    return dict(zip(keys, out.tolist()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=16)
    ap.add_argument("--brick-step", type=int, default=1)
    ap.add_argument("--thresh", type=int, nargs="+", default=[1, 4, 8, 16, 24])
    args = ap.parse_args()
    sys.path.insert(0, _ROOT)
    from bench import make_host_rays
    D, H = 512, 256
    src, tgt, _ = make_host_rays(D, H, args.poses, seed=0)
    for th in args.thresh:
        r = schedule(src.reshape(-1, 3), tgt, H, H, (D, D, D), thresh=th, brick_step=args.brick_step)
        r["thresh"] = th
        r["lanesteps_b_over_a"] = r["lanesteps_b"] / r["lanesteps_a"]
        r["issue_b_over_a"] = r["issue_b"] / r["issue_a"]
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
