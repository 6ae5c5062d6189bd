#!/bin/bash
# Memory check of the walk logic WITHOUT a GPU: builds tests/hostemu (the product's per-ray device math compiled for the CPU) with
# AddressSanitizer and walks random + exact-tie rays through exact-size heap volumes with the forward / sensitivities walks cut into
# major-axis pieces, slabs and un-cut -- an out-of-bounds voxel read (a start voxel or tail step outside its box) aborts the run.
# The device-side twin is scripts/sanitize_small.py under compute-sanitizer.
set -e
cd "$(dirname "$0")/.."
g++ -O1 -g -fsanitize=address -fno-omit-frame-pointer -ffp-contract=off -fPIC -shared -std=c++17 -Wno-unknown-pragmas \
    -o /tmp/libhostemu_asan.so tests/hostemu/hostemu.cpp
LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python - <<'PY'
import ctypes, sys
import numpy as np
sys.path.insert(0, "."); sys.path.insert(0, "tests")
from hostemu import emu
emu._lib = ctypes.CDLL("/tmp/libhostemu_asan.so")
rng = np.random.default_rng(3)
tot = 0
for trial in range(60):
    dims = tuple(int(x) for x in rng.integers(8, 40, 3))
    vol = rng.random(dims).astype(np.float32)
    n = 200
    if trial % 2:   # dyadic geometry: every crossing ties with another one
        d = rng.choice([32.0, 64.0, 128.0], size=(n, 3)) * rng.choice([-1.0, 1.0], size=(n, 3))
        through = np.stack([rng.integers(0, dims[a] + 1, n).astype(np.float64) for a in range(3)], 1) - 0.5
        src = through - d * rng.integers(1, 4, size=(n, 1)) * 0.25
        tgt = src + 2 * d
    else:
        c = np.array(dims) / 2.0
        src = c + rng.normal(size=(n, 3)) * 3 * max(dims)
        tgt = c - (src - c) * 0.8 + rng.normal(size=(n, 3)) * max(dims) * 0.4
    s, t = src.astype(np.float32).reshape(n, 1, 3), tgt.astype(np.float32).reshape(n, 1, 3)
    l = np.linalg.norm(t - s, axis=-1).reshape(n, 1, 1).astype(np.float32)
    w = np.ones((n, 1, 1), np.float32)
    for slab in (-int(rng.integers(2, 45)), int(rng.integers(2, 9)), 0):
        emu.siddon_sens(vol, s, t, l, w, slab=slab)
        tot += n
    emu.siddon_fwd_lean_pieces(vol, s, t, l, int(rng.integers(2, 45)))
print("AddressSanitizer: clean;", tot, "sensitivity walks + forward walks")
PY
