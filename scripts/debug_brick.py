#!/usr/bin/env python
"""Debug helper: where does the brick kernel differ from the slab-major kernel? (B, D, H from the environment)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

os.environ.setdefault("SMALL", "0")
from diffdrr_b200 import _lib  # noqa: E402
from diffdrr_b200.renderers import _ptr, _stream  # noqa: E402

sys.argv = [sys.argv[0]]
import importlib.util  # noqa: E402

spec = importlib.util.spec_from_file_location("tb", os.path.join(os.path.dirname(__file__), "tune_brick.py"))
os.environ["BVARIANTS"] = os.environ.get("BVARIANTS", "0")
tb = importlib.util.module_from_spec(spec)
spec.loader.exec_module(tb)
lib, dev = tb.lib, tb.dev
D, H, B = tb.D, tb.H, tb.B
vol, src, tgt, raylen, dims = tb.vol, tb.src, tb.tgt, tb.raylen, tb.dims
N = H * H
ref = torch.empty(B, N, device=dev)
tb.grid_call(vol, dims, src, tgt, raylen, ref, B, H, H)
ws = torch.empty(lib.b200drr_siddon_brick_workspace_bytes(B, H, H), dtype=torch.uint8, device=dev)
for v in [int(x) for x in os.environ.get("DVARIANTS", "0").split(",")]:
    for rep in range(3):
        out = torch.zeros(B, N, device=dev)
        tb.brick_call(vol, dims, src, tgt, raylen, out, ws, B, H, H, v)
        torch.cuda.synchronize()
        d = (out - ref).abs() / ref.abs().max()
        bad = (d > 3e-5).nonzero()
        print(f"variant {v} rep {rep}: max {float(d.max()):.2e}  bad pixels {len(bad)}", end="  ")
        for b, n in bad[:6].tolist():
            print(f"(b={b}, py={n // H}, px={n % H}, got={float(out[b, n]):.5f}, ref={float(ref[b, n]):.5f})", end=" ")
        print(flush=True)
