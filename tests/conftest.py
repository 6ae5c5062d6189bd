import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a; select with `-m gpu`)")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a box without CUDA skips the gpu-marked tests instead of failing at the first kernel call."""
    try:
        import torch

        has_cuda = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100, sm_90a)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """Golden record (dict of numpy arrays) recorded from the unmodified reference by make_golden.py."""
    rec = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    key = str(rec.pop("volume_key"))
    if key == "rand64":
        from diffdrr_b200 import synthetic

        rec["volume"] = synthetic.make_volume(64, "rand", seed=0)
    else:
        rec["volume"] = np.load(os.path.join(GOLDEN, "volumes.npz"))[key]
    return rec


def relerr(a, b):
    """max-abs error normalised by the reference's max-abs (never per-pixel relative: background is 0)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.fixture(scope="session")
def golden():
    return load_golden
