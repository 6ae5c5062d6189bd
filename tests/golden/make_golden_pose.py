#!/usr/bin/env python
"""Records the UNMODIFIED reference's pose conversions (diffdrr/pose.py: RigidTransform.convert, convert, get_se3_log) for
tests/test_pose_cpu.py.  Usage: python tests/golden/make_golden_pose.py <directory that contains the reference's diffdrr/>
Needs scipy: the reference's pose.py imports it (for its random-pose helper, which this script does not call)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, os.path.dirname(TESTS))
sys.path.insert(0, os.path.join(TESTS, "_refshim"))
sys.path.insert(0, sys.argv[1])
import diffdrr.pose as ref  # noqa: E402  (the reference's own module)

from diffdrr_b200.pose import PARAMETERIZATIONS, convert  # noqa: E402

g = torch.Generator().manual_seed(3)
rot = (torch.rand(6, 3, generator=g) * 2 - 1) * 1.2
xyz = (torch.rand(6, 3, generator=g) * 2 - 1) * 200.0
matrix = convert(rot, xyz, parameterization="euler_angles", convention="ZXY").matrix
rec = {"matrix": matrix.numpy(), "se3_log": ref.RigidTransform(matrix.clone()).get_se3_log().numpy()}
for param in PARAMETERIZATIONS:
    if param == "matrix":
        continue
    kw = dict(convention="ZXY") if param == "euler_angles" else {}
    theirs = ref.RigidTransform(matrix.clone()).convert(param, **kw)
    for i, a in enumerate(theirs):
        rec[f"{param}_{i}"] = a.numpy()
    rec[f"{param}_matrix"] = ref.convert(*theirs, parameterization=param, **kw).matrix.numpy()
np.savez_compressed(os.path.join(HERE, "pose_reference.npz"), **rec)
print({k: v.shape for k, v in rec.items()})
