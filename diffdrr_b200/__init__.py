"""diffdrr_b200 -- a Hopper-native (sm_90a) differentiable DRR projector with DiffDRR's `DRR` module surface.

Hot path (Siddon + trilinear renderers, forward and backward) = hand-written CUDA kernels behind the C ABI of
include/b200drr.h; host code (pose, detector geometry, module plumbing) = PyTorch.  No CPU fallback.
"""
__version__ = "0.1.0"

from .detector import Detector  # noqa: F401
from .drr import DRR  # noqa: F401
from .pose import RigidTransform, convert  # noqa: F401
from .renderers import Siddon, Trilinear  # noqa: F401
from .metrics import (  # noqa: F401,E402
    DoubleGeodesicSE3, GradientNormalizedCrossCorrelation2d, LogGeodesicSE3, MultiscaleNormalizedCrossCorrelation2d,
    MutualInformation, NormalizedCrossCorrelation2d, Sobel)
from .registration import (  # noqa: F401,E402
    DeformableLevenbergMarquardt, DiffeomorphicLevenbergMarquardt, LevenbergMarquardt, PolyrigidLevenbergMarquardt, Registration,
    StructuresLevenbergMarquardt)
from .structures import structures_jacobian  # noqa: F401,E402
from .polyrigid import polyrigid_jacobian, polyrigid_weights  # noqa: F401,E402
from .deform import deformed_jvp  # noqa: F401,E402
from .svf import exp_velocity, exp_velocity_jvp  # noqa: F401,E402
