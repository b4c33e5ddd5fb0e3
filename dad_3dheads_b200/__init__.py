"""dad_3dheads_b200 -- H100-native (sm_90a) DAD-3DNet image->3D-head hot path.

Host side is Python/PyTorch (device memory, streams, torch.distributed); all arithmetic on the path runs in
hand-written CUDA behind the C ABI of ``libdad3d.so`` (include/dad3d.h).  There is no CPU fallback: importing the
compute classes without the built library, or calling them without a Hopper GPU, raises.
"""
from .flame import FLAME_CONSTS, FlameParams, FLAMELayer  # noqa: F401
from .head_mesh import HeadMesh  # noqa: F401
from .heads import FlameHeads, FrozenBackboneRegression  # noqa: F401
from .losses import IoULoss, LandmarksLossWVisibility, ReprojectionLoss, Vertices3DLoss  # noqa: F401
from .metrics import FlameStepMetrics  # noqa: F401
from .training_data import FlameBatchBuilder, FlameDataset  # noqa: F401

__all__ = ["FLAME_CONSTS", "FlameBatchBuilder", "FlameDataset", "FlameHeads", "FlameParams", "FlameStepMetrics", "FLAMELayer",
           "FrozenBackboneRegression", "HeadMesh", "IoULoss",
           "LandmarksLossWVisibility", "ReprojectionLoss", "Vertices3DLoss"]
