"""reference path: model_training/metrics (metrics/__init__.py): the training step's metrics, computed by the package's
CUDA kernels (dad_3dheads_b200/metrics.py).  The classes subclass torchmetrics.Metric, as the reference's do, so they need
torchmetrics; the functions do not."""
from dad_3dheads_b200.metrics import keypoints_nme, percentage_of_errors_below_IOD, soft_iou

from .iou import SoftIoUMetric
from .keypoints import FailureRate, KeypointsNME

__all__ = ["SoftIoUMetric", "FailureRate", "KeypointsNME", "soft_iou", "keypoints_nme", "percentage_of_errors_below_IOD"]
