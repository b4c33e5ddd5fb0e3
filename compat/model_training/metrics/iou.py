"""reference path: model_training/metrics/iou.py: SoftIoUMetric over dad_3dheads_b200.metrics.soft_iou."""
from typing import Any, Callable, Optional

import torch
from torch import Tensor
from torchmetrics import Metric

from dad_3dheads_b200.metrics import soft_iou

__all__ = ["soft_iou", "SoftIoUMetric"]


class SoftIoUMetric(Metric):
    """The mean over updates of each batch's soft IoU (iou.py:34-72): states ``ious`` and ``total``, summed across
    processes."""

    def __init__(self, compute_on_step: bool = True, dist_sync_on_step: bool = False, process_group: Optional[Any] = None,
                 dist_sync_fn: Callable = None):
        super().__init__(compute_on_step=compute_on_step, dist_sync_on_step=dist_sync_on_step, process_group=process_group,
                         dist_sync_fn=dist_sync_fn)
        self.add_state("ious", default=torch.tensor(0.0), dist_reduce_fx="sum")
        self.add_state("total", default=torch.tensor(0.0), dist_reduce_fx="sum")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """preds: probabilities [B, C, H, W]; target: the target heat-maps, same shape."""
        self.ious = self.ious.to(preds.device) + soft_iou(preds, target)
        self.total = self.total.to(preds.device) + 1

    def compute(self) -> Tensor:
        return self.ious / self.total
