"""reference path: model_training/metrics/keypoints.py: FailureRate and KeypointsNME over dad_3dheads_b200.metrics."""
from typing import Any, Callable, Dict, Optional

import torch
from torch import Tensor
from torchmetrics import Metric

from dad_3dheads_b200.metrics import keypoints_nme, percentage_of_errors_below_IOD

__all__ = ["FailureRate", "KeypointsNME", "keypoints_nme", "percentage_of_errors_below_IOD"]


def _inputs(gts: Dict[str, Tensor]):
    """(keypoints, bboxes or None) of the reference's ``gts`` dict (keypoints.py:12-16)."""
    return gts["keypoints"], gts.get("bboxes")


class FailureRate(Metric):
    """The mean over updates of each batch's share of heads whose keypoint error is below (``below``) or above
    ``threshold`` times the box norm (keypoints.py:55-110): states ``failure_rate`` and ``total``, summed across processes."""

    def __init__(self, compute_on_step: bool = True, dist_sync_on_step: bool = False, process_group: Optional[Any] = None,
                 dist_sync_fn: Callable = None, threshold: float = 0.05, below: bool = True):
        super().__init__(compute_on_step=compute_on_step, dist_sync_on_step=dist_sync_on_step, process_group=process_group,
                         dist_sync_fn=dist_sync_fn)
        self.threshold = threshold
        self.below = below
        self.add_state("failure_rate", default=torch.tensor(0.0), dist_reduce_fx="sum")
        self.add_state("total", default=torch.tensor(0.0), dist_reduce_fx="sum")

    def update(self, pred_keypoints: Tensor, gts: Dict[str, Tensor]) -> None:
        """pred_keypoints [B, N, 2 or 3]; gts {"keypoints": [B, N, 2 or 3], "bboxes": int32 [B, 4] (optional)}."""
        keypoints, bboxes = _inputs(gts)
        rate = percentage_of_errors_below_IOD(pred_keypoints, keypoints, bboxes, threshold=self.threshold, below=self.below)
        self.failure_rate = self.failure_rate.to(rate.device) + rate
        self.total = self.total.to(rate.device) + 1

    def compute(self) -> Tensor:
        return self.failure_rate / self.total


class KeypointsNME(Metric):
    """``weight`` times the mean over updates of each batch's NME (keypoints.py:113-152): states ``nme`` and ``total``,
    summed across processes."""

    def __init__(self, compute_on_step: bool = True, dist_sync_on_step: bool = False, process_group: Optional[Any] = None,
                 dist_sync_fn: Callable = None, weight: int = 100):
        super().__init__(compute_on_step=compute_on_step, dist_sync_on_step=dist_sync_on_step, process_group=process_group,
                         dist_sync_fn=dist_sync_fn)
        self.weight = weight
        self.add_state("nme", default=torch.tensor(0.0), dist_reduce_fx="sum")
        self.add_state("total", default=torch.tensor(0.0), dist_reduce_fx="sum")

    def update(self, pred_keypoints: Tensor, gts: Dict[str, Tensor]) -> None:
        """pred_keypoints [B, N, 2 or 3]; gts {"keypoints": [B, N, 2 or 3], "bboxes": int32 [B, 4] (optional)}."""
        keypoints, bboxes = _inputs(gts)
        nme = keypoints_nme(pred_keypoints, keypoints, bboxes)
        self.nme = self.nme.to(nme.device) + nme
        self.total = self.total.to(nme.device) + 1

    def compute(self) -> Tensor:
        return self.weight * (self.nme / self.total)
