"""reference path: model_training/losses (losses/__init__.py): the training losses of config/loss/train_loss.yaml, computed
with their gradients by the package's CUDA kernels."""
from dad_3dheads_b200.losses import IoULoss, LandmarksLossWVisibility, ReprojectionLoss, Vertices3DLoss

__all__ = ["Vertices3DLoss", "ReprojectionLoss",
           "LandmarksLossWVisibility", "IoULoss"]
