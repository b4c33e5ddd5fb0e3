"""The reference's training losses (model_training/losses) over libdad3d.so, with their gradients.

``IoULoss``, ``LandmarksLossWVisibility``, ``ReprojectionLoss`` and ``Vertices3DLoss`` take the reference's constructor
arguments and ``forward`` inputs, and are what config/loss/train_loss.yaml instantiates; the per-loss weights and their sum
stay in the reference's own ``LossModule`` (train/loss_module.py).  Each forward is a ``torch.autograd.Function`` over the
kernels of csrc/loss.cu, so the objective backpropagates to all three network outputs (heat-map logits, 2D landmarks and
3DMM parameters).  The 3DMM parameters reach the vertices through ``HeadMesh.decode_with_grad`` (the hi/lo decode forward,
``dad3d_flame_backward`` backward).  Every tensor must be on a CUDA device; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Union

import numpy as np
import torch
import torch.nn as nn
from torch import Tensor

from . import _lib
from .flame_assets import indices_reweighing
from .head_mesh import HeadMesh

__all__ = ["Vertices3DLoss", "ReprojectionLoss", "LandmarksLossWVisibility", "IoULoss", "VertexSubsets",
           "vertex_subset_loss"]

_CRITERIA = {"l1": _lib.DAD3D_LOSS_L1, "l2": _lib.DAD3D_LOSS_L2, "smooth_l1": _lib.DAD3D_LOSS_SMOOTH_L1}


def _criterion(name: str) -> int:
    if name not in _CRITERIA.keys():
        raise ValueError(f"Unsupported discrepancy loss type {name}")
    return _CRITERIA[name]


def _f32(t: Tensor, device: torch.device) -> Tensor:
    if not t.is_cuda or t.device != device:
        raise _lib.Dad3dError(f"the losses need every tensor on {device} (there is no CPU path), got {t.device}")
    return t.detach().to(torch.float32).contiguous()


def _stream(device: torch.device):
    return torch.cuda.current_stream(device).cuda_stream


class VertexSubsets:
    """The ordered (weight, index set) pairs of a vertex-subset loss -- what ``indices_reweighing`` returns -- as
    ``dad3d_vsub`` tables, one per CUDA device.  Any index sets work (nested, overlapping, repeated indices); negative
    indices count from the end, as in ``v[:, i]``."""

    def __init__(self, indices: Sequence, weights: Sequence[float], n_vertices: int):
        if len(indices) != len(weights) or len(indices) == 0:
            raise ValueError("VertexSubsets needs one weight per index set and at least one set")
        sets = []
        for i in indices:
            a = np.asarray(i).reshape(-1).astype(np.int64)
            if a.size == 0:
                raise ValueError("VertexSubsets: an index set is empty")
            if a.min() < -n_vertices or a.max() >= n_vertices:
                raise IndexError(f"VertexSubsets: index out of range for {n_vertices} vertices")
            sets.append(np.where(a < 0, a + n_vertices, a))
        self.n_vertices = int(n_vertices)
        self.sizes = [int(a.size) for a in sets]
        self._idx = np.ascontiguousarray(np.concatenate(sets).astype(np.int32))
        self._off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int32))
        self._w = np.ascontiguousarray(np.asarray(weights, dtype=np.float32))
        self._handles: Dict[int, C.c_void_p] = {}
        self.lib = _lib.load()

    @property
    def num_sets(self) -> int:
        return len(self.sizes)

    def handle(self, device: torch.device) -> C.c_void_p:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        h = self._handles.get(idx)
        if h is None:
            h = C.c_void_p()
            _lib.check(self.lib.dad3d_vsub_create(C.byref(h), self._idx.ctypes.data, self._off.ctypes.data,
                                                  self._w.ctypes.data, self.num_sets, self.n_vertices, idx),
                       "dad3d_vsub_create")
            self._handles[idx] = h
        return h

    def __del__(self):
        for h in getattr(self, "_handles", {}).values():
            try:
                self.lib.dad3d_vsub_destroy(h)
            except Exception:
                pass
        self._handles = {}


class _VertexSubsetFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v: Tensor, target: Tensor, subsets: VertexSubsets, criterion: int, normalize: bool):
        dev = v.device
        v32, t32 = _f32(v, dev), _f32(target, dev)
        if v32.ndim != 3 or v32.shape[1] != subsets.n_vertices or v32.shape[2] not in (2, 3) or t32.shape != v32.shape:
            raise ValueError(f"vertex-subset loss: prediction {tuple(v.shape)} and target {tuple(target.shape)} must both be "
                             f"[B, {subsets.n_vertices}, 2 or 3]")
        B, _, K = v32.shape
        rec = torch.empty(B, subsets.num_sets, _lib.DAD3D_VSUB_RECORD_FLOATS, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(subsets.lib.dad3d_vsub_forward(subsets.handle(dev), v32.data_ptr(), t32.data_ptr(), B, K,
                                                      int(normalize), criterion, rec.data_ptr(), loss.data_ptr(),
                                                      _stream(dev)), "dad3d_vsub_forward")
        ctx.save_for_backward(v32, t32, rec)
        ctx.subsets, ctx.criterion, ctx.normalize, ctx.v_dtype = subsets, criterion, normalize, v.dtype
        return loss

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        v32, t32, rec = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None
        dev = v32.device
        g = grad_out.detach().to(device=dev, dtype=torch.float32).contiguous()
        grad = torch.empty_like(v32)
        B, _, K = v32.shape
        with torch.cuda.device(dev):
            _lib.check(ctx.subsets.lib.dad3d_vsub_backward(ctx.subsets.handle(dev), v32.data_ptr(), t32.data_ptr(), B, K,
                                                           int(ctx.normalize), ctx.criterion, rec.data_ptr(), g.data_ptr(),
                                                           grad.data_ptr(), _stream(dev)), "dad3d_vsub_backward")
        return grad.to(ctx.v_dtype), None, None, None, None


def vertex_subset_loss(v: Tensor, target: Tensor, subsets: VertexSubsets, criterion: str, normalize: bool) -> Tensor:
    """sum_s w_s * mean criterion(f(v[:, I_s]) - f(target[:, I_s])) over ``subsets``, f = normalize_to_cube
    (model/utils.py:55-68) when ``normalize`` else the identity; differentiable in ``v`` [B, V, 2 or 3]."""
    return _VertexSubsetFunction.apply(v, target, subsets, _criterion(criterion), bool(normalize))


class _IoUFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, t: Tensor):
        dev = x.device
        x32, t32 = _f32(x, dev), _f32(t, dev)
        if x.ndim < 2 or t32.shape != x32.shape or x32.numel() == 0:
            raise ValueError(f"IoULoss: prediction {tuple(x.shape)} and target {tuple(t.shape)} must be the same [B, C, ...]")
        planes = x32.shape[0] * x32.shape[1]
        hw = x32.numel() // planes
        stats = torch.empty(planes, 4, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        lib = _lib.load()
        with torch.cuda.device(dev):
            _lib.check(lib.dad3d_iou_forward(x32.data_ptr(), t32.data_ptr(), planes, hw, stats.data_ptr(), loss.data_ptr(),
                                             _stream(dev)), "dad3d_iou_forward")
        ctx.save_for_backward(x32, t32, stats)
        ctx.x_dtype = x.dtype
        return loss

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x32, t32, stats = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None
        dev = x32.device
        g = grad_out.detach().to(device=dev, dtype=torch.float32).contiguous()
        grad = torch.empty_like(x32)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().dad3d_iou_backward(x32.data_ptr(), t32.data_ptr(), stats.shape[0],
                                                      x32.numel() // stats.shape[0], stats.data_ptr(), g.data_ptr(),
                                                      grad.data_ptr(), _stream(dev)), "dad3d_iou_backward")
        return grad.to(ctx.x_dtype), None


class _LandmarksFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p: Tensor, pm: Tensor, t: Tensor, tm: Tensor, criterion: int):
        dev = p.device
        p32, pm32, t32, tm32 = (_f32(a, dev) for a in (p, pm, t, tm))
        if p32.ndim != 3 or p32.shape[2] != 2 or t32.shape != p32.shape or pm32.shape != p32.shape[:2] \
                or tm32.shape != p32.shape[:2] or p32.numel() == 0:
            raise ValueError(f"LandmarksLossWVisibility: landmarks {tuple(p.shape)}, {tuple(t.shape)} must be [B, N, 2] and "
                             f"presences {tuple(pm.shape)}, {tuple(tm.shape)} [B, N]")
        B, N, _ = p32.shape
        partial = torch.empty(B, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().dad3d_landmarks_forward(p32.data_ptr(), pm32.data_ptr(), t32.data_ptr(), tm32.data_ptr(),
                                                           B, N, criterion, partial.data_ptr(), loss.data_ptr(),
                                                           _stream(dev)), "dad3d_landmarks_forward")
        ctx.save_for_backward(p32, pm32, t32, tm32)
        ctx.criterion, ctx.p_dtype = criterion, p.dtype
        return loss

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        p32, pm32, t32, tm32 = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None
        dev = p32.device
        g = grad_out.detach().to(device=dev, dtype=torch.float32).contiguous()
        grad = torch.empty_like(p32)
        B, N, _ = p32.shape
        with torch.cuda.device(dev):
            _lib.check(_lib.load().dad3d_landmarks_backward(p32.data_ptr(), pm32.data_ptr(), t32.data_ptr(), tm32.data_ptr(),
                                                            B, N, ctx.criterion, g.data_ptr(), grad.data_ptr(), _stream(dev)),
                       "dad3d_landmarks_backward")
        return grad.to(ctx.p_dtype), None, None, None, None


class IoULoss(nn.Module):
    """losses/keypoint_losses.py:5-31: 1 - mean over (b, c) of the soft IoU of sigmoid(y_pred) and y_true."""

    def forward(self, y_pred: Tensor, y_true: Tensor) -> Tensor:
        return _IoUFunction.apply(y_pred, y_true)


class LandmarksLossWVisibility(nn.Module):
    """losses/landmarks_loss_w_visibility.py:10-26: criterion(p * p_presence, t * t_presence); only p gets a gradient."""

    def __init__(self, criterion):
        super().__init__()
        self._criterion = _criterion(criterion)
        self.criterion_name = criterion

    def forward(self, predicted: List[Tensor], target: List[Tensor]) -> Tensor:
        """predicted, target: [Tensor[B,N,2] of landmarks, Tensor[B,N] of their presence]."""
        return _LandmarksFunction.apply(predicted[0], predicted[1], target[0], target[1], self._criterion)


class Vertices3DLoss(nn.Module):
    """losses/vertices_3d_loss.py:14-48: sum over the weighted subsets of the criterion between normalize_to_cube of the
    predicted (zero rotation) and the target vertices [B, V, 3]."""

    def __init__(self, criterion, batch_size, consts, weights_and_indices):
        super().__init__()
        self._criterion = _criterion(criterion)
        self.criterion_name = criterion
        self.head_mesh = HeadMesh(flame_config=consts, batch_size=batch_size)
        self.weights, self.indices = indices_reweighing(weights_and_indices)
        self.subsets = VertexSubsets(self.indices, self.weights, int(self.head_mesh.flame.v_template.shape[0]))

    def forward(self, predicted: Tensor, target: Tensor) -> Tensor:
        """predicted: [B, num_params] 3DMM parameters; target: [B, V, 3] vertices."""
        v3, _ = self.head_mesh.decode_with_grad(predicted, zero_rotation=True)
        return _VertexSubsetFunction.apply(v3, target, self.subsets, self._criterion, True)


class ReprojectionLoss(nn.Module):
    """losses/reprojection_loss.py:13-46: sum over the weighted subsets of the criterion between the reprojected 2D vertices
    and the target [B, V, 2] (or a list whose first element it is).  Like the reference, zeroes translation z of
    ``predicted`` in place (head_mesh.py:41), recorded by autograd."""

    def __init__(self, criterion, batch_size, consts, img_size, weights_and_indices):
        super().__init__()
        self._criterion = _criterion(criterion)
        self.criterion_name = criterion
        self.weights, self.indices = indices_reweighing(weights_and_indices)
        self.head_mesh = HeadMesh(flame_config=consts, batch_size=batch_size, image_size=img_size)
        self.subsets = VertexSubsets(self.indices, self.weights, int(self.head_mesh.flame.v_template.shape[0]))

    def forward(self, predicted: Tensor, target: Union[Tensor, List[Tensor]]) -> Tensor:
        _, projected = self.head_mesh.decode_with_grad(predicted, to_2d=True)
        self.head_mesh.flame_params(predicted).translation[..., 2] = 0.0
        full_target = target[0] if isinstance(target, list) else target
        return _VertexSubsetFunction.apply(projected, full_target, self.subsets, self._criterion, False)
