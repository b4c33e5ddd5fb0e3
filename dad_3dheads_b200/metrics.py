"""The reference's training metrics (model_training/metrics) and the metric block of its training step, over libdad3d.so.

``soft_iou``, ``keypoints_nme`` and ``percentage_of_errors_below_IOD`` take the reference's signatures (metrics/iou.py:15-31,
metrics/keypoints.py:19-52) and return 0-dim fp32 device tensors ([B] for ``keypoints_nme(..., reduce != "mean")``).
``FlameStepMetrics`` is the metric block of ``FlameLightningModel._step_fn`` (train/flame_lightning_model.py:299-357): the
ten values it logs per batch, and their batch-size-weighted epoch means.  All arithmetic runs in the kernels of
csrc/metrics.cu; every tensor must be on a CUDA device (there is no CPU path), and nothing synchronises with the host.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .encoder import OUTPUT_2D_LANDMARKS, OUTPUT_3DMM_PARAMS, OUTPUT_LANDMARKS_HEATMAP
from .flame import load_flame_static
from .head_mesh import HeadMesh
from .training_data import (INPUT_BBOX_KEY, TARGET_2D_FULL_LANDMARKS, TARGET_2D_LANDMARKS, TARGET_2D_LANDMARKS_PRESENCE,
                            TARGET_3D_MODEL_VERTICES, TARGET_LANDMARKS_HEATMAP)

__all__ = ["soft_iou", "keypoints_nme", "percentage_of_errors_below_IOD", "FlameStepMetrics"]

def _device_tensor(t, name: str, device: Optional[torch.device] = None) -> Tensor:
    if not isinstance(t, Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(t).__name__}")
    if not t.is_cuda or (device is not None and t.device != device):
        raise _lib.Dad3dError(f"the metrics need every tensor on a CUDA device{'' if device is None else f' ({device})'} "
                              f"(there is no CPU path); {name} is on {t.device}")
    return t


def _check_float(t, name: str) -> Tensor:
    if not isinstance(t, Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(t).__name__}")
    if not t.is_floating_point():
        raise TypeError(f"{name} must be a floating-point tensor, got {t.dtype}")
    return t


def _float(t, name: str, device: Optional[torch.device] = None) -> Tensor:
    t = _device_tensor(_check_float(t, name), name, device)
    return t.detach().to(torch.float32).contiguous()


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _box_columns(bbox, B: int, device: torch.device) -> Tuple[Tensor, Tensor]:
    """The widths and heights of ``bbox``: a [B, 4] int32 tensor (x, y, w, h) or a sequence of four [B] int32 tensors."""
    if isinstance(bbox, (list, tuple)):
        if len(bbox) != 4:
            raise ValueError(f"bbox as a sequence holds four [B] tensors (x, y, w, h), got {len(bbox)}")
        w, h = (_device_tensor(c, "bbox", device) for c in bbox[2:])
        if w.shape != (B,) or h.shape != (B,):
            raise ValueError(f"bbox columns {tuple(w.shape)}, {tuple(h.shape)} must be [{B}]")
    else:
        bbox = _device_tensor(bbox, "bbox", device)
        if bbox.shape != (B, 4):
            raise ValueError(f"bbox {tuple(bbox.shape)} must be [{B}, 4]")
        w, h = bbox[:, 2], bbox[:, 3]
    if w.dtype != torch.int32 or h.dtype != torch.int32:
        raise TypeError(f"bbox must be int32 (the dtype of the reference's batch), got {w.dtype}")
    if w.stride(0) != h.stride(0):
        w, h = w.contiguous(), h.contiguous()
    return w, h


class _Group:
    """One dad3d_kp_group and the tensors it points into (kept alive until the launch is enqueued)."""

    def __init__(self, pred: Tensor, target: Tensor, index: Optional[Tensor] = None, presence: Optional[Tensor] = None,
                 box=None, pred_scale: float = 1.0, target_scale: float = 1.0, normalize: bool = False):
        B, _, K = pred.shape
        n = int(index.numel()) if index is not None else int(pred.shape[1])
        self.keep = [pred, target, index, presence]
        g = _lib.KpGroup(pred_d=pred.data_ptr(), target_d=target.data_ptr(), pred_stride=pred.stride(0),
                         target_stride=target.stride(0), pred_scale=pred_scale, target_scale=target_scale, n=n, k=K,
                         normalize=int(normalize))
        if index is not None:
            g.index_d = index.data_ptr()
        if presence is not None:
            g.presence_d, g.presence_stride = presence.data_ptr(), presence.stride(0)
        if box is not None:
            w, h = box
            self.keep += [w, h]
            g.box_w_d, g.box_h_d, g.box_stride = w.data_ptr(), h.data_ptr(), w.stride(0)
        self.struct = g


def _keypoint_errors(groups: Sequence[_Group], B: int, device: torch.device) -> Tensor:
    """records [B, G, 2] = (err, norm) per head and group (one launch)."""
    arr = (_lib.KpGroup * len(groups))(*[g.struct for g in groups])
    rec = torch.empty(B, len(groups), 2, dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _lib.check(_lib.load().dad3d_keypoint_errors(arr, len(groups), B, rec.data_ptr(), _stream(device)),
                   "dad3d_keypoint_errors")
    return rec


def _reduce(device: torch.device, n_values: int, stats: Optional[Tensor] = None, eps: float = 1e-6,
            records: Optional[Tensor] = None, nme_scale: float = 1.0, below: bool = True, thresholds: Sequence[float] = (),
            per_head: Optional[Tensor] = None, epoch: Optional[Tuple[Tensor, Tensor]] = None, weight: float = 0.0) -> Tensor:
    values = torch.empty(n_values, dtype=torch.float32, device=device)
    thr = np.asarray(thresholds, dtype=np.float32)
    B, G = (int(records.shape[0]), int(records.shape[1])) if records is not None else (0, 0)
    acc, ev = epoch if epoch is not None else (None, None)
    with torch.cuda.device(device):
        _lib.check(_lib.load().dad3d_metrics_reduce(
            stats.data_ptr() if stats is not None else None, int(stats.shape[0]) if stats is not None else 0, float(eps),
            records.data_ptr() if records is not None else None, B, G, float(nme_scale), int(bool(below)),
            thr.ctypes.data if thr.size else None, int(thr.size), float(weight), values.data_ptr(),
            per_head.data_ptr() if per_head is not None else None, acc.data_ptr() if acc is not None else None,
            ev.data_ptr() if ev is not None else None, _stream(device)), "dad3d_metrics_reduce")
    return values


def _iou_stats(x: Tensor, t: Tensor, logits: bool) -> Tensor:
    planes = x.shape[0] * x.shape[1]
    stats = torch.empty(planes, 4, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().dad3d_iou_stats(x.data_ptr(), t.data_ptr(), int(t.dtype == torch.uint8), int(logits), planes,
                                               x.numel() // planes, stats.data_ptr(), _stream(x.device)), "dad3d_iou_stats")
    return stats


def _check_heatmaps(output: Tensor, target: Tensor, what: str):
    if output.ndim != 4 or target.shape != output.shape or output.numel() == 0:
        raise ValueError(f"{what}: output {tuple(output.shape)} and target {tuple(target.shape)} must be the same non-empty "
                         f"[B, C, H, W]")


def soft_iou(output: Tensor, target: Tensor, eps: float = 1e-6) -> Tensor:
    """metrics/iou.py:15-31: mean over the (b, c) planes of (sum t o + eps) / (sum t^2 + sum o^2 - sum t o + eps), with
    ``output`` probabilities and ``target`` [B, C, H, W] floating-point tensors."""
    _check_heatmaps(_check_float(output, "output"), _check_float(target, "target"), "soft_iou")
    o = _float(output, "output")
    t = _float(target, "target", o.device)
    return _reduce(o.device, 1, stats=_iou_stats(o, t, logits=False), eps=eps)[0]


def _keypoint_inputs(output_kp, target_kp, bbox):
    p, t = _check_float(output_kp, "output_kp"), _check_float(target_kp, "target_kp")
    if p.ndim != 3 or p.shape[2] not in (2, 3) or t.shape != p.shape or p.shape[0] == 0 or p.shape[1] == 0:
        raise ValueError(f"keypoints {tuple(p.shape)} and {tuple(t.shape)} must both be non-empty [B, N, 2 or 3]")
    p = _float(p, "output_kp")
    t = _float(t, "target_kp", p.device)
    box = _box_columns(bbox, p.shape[0], p.device) if bbox is not None else None
    return _Group(p, t, box=box), p.shape[0], p.device


def keypoints_nme(output_kp: Tensor, target_kp: Tensor, bbox: Tensor = None, reduce: str = "mean") -> Tensor:
    """metrics/keypoints.py:19-35: err / norm per head, err the mean keypoint distance and norm sqrt(w * h) of ``bbox``
    (int32 [B, 4] x, y, w, h) or 2.0 without one; the mean over heads when ``reduce == "mean"``, else the [B] values."""
    g, B, dev = _keypoint_inputs(output_kp, target_kp, bbox)
    rec = _keypoint_errors([g], B, dev)
    if reduce == "mean":
        return _reduce(dev, 1, records=rec)[0]
    per_head = torch.empty(B, dtype=torch.float32, device=dev)
    _reduce(dev, 1, records=rec, per_head=per_head)
    return per_head


def percentage_of_errors_below_IOD(output_kp: Tensor, target_kp: Tensor, bbox: Tensor = None, threshold: float = 0.05,
                                   below: bool = True) -> Tensor:
    """metrics/keypoints.py:38-52: the share of heads whose err is below ``threshold * norm`` (above, when ``below`` is
    False).  The reference's training step logs it as a "failure rate" (fr_*); the name and the direction are its own."""
    g, B, dev = _keypoint_inputs(output_kp, target_kp, bbox)
    rec = _keypoint_errors([g], B, dev)
    return _reduce(dev, 2, records=rec, below=below, thresholds=[threshold])[1]


def _threshold_name(t: float) -> str:
    return str(t).replace(".", "")          # 0.05 -> "005", 0.1 -> "01": the reference's metric names


class FlameStepMetrics:
    """The metric block of ``FlameLightningModel._step_fn`` (train/flame_lightning_model.py:299-357).

    ``step(outputs, batch, loader_name)`` returns, as 0-dim fp32 device tensors keyed ``f"{loader_name}/metrics/{name}"``,
    what the reference logs per batch: ``heatmap_iou`` (soft IoU of sigmoid(heat-map logits) and the target heat-map);
    ``fr_2d_*`` and ``nme_2d`` on the 2D landmarks (``OUTPUT_2D_LANDMARKS * img_size`` and the target, both masked by
    presence, normalised by the crop box); ``reproject_*`` on the ``face`` vertices of ``reprojected_vertices(to_2d=True)``
    against ``TARGET_2D_FULL_LANDMARKS``; ``*_3d`` on ``normalize_to_cube`` of the ``face`` vertices of
    ``vertices_3d(zero_rotation=True)`` and of ``TARGET_3D_MODEL_VERTICES``, with norm 2.0.  ``nme_*`` are KeypointsNME's
    values (100 x the mean), ``fr_*`` the share of heads below ``threshold * norm`` for each of ``thresholds``.

    ``outputs`` is the encoder's dict; ``batch`` is what ``FlameBatchBuilder`` returns (uint8 heat-map, bbox as four [B]
    int32 tensors) or what ``KeypointsDataMixin.get_input`` makes of it (float heat-map, [B, 4] bbox); both give the same
    bits.  The parameters are decoded with the hi/lo decode the losses use, and the caller's tensor is not modified: the
    reference zeroes translation z in place (head_mesh.py:41), but z enters neither vertex set read here
    (``vertices_3d`` does not translate, and ``to_2d`` drops the z coordinate it would move), so no value depends on it.  A step is 7 launches of this library whatever B: two decodes of two launches each, then the IoU
    statistics, the per-head errors and the reduction.

    ``compute()`` gives the epoch values: the means of the per-batch values weighted by batch size over the steps since
    ``reset()``, what Lightning reports for ``self.log(..., on_epoch=True)``; the sums are fp64 on the device.
    """

    NME_WEIGHT = 100.0            # KeypointsNME(weight=100), metrics/keypoints.py:126

    def __init__(self, img_size: int = 256, face_indices=None, thresholds: Sequence[float] = (0.05, 0.1)):
        if not 1 <= len(thresholds) <= _lib.DAD3D_METRIC_MAX_THRESHOLDS:
            raise ValueError(f"1 to {_lib.DAD3D_METRIC_MAX_THRESHOLDS} thresholds, got {len(thresholds)}")
        st = load_flame_static()
        self.n_vertices = int(np.asarray(st["v_template"]).shape[0])
        face = np.asarray(st["flame_indices_face"] if face_indices is None else face_indices).reshape(-1).astype(np.int64)
        if face.size == 0 or face.min() < -self.n_vertices or face.max() >= self.n_vertices:
            raise ValueError(f"face_indices must be a non-empty index set into the {self.n_vertices} vertices")
        self.face = np.where(face < 0, face + self.n_vertices, face).astype(np.int32)
        self.img_size = int(img_size)
        self.thresholds = tuple(float(t) for t in thresholds)
        self.head_mesh = HeadMesh(image_size=self.img_size)
        groups = [("2d", ""), ("2d", "reproject_"), ("3d", "")]
        self.names = ["heatmap_iou"]
        for dim, prefix in groups:
            self.names += [f"{prefix}nme_{dim}"] + [f"{prefix}fr_{dim}_{_threshold_name(t)}" for t in self.thresholds]
        self._face_d: Dict[torch.device, Tensor] = {}
        self._epoch: Optional[Tuple[Tensor, Tensor]] = None

    @property
    def launches_per_step(self) -> int:
        return 7

    def _face(self, device: torch.device) -> Tensor:
        f = self._face_d.get(device)
        if f is None:
            f = self._face_d[device] = torch.from_numpy(self.face).to(device)
        return f

    def _epoch_buffers(self, device: torch.device) -> Tuple[Tensor, Tensor]:
        if self._epoch is None:
            n = len(self.names)
            self._epoch = (torch.zeros(n + 1, dtype=torch.float64, device=device),
                           torch.full((n,), float("nan"), dtype=torch.float32, device=device))
        elif self._epoch[0].device != device:
            raise ValueError(f"this FlameStepMetrics accumulates on {self._epoch[0].device}; reset() before using {device}")
        return self._epoch

    def step(self, outputs: Dict[str, Tensor], batch: Dict[str, object], loader_name: str = "valid") -> Dict[str, Tensor]:
        if OUTPUT_2D_LANDMARKS not in outputs:
            raise ValueError("FlameStepMetrics needs OUTPUT_2D_LANDMARKS (the heat-map argmax fallback is not supported)")
        params = _float(outputs[OUTPUT_3DMM_PARAMS], OUTPUT_3DMM_PARAMS)
        dev = params.device
        lm = _float(outputs[OUTPUT_2D_LANDMARKS], OUTPUT_2D_LANDMARKS, dev)
        hm = _float(outputs[OUTPUT_LANDMARKS_HEATMAP], OUTPUT_LANDMARKS_HEATMAP, dev)
        hm_t = _device_tensor(batch[TARGET_LANDMARKS_HEATMAP], TARGET_LANDMARKS_HEATMAP, dev)
        hm_t = hm_t.contiguous() if hm_t.dtype == torch.uint8 else _float(hm_t, TARGET_LANDMARKS_HEATMAP, dev)
        _check_heatmaps(hm, hm_t, "heat-map")
        B = int(params.shape[0])
        lm_t = _float(batch[TARGET_2D_LANDMARKS], TARGET_2D_LANDMARKS, dev)
        pres = _device_tensor(batch[TARGET_2D_LANDMARKS_PRESENCE], TARGET_2D_LANDMARKS_PRESENCE, dev)
        if pres.dtype not in (torch.bool, torch.uint8):
            raise TypeError(f"{TARGET_2D_LANDMARKS_PRESENCE} must be bool, got {pres.dtype}")
        pres = pres.contiguous().view(torch.uint8)
        full_t = _float(batch[TARGET_2D_FULL_LANDMARKS], TARGET_2D_FULL_LANDMARKS, dev)
        v3_t = _float(batch[TARGET_3D_MODEL_VERTICES], TARGET_3D_MODEL_VERTICES, dev)
        V = self.n_vertices
        if (lm.ndim != 3 or lm.shape[0] != B or lm.shape[2] != 2 or lm_t.shape != lm.shape
                or pres.shape != lm.shape[:2] or full_t.shape != (B, V, 2) or v3_t.shape != (B, V, 3)
                or hm.shape[0] != B or lm.shape[1] == 0):
            raise ValueError(f"step: landmarks {tuple(lm.shape)} / {tuple(lm_t.shape)}, presence {tuple(pres.shape)}, "
                             f"full landmarks {tuple(full_t.shape)}, vertices {tuple(v3_t.shape)} and heat-maps "
                             f"{tuple(hm.shape)} do not describe one batch of {B} heads with {V} vertices")
        box = _box_columns(batch[INPUT_BBOX_KEY], B, dev)
        dec = self.head_mesh.flame.decoder(dev)
        if params.shape != (B, dec.num_params):
            raise ValueError(f"{OUTPUT_3DMM_PARAMS} {tuple(params.shape)} must be [B, {dec.num_params}]")
        v3, _ = dec.decode(params, want_vertices=True, want_projected=False, zero_rot=True, hilo=True)
        _, pj = dec.decode(params, want_vertices=False, want_projected=True, to_2d=True,
                           image_size=float(self.img_size), hilo=True)
        face = self._face(dev)
        s = float(self.img_size)
        groups = [_Group(lm, lm_t, presence=pres, box=box, pred_scale=s, target_scale=s),
                  _Group(pj, full_t, index=face, box=box),
                  _Group(v3, v3_t, index=face, normalize=True)]
        stats = _iou_stats(hm, hm_t, logits=True)
        rec = _keypoint_errors(groups, B, dev)
        values = _reduce(dev, len(self.names), stats=stats, records=rec, nme_scale=self.NME_WEIGHT, below=True,
                         thresholds=self.thresholds, epoch=self._epoch_buffers(dev), weight=float(B))
        return {f"{loader_name}/metrics/{n}": values[i] for i, n in enumerate(self.names)}

    __call__ = step

    def compute(self, loader_name: str = "valid") -> Dict[str, Tensor]:
        """The batch-size-weighted means since the last ``reset()`` (NaN before any step)."""
        if self._epoch is None:
            return {f"{loader_name}/metrics/{n}": torch.tensor(float("nan")) for n in self.names}
        ev = self._epoch[1].clone()
        return {f"{loader_name}/metrics/{n}": ev[i] for i, n in enumerate(self.names)}

    def reset(self) -> None:
        if self._epoch is not None:
            self._epoch[0].zero_()
            self._epoch[1].fill_(float("nan"))
