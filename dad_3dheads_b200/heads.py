"""Trainable regression heads of DAD-3DNet over a frozen backbone.

``FlameHeads`` holds the three ClassificationHeads (flame_regression.py:45-59: Linear 2048->512, ReLU, Dropout, Linear
512->{403, 10, 136}) with their epilogue (:96-100) in packed form and runs them with csrc/heads.cu; its backward gives the
weight gradients.  ``FrozenBackboneRegression`` puts it behind ``Dad3dEncoder.features`` and returns the reference model's
output dict, so the package losses, the reference's ``LossModule`` and ``FlameStepMetrics`` consume it unchanged.
"""
from __future__ import annotations

from typing import Dict

import torch
from torch import Tensor, nn

from . import _lib
from .encoder import OUTPUT_2D_LANDMARKS, OUTPUT_3DMM_PARAMS, OUTPUT_LANDMARKS_HEATMAP, Dad3dEncoder
from .encoder_weights import HEAD_OUT, LINEAR_SIZE

FEATURES = 2048
HIDDEN = LINEAR_SIZE * len(HEAD_OUT)            # 1536
OUTPUTS = sum(n for _, n in HEAD_OUT)           # 549
MAX_BATCH = 8 * 65535                           # include/dad3d.h


def _stream(dev: torch.device):
    return torch.cuda.current_stream(dev).cuda_stream


def _check(t: Tensor, name: str, shape) -> None:
    if not t.is_cuda or t.dtype != torch.float32:
        raise TypeError(f"{name} must be a float32 CUDA tensor, got {t.dtype} on {t.device}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")


class _HeadsFunction(torch.autograd.Function):
    """Saves y and the bit masks, not params: ReprojectionLoss zeroes translation z of params in place (losses.py:258)."""

    @staticmethod
    def forward(ctx, f, w1, b1, w2, b2, heads):
        B = f.shape[0]
        dev = f.device
        lib = _lib.load()
        params = torch.empty(B, 413, dtype=torch.float32, device=dev)
        lms = torch.empty(B, OUTPUTS - 413, dtype=torch.float32, device=dev)
        h = torch.empty(B, HIDDEN, dtype=torch.float32, device=dev)
        d = torch.empty_like(h)
        mask = torch.empty(B, HIDDEN // 32, dtype=torch.int32, device=dev)
        y = torch.empty(B, 403, dtype=torch.float32, device=dev)
        obits = torch.empty(B, (OUTPUTS + 31) // 32, dtype=torch.int32, device=dev)
        ws = torch.empty(int(lib.dad3d_heads_workspace_bytes(B)), dtype=torch.uint8, device=dev)
        train = heads.training
        with torch.cuda.device(dev):             # the launches go to the tensors' device, not the current one
            _lib.check(lib.dad3d_heads_forward(f.data_ptr(), B, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                               heads.limit_value, int(train), heads.dropout, heads.seed,
                                               heads.counter.data_ptr() if train else None, params.data_ptr(),
                                               lms.data_ptr(), h.data_ptr(), d.data_ptr(), mask.data_ptr(), y.data_ptr(),
                                               obits.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)),
                       "dad3d_heads_forward")
        ctx.save_for_backward(f, w2, h, d, mask, y, obits)
        ctx.cfg = (train, heads.dropout, heads.limit_value)
        return params, lms.view(B, -1, 2)

    @staticmethod
    def backward(ctx, dparams, dlms):
        f, w2, h, d, mask, y, obits = ctx.saved_tensors
        train, p, limit = ctx.cfg
        B = f.shape[0]
        dparams = torch.zeros(B, 413, device=f.device) if dparams is None else dparams.contiguous()
        dlms = torch.zeros(B, OUTPUTS - 413, device=f.device) if dlms is None else dlms.contiguous()
        dw1 = torch.empty(HIDDEN, FEATURES, dtype=torch.float32, device=f.device)
        db1 = torch.empty(HIDDEN, dtype=torch.float32, device=f.device)
        dw2 = torch.empty(OUTPUTS, LINEAR_SIZE, dtype=torch.float32, device=f.device)
        db2 = torch.empty(OUTPUTS, dtype=torch.float32, device=f.device)
        lib = _lib.load()
        ws = torch.empty(int(lib.dad3d_heads_workspace_bytes(B)), dtype=torch.uint8, device=f.device)
        with torch.cuda.device(f.device):
            _lib.check(lib.dad3d_heads_backward(dparams.data_ptr(), dlms.data_ptr(), f.data_ptr(), B, w2.data_ptr(), limit,
                                                int(train), p, h.data_ptr(), d.data_ptr(), mask.data_ptr(), y.data_ptr(),
                                                obits.data_ptr(), dw1.data_ptr(), db1.data_ptr(), dw2.data_ptr(),
                                                db2.data_ptr(), ws.data_ptr(), ws.numel(), _stream(f.device)),
                       "dad3d_heads_backward")
        return None, dw1, db1, dw2, db2, None


class FlameHeads(nn.Module):
    """The shape, pose and landmark heads in packed form: w1 [1536, 2048], b1 [1536], w2 [549, 512], b2 [549] (rows in
    HEAD_OUT order).  ``heads(features [B, 2048]) -> (params [B, 413], landmarks [B, 68, 2])``.  Dropout draws from
    Philox4x32-10 keyed by ``seed``; its step counter lives on the device and advances with every training forward."""

    def __init__(self, dropout: float = 0.3, limit_value: float = 3.0, seed: int = 0):
        super().__init__()
        if not 0.0 <= dropout < 1.0:
            raise ValueError(f"dropout must be in [0, 1), got {dropout}")
        self.dropout, self.limit_value, self.seed = float(dropout), float(limit_value), int(seed) & (2 ** 64 - 1)
        self.w1 = nn.Parameter(torch.zeros(HIDDEN, FEATURES))
        self.b1 = nn.Parameter(torch.zeros(HIDDEN))
        self.w2 = nn.Parameter(torch.zeros(OUTPUTS, LINEAR_SIZE))
        self.b2 = nn.Parameter(torch.zeros(OUTPUTS))
        self.register_buffer("counter", torch.zeros(1, dtype=torch.int64))

    @classmethod
    def from_state_dict(cls, sd: Dict[str, Tensor], **kw) -> "FlameHeads":
        """Packs the reference keys {shape,pose,landmarks}.logit_image.{0,3}.{weight,bias}."""
        heads = cls(**kw)
        g = lambda k: sd[k].detach().to(torch.float32)     # noqa: E731
        with torch.no_grad():
            heads.w1.copy_(torch.cat([g(f"{n}.logit_image.0.weight") for n, _ in HEAD_OUT], 0))
            heads.b1.copy_(torch.cat([g(f"{n}.logit_image.0.bias") for n, _ in HEAD_OUT], 0))
            heads.w2.copy_(torch.cat([g(f"{n}.logit_image.3.weight") for n, _ in HEAD_OUT], 0))
            heads.b2.copy_(torch.cat([g(f"{n}.logit_image.3.bias") for n, _ in HEAD_OUT], 0))
        return heads

    def reference_state_dict(self) -> Dict[str, Tensor]:
        """The reference keys of the current weights (CPU copies): ``sd.update(heads.reference_state_dict())``."""
        out, r = {}, 0
        for i, (n, rows) in enumerate(HEAD_OUT):
            hid = slice(i * LINEAR_SIZE, (i + 1) * LINEAR_SIZE)
            out[f"{n}.logit_image.0.weight"] = self.w1.detach()[hid].cpu().clone()
            out[f"{n}.logit_image.0.bias"] = self.b1.detach()[hid].cpu().clone()
            out[f"{n}.logit_image.3.weight"] = self.w2.detach()[r:r + rows].cpu().clone()
            out[f"{n}.logit_image.3.bias"] = self.b2.detach()[r:r + rows].cpu().clone()
            r += rows
        return out

    def forward(self, features: Tensor):
        if features.ndim != 2:
            raise ValueError(f"features must be [B, {FEATURES}], got {tuple(features.shape)}")
        _check(features, "features", (features.shape[0], FEATURES))
        for name, t in (("w1", self.w1), ("b1", self.b1), ("w2", self.w2), ("b2", self.b2)):
            _check(t, name, t.shape)
            if t.device != features.device or not t.is_contiguous():
                raise ValueError(f"{name} must be contiguous on {features.device}")
        if self.training and self.counter.device != features.device:
            raise ValueError(f"the dropout counter must be on {features.device}")
        if not 1 <= features.shape[0] <= MAX_BATCH:
            raise ValueError(f"batch must be 1 to {MAX_BATCH}, got {features.shape[0]}")
        return _HeadsFunction.apply(features.contiguous(), self.w1, self.b1, self.w2, self.b2, self)


class FrozenBackboneRegression(nn.Module):
    """``model(images [B,3,256,256]) -> {OUTPUT_3DMM_PARAMS, OUTPUT_2D_LANDMARKS, OUTPUT_LANDMARKS_HEATMAP}`` with the
    backbone frozen in eval mode (``Dad3dEncoder.features``) and the heads trainable; ``parameters()`` are the heads'."""

    def __init__(self, encoder: Dad3dEncoder, heads: FlameHeads):
        super().__init__()
        self.__dict__["encoder"] = encoder          # not a submodule: it has no parameters to train
        self.heads = heads

    def forward(self, images: Tensor) -> Dict[str, Tensor]:
        features, heatmap = self.encoder.features(images, want_heatmap=True)
        params, lms = self.heads(features)
        return {OUTPUT_3DMM_PARAMS: params, OUTPUT_2D_LANDMARKS: lms, OUTPUT_LANDMARKS_HEATMAP: heatmap}
