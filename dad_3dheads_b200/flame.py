"""Host-side mirror of the reference's FLAME interface (model_training/model/flame.py) over libdad3d.so.

Same names, argument meaning and error behaviour as the reference: ``FLAME_CONSTS`` (flame.py:17-26), ``FlameParams``
(:29-101) and ``FLAMELayer`` (:117-229).  The arithmetic of ``FLAMELayer.forward`` (blend shapes, pose correctives,
skinning, z offset, 6-DoF rotation) runs in the CUDA kernels of csrc/flame.cu; nothing is computed on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Dict, Optional

import numpy as np
import torch
import torch.nn as nn
from torch import Tensor

from . import _lib

FLAME_CONSTS = {
    "shape": 300,
    "expression": 100,
    "rotation": 6,
    "jaw": 3,
    "eyeballs": 0,
    "neck": 0,
    "translation": 3,
    "scale": 1,
}

MAX_SHAPE = 300
MAX_EXPRESSION = 100
ROT_COEFFS = 3
JAW_COEFFS = 3
EYE_COEFFS = 6
NECK_COEFFS = 3
MESH_OFFSET_Z = 0.05

_FIELD_ORDER = ("shape", "expression", "jaw", "rotation", "eyeballs", "neck", "translation", "scale")
_ASSET = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets", "flame_static.npz")


@dataclass
class FlameParams:
    """Views into a [B, num_params] 3DMM tensor (reference: flame.py:29-101)."""

    shape: Tensor
    expression: Tensor
    rotation: Tensor
    translation: Tensor
    scale: Tensor
    jaw: Tensor
    eyeballs: Tensor
    neck: Tensor

    @classmethod
    def from_3dmm(cls, tensor_3dmm: Tensor, constants: Dict[str, int], zero_expr: bool = False) -> "FlameParams":
        assert tensor_3dmm.ndim == 2
        fields, cur = {}, 0
        for name in _FIELD_ORDER:                       # slicing order is fixed, independent of the dict order
            width = constants[name]
            fields[name] = tensor_3dmm[:, cur:cur + width]
            cur += width
        if zero_expr:
            fields["expression"] = torch.zeros_like(fields["expression"])
        return cls(**fields)

    def to_3dmm_tensor(self) -> Tensor:
        # the reference concatenates rotation BEFORE jaw here (flame.py:86-99) although from_3dmm reads jaw first
        # (SURVEY App. D.6); mirrored as is.
        return torch.cat([self.shape, self.expression, self.rotation, self.jaw, self.eyeballs, self.neck,
                          self.translation, self.scale], -1)

    def packed(self) -> Tensor:
        """[B, num_params] in from_3dmm order -- what the decode kernels consume."""
        return torch.cat([getattr(self, n) for n in _FIELD_ORDER], dim=-1).contiguous()


def load_flame_static(path: Optional[str] = None) -> Dict[str, np.ndarray]:
    """The FLAME constants: the packed ``assets/flame_static.npz`` by default, or -- like the reference's
    ``get_flame_model(flame_path)`` (model/utils.py:84-89) -- a ``flame.pkl`` given by path (flame_assets.py)."""
    from .flame_assets import load_static
    return load_static(path, _ASSET)


class _Workspace:
    """Per-device scratch cache (torch owns the memory; the library only borrows pointers)."""

    def __init__(self):
        self._buf: Dict[int, Tensor] = {}
        self.generation = 0             # bumped on every reallocation (CUDA graphs bake in the buffer address)

    def get(self, device: torch.device, nbytes: int) -> Tensor:
        key = device.index if device.index is not None else torch.cuda.current_device()
        buf = self._buf.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
            self._buf[key] = buf
            self.generation += 1
        return buf


class FlameDecoder:
    """Owns one ``dad3d_flame`` handle (C ABI) on one device.  ``decode`` = vertices_3d + reprojected_vertices in one pass."""

    def __init__(self, static: Dict[str, np.ndarray], consts: Dict[str, int], device: torch.device):
        if not torch.cuda.is_available():
            raise _lib.Dad3dError("dad_3dheads_b200 needs a CUDA (sm_90a) device: there is no CPU path")
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.Dad3dError(f"FlameDecoder needs a cuda device, got {self.device}")
        self.consts = dict(consts)
        f32 = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float32))
        sd = f32(static["shapedirs"])
        self.n_vertices = int(sd.shape[0])
        sd = sd.reshape(self.n_vertices * 3, -1)
        pd = f32(static["posedirs"])
        vt = f32(static["v_template"]).reshape(-1)
        jr = f32(static["J_regressor"])
        par = np.ascontiguousarray(np.asarray(static["parents"], dtype=np.int32))
        w = f32(static["lbs_weights"])
        lay = _lib.FlameLayout(**{k: int(self.consts[k]) for k in _FIELD_ORDER})
        h = C.c_void_p()
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        _lib.check(self.lib.dad3d_flame_create(C.byref(h), sd.ctypes.data, pd.ctypes.data, vt.ctypes.data,
                                               jr.ctypes.data, par.ctypes.data, w.ctypes.data, self.n_vertices,
                                               sd.shape[1], jr.shape[0], C.byref(lay), dev_index),
                   "dad3d_flame_create")
        self._h = h
        self.num_params = int(self.lib.dad3d_flame_num_params(h))
        self._ws = _Workspace()

    @property
    def ws_generation(self) -> int:
        return self._ws.generation

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self.lib.dad3d_flame_destroy(h)
            except Exception:
                pass
            self._h = None

    def decode(self, params: Tensor, *, want_vertices: bool = True, want_projected: bool = False, to_2d: bool = True,
               zero_rot: bool = False, zero_jaw: bool = False, image_size: float = 256.0, fast: bool = False,
               simt: bool = False, unfused: bool = False, cluster: bool = False, hilo: bool = False, pair: bool = False):
        """params: [B, num_params] fp32 CUDA tensor on this decoder's device.  Returns (vertices3d|None, projected|None).

        Default = the dedicated one-product decode kernel (fp16 operands, fp32 accumulate; vertices relL2 ~1.5e-5 vs fp64,
        inside the 1e-4 contract).  ``hilo=True`` = fp16 hi/lo split operands, 3 tensor-core products (relL2 ~2e-7).
        ``fast`` is the old name of today's default and has no effect; ``pair`` / ``cluster`` / ``unfused`` / ``simt`` are
        A/B and verification switches (include/dad3d.h)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.ndim == 2
        assert params.shape[1] == self.num_params, (params.shape, self.num_params)
        params = params.contiguous()
        B = params.shape[0]
        v3 = torch.empty(B, self.n_vertices, 3, dtype=torch.float32, device=params.device) if want_vertices else None
        pj = (torch.empty(B, self.n_vertices, 2 if to_2d else 3, dtype=torch.float32, device=params.device)
              if want_projected else None)
        if B == 0:
            return v3, pj
        flags = ((_lib.DAD3D_ZERO_ROT if zero_rot else 0) | (_lib.DAD3D_ZERO_JAW if zero_jaw else 0) |
                 (_lib.DAD3D_BLEND_FAST if fast else 0) | (_lib.DAD3D_BLEND_SIMT if simt else 0) |
                 (_lib.DAD3D_DECODE_UNFUSED if unfused else 0) | (_lib.DAD3D_DECODE_CLUSTER if cluster else 0) |
                 (_lib.DAD3D_BLEND_HILO if (hilo or cluster) else 0) | (_lib.DAD3D_DECODE_PAIR if pair else 0))
        nbytes = int(self.lib.dad3d_flame_workspace_bytes(self._h, B))
        ws = self._ws.get(params.device, nbytes)
        stream = torch.cuda.current_stream(params.device).cuda_stream
        with torch.cuda.device(params.device):
            _lib.check(self.lib.dad3d_flame_decode(self._h, params.data_ptr(), B, flags,
                                                   v3.data_ptr() if v3 is not None else None,
                                                   pj.data_ptr() if pj is not None else None,
                                                   float(image_size), 1 if to_2d else 0, ws.data_ptr(), ws.numel(),
                                                   stream), "dad3d_flame_decode")
        return v3, pj

    # ---- test hooks: the two stages of a decode pass on caller buffers (include/dad3d.h)
    def describe(self, B: int, flags: int = 0) -> Dict[str, Any]:
        """Packing constants and, per pass of a decode of ``B`` heads with ``flags``, the launch the library would make."""
        import json
        buf = C.create_string_buffer(1 << 16)
        _lib.check(self.lib.dad3d_flame_describe(self._h, int(B), int(flags), buf, len(buf)), "dad3d_flame_describe")
        return json.loads(buf.value.decode())

    def prep(self, params: Tensor, *, flags: int = 0, permute: bool = False):
        """flame_prep_kernel alone: (coef_hi, coef_lo) [B rounded up to 256, 448] fp16 (padding rows unwritten: zeros here)
        and the [B, 68] transform records."""
        assert params.is_cuda and params.dtype == torch.float32 and params.shape[1] == self.num_params
        params = params.contiguous()
        B = params.shape[0]
        rows = (B + 255) // 256 * 256
        hi = torch.zeros(rows, 448, dtype=torch.float16, device=params.device)
        lo = torch.zeros_like(hi)
        xf = torch.empty(B, 68, dtype=torch.float32, device=params.device)
        with torch.cuda.device(params.device):
            _lib.check(self.lib.dad3d_flame_prep(self._h, params.data_ptr(), B, int(flags), hi.data_ptr(), lo.data_ptr(),
                                                 xf.data_ptr(), 1 if permute else 0,
                                                 torch.cuda.current_stream(params.device).cuda_stream), "dad3d_flame_prep")
        return hi, lo, xf

    def decode_from(self, coef_hi: Tensor, coef_lo: Tensor, xf: Tensor, *, flags: int = 0, vertices: Optional[Tensor] = None,
                    projected: Optional[Tensor] = None, image_size: float = 256.0, to_2d: bool = True) -> None:
        """The stage after prep for one pass of ``xf.shape[0]`` heads, written into the caller's ``vertices`` [B,V,3] /
        ``projected`` [B,V,2|3] views (either may be None).  Rows are permuted for the dedicated kernel only."""
        B = xf.shape[0]
        for t in (coef_hi, coef_lo):
            assert t.dtype == torch.float16 and t.is_contiguous() and t.shape[1] == 448 and t.shape[0] >= (B + 255) // 256 * 256
        assert xf.dtype == torch.float32 and xf.is_contiguous() and xf.shape == (B, 68)
        self._check_out(vertices, B, 3)
        self._check_out(projected, B, 2 if to_2d else 3)
        nbytes = int(self.lib.dad3d_flame_workspace_bytes(self._h, B))
        ws = self._ws.get(xf.device, nbytes)
        with torch.cuda.device(xf.device):
            _lib.check(self.lib.dad3d_flame_decode_from(
                self._h, coef_hi.data_ptr(), coef_lo.data_ptr(), xf.data_ptr(), B, int(flags),
                vertices.data_ptr() if vertices is not None else None, projected.data_ptr() if projected is not None else None,
                float(image_size), 1 if to_2d else 0, ws.data_ptr(), ws.numel(),
                torch.cuda.current_stream(xf.device).cuda_stream), "dad3d_flame_decode_from")

    def decode_into(self, params: Tensor, *, flags: int = 0, vertices: Optional[Tensor] = None,
                    projected: Optional[Tensor] = None, image_size: float = 256.0, to_2d: bool = True) -> None:
        """``dad3d_flame_decode`` into caller-owned output views (``decode`` allocates its own): for guard-band tests."""
        assert params.is_cuda and params.dtype == torch.float32 and params.shape[1] == self.num_params
        params = params.contiguous()
        B = params.shape[0]
        self._check_out(vertices, B, 3)
        self._check_out(projected, B, 2 if to_2d else 3)
        nbytes = int(self.lib.dad3d_flame_workspace_bytes(self._h, B))
        ws = self._ws.get(params.device, nbytes)
        with torch.cuda.device(params.device):
            _lib.check(self.lib.dad3d_flame_decode(
                self._h, params.data_ptr(), B, int(flags), vertices.data_ptr() if vertices is not None else None,
                projected.data_ptr() if projected is not None else None, float(image_size), 1 if to_2d else 0,
                ws.data_ptr(), ws.numel(), torch.cuda.current_stream(params.device).cuda_stream), "dad3d_flame_decode")

    # ---- test hooks: the stages of a backward pass on caller buffers (include/dad3d.h); B <= 4096 heads
    def _npad(self) -> int:
        return (3 * self.n_vertices + 127) // 128 * 128

    def backward_blend(self, coef_hi: Tensor, coef_lo: Tensor, B: int, vposed: Tensor) -> None:
        """The recomputed forward blend product: unpermuted prep rows -> ``vposed`` [B, npad] fp32 (v_posed * basis_scale)."""
        for t in (coef_hi, coef_lo):
            assert t.dtype == torch.float16 and t.is_contiguous() and t.shape[1] == 448 and t.shape[0] >= (B + 255) // 256 * 256
        assert vposed.dtype == torch.float32 and vposed.is_contiguous() and vposed.shape == (B, self._npad())
        with torch.cuda.device(vposed.device):
            _lib.check(self.lib.dad3d_flame_backward_blend(self._h, coef_hi.data_ptr(), coef_lo.data_ptr(), int(B),
                                                           vposed.data_ptr(),
                                                           torch.cuda.current_stream(vposed.device).cuda_stream),
                       "dad3d_flame_backward_blend")

    def backward_vertex(self, vposed: Tensor, xf: Tensor, grad_vertices: Optional[Tensor], grad_projected: Optional[Tensor], *,
                        sigma: Tensor, d_hi: Tensor, d_lo: Tensor, partial: Tensor, image_size: float = 256.0,
                        to_2d: bool = True) -> None:
        """Vertex stage: ``sigma`` [B], ``d_hi`` / ``d_lo`` [B, npad] fp16 and ``partial`` [B, ceil(V / 256), 32]."""
        B, nv = xf.shape[0], self.n_vertices
        assert vposed.dtype == torch.float32 and vposed.is_contiguous() and vposed.shape == (B, self._npad())
        assert xf.dtype == torch.float32 and xf.is_contiguous() and xf.shape == (B, 68)
        for t, shape in ((grad_vertices, (B, nv, 3)), (grad_projected, (B, nv, 2 if to_2d else 3))):
            assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.shape == shape)
        assert sigma.dtype == torch.float32 and sigma.is_contiguous() and sigma.shape == (B,)
        for t in (d_hi, d_lo):
            assert t.dtype == torch.float16 and t.is_contiguous() and t.shape == (B, self._npad())
        assert partial.dtype == torch.float32 and partial.is_contiguous() and partial.shape == (B, (nv + 255) // 256, 32)
        with torch.cuda.device(xf.device):
            _lib.check(self.lib.dad3d_flame_backward_vertex(
                self._h, vposed.data_ptr(), xf.data_ptr(), grad_vertices.data_ptr() if grad_vertices is not None else None,
                grad_projected.data_ptr() if grad_projected is not None else None, B, float(image_size), 1 if to_2d else 0,
                sigma.data_ptr(), d_hi.data_ptr(), d_lo.data_ptr(), partial.data_ptr(),
                torch.cuda.current_stream(xf.device).cuda_stream), "dad3d_flame_backward_vertex")

    def backward_dense(self, d_hi: Tensor, d_lo: Tensor, dcoef: Tensor) -> None:
        """Dense stage: ``d_hi`` / ``d_lo`` [B, npad] fp16 -> ``dcoef`` [B, 448] fp32."""
        B = dcoef.shape[0]
        for t in (d_hi, d_lo):
            assert t.dtype == torch.float16 and t.is_contiguous() and t.shape == (B, self._npad())
        assert dcoef.dtype == torch.float32 and dcoef.is_contiguous() and dcoef.shape == (B, 448)
        with torch.cuda.device(dcoef.device):
            _lib.check(self.lib.dad3d_flame_backward_dense(self._h, d_hi.data_ptr(), d_lo.data_ptr(), B, dcoef.data_ptr(),
                                                           torch.cuda.current_stream(dcoef.device).cuda_stream),
                       "dad3d_flame_backward_dense")

    def backward_finalize(self, params: Tensor, dcoef: Tensor, partial: Tensor, sigma: Tensor, grad_params: Tensor, *,
                          flags: int = 0) -> None:
        """Finalize stage: the parameter gradients [B, num_params] from ``dcoef``, ``partial`` and ``sigma``."""
        B = params.shape[0]
        assert params.dtype == torch.float32 and params.is_contiguous() and params.shape == (B, self.num_params)
        assert dcoef.dtype == torch.float32 and dcoef.is_contiguous() and dcoef.shape == (B, 448)
        assert partial.dtype == torch.float32 and partial.is_contiguous()
        assert partial.shape == (B, (self.n_vertices + 255) // 256, 32)
        assert sigma.dtype == torch.float32 and sigma.is_contiguous() and sigma.shape == (B,)
        assert grad_params.dtype == torch.float32 and grad_params.is_contiguous() and grad_params.shape == params.shape
        with torch.cuda.device(params.device):
            _lib.check(self.lib.dad3d_flame_backward_finalize(
                self._h, params.data_ptr(), B, int(flags), dcoef.data_ptr(), partial.data_ptr(), sigma.data_ptr(),
                grad_params.data_ptr(), torch.cuda.current_stream(params.device).cuda_stream), "dad3d_flame_backward_finalize")

    def _check_out(self, t: Optional[Tensor], B: int, nc: int) -> None:
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous() and t.shape == (B, self.n_vertices, nc), t.shape

    def backward(self, params: Tensor, grad_vertices: Optional[Tensor], grad_projected: Optional[Tensor], *, to_2d: bool = True,
                 zero_rot: bool = False, zero_jaw: bool = False, image_size: float = 256.0) -> Tensor:
        """d L / d params [B, num_params] from d L / d vertices3d [B,V,3] and / or d L / d projected [B,V,2|3] (either may be
        None): the backward of :meth:`decode` (csrc/flame.cu ``dad3d_flame_backward``; dense part on wgmma)."""
        assert params.is_cuda and params.dtype == torch.float32 and params.ndim == 2 and params.shape[1] == self.num_params
        assert grad_vertices is not None or grad_projected is not None
        params = params.contiguous()
        B = params.shape[0]
        out = torch.zeros(B, self.num_params, dtype=torch.float32, device=params.device)
        if B == 0:
            return out
        gv = grad_vertices.to(torch.float32).contiguous() if grad_vertices is not None else None
        gp = grad_projected.to(torch.float32).contiguous() if grad_projected is not None else None
        if gv is not None:
            assert gv.shape == (B, self.n_vertices, 3)
        if gp is not None:
            assert gp.shape == (B, self.n_vertices, 2 if to_2d else 3)
        flags = (_lib.DAD3D_ZERO_ROT if zero_rot else 0) | (_lib.DAD3D_ZERO_JAW if zero_jaw else 0)
        nbytes = int(self.lib.dad3d_flame_backward_workspace_bytes(self._h, B))
        ws = self._ws.get(params.device, nbytes)
        stream = torch.cuda.current_stream(params.device).cuda_stream
        with torch.cuda.device(params.device):
            _lib.check(self.lib.dad3d_flame_backward(self._h, params.data_ptr(), B, flags,
                                                     gv.data_ptr() if gv is not None else None,
                                                     gp.data_ptr() if gp is not None else None, float(image_size),
                                                     1 if to_2d else 0, out.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                       "dad3d_flame_backward")
        return out

    def gather(self, src: Tensor, idx: Tensor) -> Tensor:
        """out[b,l,:] = src[b, idx[l], :]  (demo_utils.py:37-47 np.take)."""
        assert src.is_cuda and src.ndim == 3 and src.dtype == torch.float32
        src = src.contiguous()
        idx = idx.to(device=src.device, dtype=torch.int32).contiguous()
        B, V, nc = src.shape
        out = torch.empty(B, idx.numel(), nc, dtype=torch.float32, device=src.device)
        if out.numel() == 0:
            return out
        with torch.cuda.device(src.device):
            _lib.check(self.lib.dad3d_gather_landmarks(src.data_ptr(), B, V, nc, idx.data_ptr(), idx.numel(),
                                                       out.data_ptr(),
                                                       torch.cuda.current_stream(src.device).cuda_stream),
                       "dad3d_gather_landmarks")
        return out

    def gather_bary(self, src: Tensor, tri_idx: Tensor, bary: Tensor) -> Tensor:
        """out[b,l,:] = sum_k bary[l,k] * src[b, tri_idx[l,k], :]  (data/utils.py:120-206)."""
        assert src.is_cuda and src.ndim == 3 and src.dtype == torch.float32
        src = src.contiguous()
        tri_idx = tri_idx.to(device=src.device, dtype=torch.int32).contiguous()
        bary = bary.to(device=src.device, dtype=torch.float32).contiguous()
        B, V, nc = src.shape
        L = tri_idx.shape[0]
        out = torch.empty(B, L, nc, dtype=torch.float32, device=src.device)
        if out.numel() == 0:
            return out
        with torch.cuda.device(src.device):
            _lib.check(self.lib.dad3d_gather_landmarks_bary(src.data_ptr(), B, V, nc, tri_idx.data_ptr(),
                                                            bary.data_ptr(), L, out.data_ptr(),
                                                            torch.cuda.current_stream(src.device).cuda_stream),
                       "dad3d_gather_landmarks_bary")
        return out


class DecodeFunction(torch.autograd.Function):
    """``(vertices3d, projected) = decode(params)`` with a hand-written backward: makes the GPU decoder usable under autograd
    (training-side callers: losses/vertices_3d_loss.py:30-47, losses/reprojection_loss.py:22-46).  The forward uses the strict
    hi/lo blend; the backward is dad3d_flame_backward."""

    @staticmethod
    def forward(ctx, params: Tensor, decoder: "FlameDecoder", to_2d: bool, zero_rot: bool, image_size: float):
        p = params.detach().to(torch.float32).contiguous()
        v3, pj = decoder.decode(p, want_vertices=True, want_projected=True, to_2d=to_2d, zero_rot=zero_rot,
                                image_size=image_size, hilo=True)
        ctx.save_for_backward(p)
        ctx.decoder, ctx.to_2d, ctx.zero_rot, ctx.image_size = decoder, to_2d, zero_rot, image_size
        return v3, pj

    @staticmethod
    def backward(ctx, grad_v, grad_p):
        (p,) = ctx.saved_tensors
        g = ctx.decoder.backward(p, grad_v, grad_p, to_2d=ctx.to_2d, zero_rot=ctx.zero_rot, image_size=ctx.image_size)
        return g, None, None, None, None


class FLAMELayer(nn.Module):
    """Drop-in for the reference FLAMELayer (flame.py:117-229): same constructor and ``forward`` signature.

    ``forward`` accepts CPU or CUDA tensors inside ``flame_params``; the result lives where the inputs live (the
    reference keeps HeadMesh on the CPU, predictor.py:74), but the computation always happens on the GPU
    (``cuda:<cuda_id>``, default current device).
    """

    def __init__(self, consts: Dict[str, Any], batch_size: int = 1, flame_path: Optional[str] = None,
                 cuda_id: Optional[int] = None, static: Optional[Dict[str, np.ndarray]] = None) -> None:
        super().__init__()
        st = static if static is not None else load_flame_static(flame_path)
        self._static = st
        self.flame_constants = consts
        self.batch_size = batch_size
        self.dtype = torch.float32
        self._cuda_id = cuda_id
        self.strict = True      # the reference-facing ``forward`` (per-image calls) uses the 3-product hi/lo blend (2e-7)
        self._decoders: Dict[int, FlameDecoder] = {}
        # attributes other reference code reads (inference/pncc_estimator.py:72,90, demo_utils.py:108-111)
        self.flame_model = SimpleNamespace(v_template=st["v_template"], f=st.get("faces"))
        self.faces = st.get("faces")
        if self.faces is not None:
            self.register_buffer("faces_tensor", torch.as_tensor(np.asarray(self.faces, dtype=np.int64)))
        if "indices_2d" in st:
            self.register_buffer("indices_2d", torch.as_tensor(np.asarray(st["indices_2d"], dtype=np.int64)))
        self.register_buffer("v_template", torch.as_tensor(np.asarray(st["v_template"], dtype=np.float32)))

    def decoder(self, device: Optional[torch.device] = None) -> FlameDecoder:
        if device is None or torch.device(device).type != "cuda":
            if not torch.cuda.is_available():
                raise _lib.Dad3dError("FLAMELayer needs a CUDA (sm_90a) device: there is no CPU path")
            idx = self._cuda_id if self._cuda_id is not None else torch.cuda.current_device()
        else:
            device = torch.device(device)
            idx = device.index if device.index is not None else torch.cuda.current_device()
        dec = self._decoders.get(idx)
        if dec is None:
            dec = FlameDecoder(self._static, self.flame_constants, torch.device("cuda", idx))
            self._decoders[idx] = dec
        return dec

    def forward(self, flame_params: FlameParams, zero_rot: bool = False, zero_jaw: bool = False) -> torch.Tensor:
        """vertices: B x V x 3 (reference flame.py:182-229)."""
        packed = flame_params.packed().to(torch.float32)
        src_device = packed.device
        dec = self.decoder(src_device)
        v3, _ = dec.decode(packed.to(dec.device, non_blocking=True), want_vertices=True, want_projected=False,
                           zero_rot=zero_rot, zero_jaw=zero_jaw, hilo=self.strict)
        return v3 if src_device.type == "cuda" else v3.to(src_device)
