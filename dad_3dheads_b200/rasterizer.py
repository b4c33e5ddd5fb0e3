"""GPU drop-in for the reference's ``Sim3DR`` package (Sim3DR/Sim3DR.py:8-29): ``rasterize`` and ``get_normal`` with the same
signatures, numpy in / numpy out, bit-exact with the C++ rasteriser they wrap (csrc/rasterize.cu, SURVEY §8f row 4).  Used by
the reference's ``inference/pncc_estimator.py`` through ``compat/Sim3DR``.  No CPU fallback."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import _lib


def _device(cuda_id: Optional[int]) -> torch.device:
    if not torch.cuda.is_available():
        raise _lib.Dad3dError("dad_3dheads_b200.rasterizer needs a CUDA (sm_90a) device: there is no CPU path")
    return torch.device("cuda", torch.cuda.current_device() if cuda_id is None else cuda_id)


def rasterize(vertices: np.ndarray, triangles: np.ndarray, colors: np.ndarray, bg: Optional[np.ndarray] = None,
              height: Optional[int] = None, width: Optional[int] = None, channel: Optional[int] = None, reverse: bool = False,
              cuda_id: Optional[int] = None) -> np.ndarray:
    """Sim3DR.rasterize: z-buffer rendering of per-vertex colours onto ``bg`` (modified in place and returned, like the
    reference) or onto a black ``height x width x channel`` image.  vertices [N,3] float32 (pixels, depth), triangles [M,3] int,
    colors [N,C] in [0,1]."""
    lib = _lib.load()
    dev = _device(cuda_id)
    if bg is not None:
        height, width, channel = bg.shape
    else:
        assert height is not None and width is not None and channel is not None
        bg = np.zeros((height, width, channel), dtype=np.uint8)
    assert bg.dtype == np.uint8
    with torch.cuda.device(dev):
        v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float32)).to(dev)
        t = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int32)).to(dev)
        c = torch.from_numpy(np.ascontiguousarray(colors, dtype=np.float32)).to(dev)
        assert c.shape[1] == channel and v.shape[1] == 3 and t.shape[1] == 3
        img = torch.from_numpy(np.ascontiguousarray(bg)).to(dev)
        depth = torch.full((height, width), -1e8, dtype=torch.float32, device=dev)      # Sim3DR.py:22
        key = torch.empty(height * width, dtype=torch.int64, device=dev)
        _lib.check(lib.dad3d_rasterize(v.data_ptr(), t.data_ptr(), c.data_ptr(), int(t.shape[0]), img.data_ptr(), depth.data_ptr(),
                                       key.data_ptr(), height, width, channel, 1 if reverse else 0,
                                       torch.cuda.current_stream(dev).cuda_stream), "dad3d_rasterize")
        out = img.cpu().numpy()
    np.copyto(bg, out)
    return bg


def vertex_adjacency(triangles: np.ndarray, nver: int):
    """CSR list of the triangles around every vertex, ascending (the order of the reference's accumulation loop)."""
    t = np.asarray(triangles, dtype=np.int64)
    vert = t.reshape(-1)
    tri = np.repeat(np.arange(t.shape[0], dtype=np.int64), 3)
    order = np.lexsort((tri, vert))                       # by vertex, then by triangle index
    counts = np.bincount(vert, minlength=nver)
    offsets = np.zeros(nver + 1, dtype=np.int32)
    offsets[1:] = np.cumsum(counts)
    return offsets, tri[order].astype(np.int32)


def get_normal(vertices: np.ndarray, triangles: np.ndarray, cuda_id: Optional[int] = None) -> np.ndarray:
    """Sim3DR.get_normal: per-vertex normals [N,3] float32."""
    lib = _lib.load()
    dev = _device(cuda_id)
    nver = int(vertices.shape[0])
    off, adj = vertex_adjacency(triangles, nver)
    with torch.cuda.device(dev):
        v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float32)).to(dev)
        t = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int32)).to(dev)
        o = torch.from_numpy(off).to(dev)
        a = torch.from_numpy(adj).to(dev)
        out = torch.empty(nver, 3, dtype=torch.float32, device=dev)
        _lib.check(lib.dad3d_vertex_normals(v.data_ptr(), t.data_ptr(), o.data_ptr(), a.data_ptr(), nver, out.data_ptr(),
                                            torch.cuda.current_stream(dev).cuda_stream), "dad3d_vertex_normals")
        return out.cpu().numpy()
