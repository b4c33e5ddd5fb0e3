"""The demo's UV texture of every boxed head on the GPU (csrc/uv_texture.cu).

``demo.py``'s ``uv_texture`` output is ``UVTextureCreator._compute_texture_map`` (inference/uv_texture.py:21-47): a Python
loop over the 237 456 texels of ``texture_data.npy`` that samples the source image at each texel's barycentric point of the
head mesh, skipping texels whose interpolated psbody vertex normal faces away.  :func:`uv_textures` computes the same bytes
for a whole batch of heads, from device tensors and without a host synchronisation, so it runs inside a captured step.
The rules are restated in ``tests/uv_model.py``; DESIGN §4.13 lists them.

The table is the reference's own file, read at run time from a path the caller gives (:meth:`UvTextureTable.load`); the
repository does not carry it.
"""
from __future__ import annotations

import ctypes as C
import pickle
from typing import Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib

N_VERTICES = 5023                                     # FLAME's vertex count: the table's vertex ids index it


class _TableUnpickler(pickle.Unpickler):
    """texture_data.npy is a 0-d object array holding a dict of numpy arrays and ints.  Its pickle names exactly numpy's
    ndarray, dtype and array reconstructor; every other global is refused."""

    _ALLOWED = {("numpy", "ndarray"), ("numpy", "dtype"), ("numpy.core.multiarray", "_reconstruct"),
                ("numpy._core.multiarray", "_reconstruct")}

    def find_class(self, module, name):
        if (module, name) not in self._ALLOWED:
            raise pickle.UnpicklingError(f"texture table: global {module}.{name} is not allowed")
        if module == "numpy":
            return getattr(np, name)
        from numpy._core.multiarray import _reconstruct
        return _reconstruct


def read_table(path: str) -> Dict[str, object]:
    """The dict of the reference's ``texture_data.npy``, read as ``np.load(path, allow_pickle=True).item()`` does but
    through :class:`_TableUnpickler`."""
    with open(path, "rb") as f:
        version = np.lib.format.read_magic(f)
        if version == (1, 0):
            shape, _, dtype = np.lib.format.read_array_header_1_0(f)
        elif version == (2, 0):
            shape, _, dtype = np.lib.format.read_array_header_2_0(f)
        else:
            raise ValueError(f"{path}: unsupported .npy version {version}")
        if shape != () or dtype != np.dtype(object):
            raise ValueError(f"{path}: expected a 0-d object array, got {dtype} {shape}")
        obj = _TableUnpickler(f, encoding="latin1").load()
    if isinstance(obj, np.ndarray) and obj.shape == () and obj.dtype == object:
        obj = obj.item()
    if not isinstance(obj, dict):
        raise ValueError(f"{path}: expected a dict, got {type(obj).__name__}")
    return obj


def compact_table(table: Dict[str, object], n_vertices: int = N_VERTICES) -> Tuple[int, np.ndarray, np.ndarray, np.ndarray]:
    """The table's dict -> (img_size, texel [T] int32, vertex_ids [T,3] int32, bary [T,3] float64): entry i writes texel
    ``int(y_coords[id]) * img_size + int(x_coords[id])`` (id = valid_pixel_ids[i], truncated as ``.astype(int)``) from
    ``valid_pixel_3d_faces[i]`` with ``valid_pixel_b_coords[i]``.  Out-of-range ids, vertex ids or texels and duplicate
    texels raise ValueError: with distinct texels the reference loop's write order never matters."""
    try:
        S = int(table["img_size"])
        xs = np.asarray(table["x_coords"], dtype=np.float64).reshape(-1)
        ys = np.asarray(table["y_coords"], dtype=np.float64).reshape(-1)
        ids = np.asarray(table["valid_pixel_ids"])
        faces = np.asarray(table["valid_pixel_3d_faces"])
        bary = np.asarray(table["valid_pixel_b_coords"], dtype=np.float64)
    except KeyError as e:
        raise ValueError(f"texture table: missing {e}") from None
    T = int(ids.shape[0]) if ids.ndim == 1 else -1
    if T < 0 or faces.shape != (T, 3) or bary.shape != (T, 3) or xs.shape != ys.shape:
        raise ValueError("texture table: valid_pixel_ids [T], valid_pixel_3d_faces [T,3], valid_pixel_b_coords [T,3] and "
                         "x_coords / y_coords of one length")
    if not (1 <= S <= 16384):
        raise ValueError(f"texture table: img_size {S} outside [1, 16384]")
    if not (np.issubdtype(ids.dtype, np.integer) and np.issubdtype(faces.dtype, np.integer)):
        raise ValueError("texture table: valid_pixel_ids and valid_pixel_3d_faces must be integers")
    ids = ids.astype(np.int64)
    if T and (ids.min() < 0 or ids.max() >= xs.shape[0]):
        raise ValueError("texture table: valid_pixel_ids outside x_coords")
    faces = faces.astype(np.int64)
    if T and (faces.min() < 0 or faces.max() >= n_vertices):
        raise ValueError(f"texture table: vertex ids outside [0, {n_vertices})")
    x, y = xs[ids], ys[ids]
    if not (np.isfinite(x).all() and np.isfinite(y).all()):
        raise ValueError("texture table: texel coordinates are not finite")
    x, y = x.astype(np.int64), y.astype(np.int64)
    if T and (x.min() < 0 or x.max() >= S or y.min() < 0 or y.max() >= S):
        raise ValueError(f"texture table: texels outside the {S}x{S} image")
    texel = y * S + x
    if np.unique(texel).shape[0] != T:
        raise ValueError("texture table: duplicate texels")
    return S, texel.astype(np.int32), faces.astype(np.int32), np.ascontiguousarray(bary)


def faces_by_vertex(faces: np.ndarray, n_vertices: int) -> Tuple[np.ndarray, np.ndarray]:
    """psbody's ``faces_by_vertex(as_sparse_matrix=True)`` as CSR rows: (row [V+1], col [nnz]) int32, each vertex's
    distinct faces ascending."""
    f = np.asarray(faces, dtype=np.int64)
    v = f.reshape(-1)
    fid = np.repeat(np.arange(f.shape[0], dtype=np.int64), 3)
    pairs = np.unique(v * f.shape[0] + fid)                   # sorted by vertex, then face; one entry per (vertex, face)
    rows = pairs // f.shape[0]
    row = np.zeros(n_vertices + 1, dtype=np.int64)
    np.add.at(row, rows + 1, 1)
    return np.cumsum(row).astype(np.int32), (pairs % f.shape[0]).astype(np.int32)


class UvTextureTable:
    """The compacted texture table and the mesh's faces, uploaded once to one CUDA device (about 8 MB), so later calls
    and graph captures only read it."""

    def __init__(self, img_size: int, texel: np.ndarray, vertex_ids: np.ndarray, bary: np.ndarray, faces: np.ndarray,
                 device, n_vertices: int = N_VERTICES):
        self.img_size = int(img_size)
        self.n_vertices = int(n_vertices)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"UvTextureTable needs a CUDA device, got {self.device}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.texel = np.ascontiguousarray(texel, dtype=np.int32)
        self.vertex_ids = np.ascontiguousarray(vertex_ids, dtype=np.int32)
        self.bary = np.ascontiguousarray(bary, dtype=np.float64)
        self.faces = np.ascontiguousarray(faces, dtype=np.int32)
        row, col = faces_by_vertex(self.faces, self.n_vertices)
        self.lib = _lib.load()
        self.handle = C.c_void_p()
        _lib.check(self.lib.dad3d_uv_create(C.byref(self.handle), self.img_size, self.texel.ctypes.data,
                                            self.vertex_ids.ctypes.data, self.bary.ctypes.data, int(self.texel.shape[0]),
                                            self.faces.ctypes.data, int(self.faces.shape[0]), row.ctypes.data,
                                            col.ctypes.data, self.n_vertices, self.device.index), "dad3d_uv_create")

    @classmethod
    def load(cls, path: str, device, faces: Optional[np.ndarray] = None) -> "UvTextureTable":
        """The reference's ``inference/texture_data.npy`` at ``path`` on ``device``.  ``faces``: the mesh's triangles
        (default: FLAME's, ``assets/flame_static.npz``, which are the reference's ``generic_model.pkl['f']``)."""
        if faces is None:
            from .flame import load_flame_static
            faces = load_flame_static()["faces"]
        S, texel, vids, bary = compact_table(read_table(path))
        return cls(S, texel, vids, bary, faces, device)

    def __del__(self):
        h = getattr(self, "handle", None)
        if h:
            try:
                self.lib.dad3d_uv_destroy(h)
            except Exception:
                pass
            self.handle = None


def uv_textures(table: UvTextureTable, frames: Tensor, vertices: Tensor, frame_index: Optional[Tensor] = None,
                valid: Optional[Tensor] = None) -> Tensor:
    """The reference's ``_compute_texture_map(frames[frame_index[r]], Mesh(vertices[r], faces))`` of every head r ->
    [R, img_size, img_size, 3] uint8, on the tensors' device and that device's current stream.

    frames [F,H,W,3] uint8, vertices [R,V,3] fp32 (frame pixels with depth: ``projected_vertices`` of ``to_2d=False``),
    frame_index [R] int32 (None: every head on frame 0), valid [R] bool (None: all valid), all on ``table.device``.  Heads
    that are not valid, or whose frame index is outside [0, F), get an all-zero texture."""
    dev = vertices.device
    if dev != table.device:
        raise ValueError(f"uv_textures: the table is on {table.device}, the vertices on {dev}")
    if not (frames.dtype == torch.uint8 and frames.ndim == 4 and frames.shape[3] == 3 and frames.is_contiguous()
            and frames.device == dev and min(frames.shape[:3]) >= 1):
        raise ValueError("uv_textures: frames must be one contiguous non-empty [F,H,W,3] uint8 tensor on the vertices' device")
    if not (vertices.dtype == torch.float32 and vertices.ndim == 3 and vertices.shape[1:] == (table.n_vertices, 3)
            and vertices.is_contiguous()):
        raise ValueError(f"uv_textures: vertices must be a contiguous [R,{table.n_vertices},3] fp32 tensor")
    R = int(vertices.shape[0])
    if R > 65535:
        raise ValueError(f"uv_textures: at most 65535 heads per call, got {R}")
    for name, t, dt in (("frame_index", frame_index, torch.int32), ("valid", valid, torch.bool)):
        if t is not None and not (t.dtype == dt and tuple(t.shape) == (R,) and t.is_contiguous() and t.device == dev):
            raise ValueError(f"uv_textures: {name} must be a contiguous [{R}] {dt} tensor on the vertices' device")
    F, H, W = (int(d) for d in frames.shape[:3])
    S = table.img_size
    out = torch.empty(R, S, S, 3, dtype=torch.uint8, device=dev)
    lib = table.lib
    ws_bytes = int(lib.dad3d_uv_workspace_bytes(table.handle, R))
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.dad3d_uv_texture(table.handle, vertices.data_ptr(), R,
                                        valid.data_ptr() if valid is not None else None, frames.data_ptr(), F, H, W,
                                        frame_index.data_ptr() if frame_index is not None else None, out.data_ptr(),
                                        ws.data_ptr(), ws_bytes, torch.cuda.current_stream(dev).cuda_stream),
                   "dad3d_uv_texture")
    return out
