"""Exact numpy model of several heads drawn into one frame (dad3d_rasterize_frames, PnccRenderer.render_frames), built on
tests/raster_model.py.

A frame's heads r1 < r2 < ... < rk form one union mesh: their vertices concatenated in head order, each head's triangles
offset by its vertex base, its colours repeated.  The reference's rasteriser called once on that mesh is the same
computation as calling it once per head, in head order, with the image and depth buffer carried from one call to the next
(both visit the same triangles in the same order against the same buffers).  The union mesh's winning triangle
u = rank * ntri + t splits into the head (the rank-th head of the frame) and the triangle t within it."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from tests import raster_model


def union_mesh(vertices: np.ndarray, triangles: np.ndarray, colors: Optional[np.ndarray]):
    """vertices [k,nv,3] -> (vertices [k*nv,3], triangles [k*ntri,3], colors [k*nv,c] or None)."""
    k, nv = vertices.shape[:2]
    t = np.asarray(triangles, np.int64)
    tris = (t[None] + (np.arange(k) * nv)[:, None, None]).reshape(-1, 3)
    cols = None if colors is None else np.tile(np.asarray(colors, np.float32), (k, 1))
    return np.ascontiguousarray(vertices, np.float32).reshape(-1, 3), tris, cols


def render_frame(vertices: np.ndarray, triangles: np.ndarray, colors: Optional[np.ndarray], h: int, w: int,
                 heads: Optional[np.ndarray] = None) -> Tuple[Optional[np.ndarray], np.ndarray, np.ndarray, np.ndarray]:
    """One frame.  vertices [k,nv,3] (z as depth: larger wins), the frame's heads in head order; ``heads`` [k] their head
    numbers (default 0..k-1).  Returns (image [h,w,c] uint8 on black or None, depth [h,w] from -1e8, tri_index [h,w],
    head_index [h,w]), -1 for background in both index maps."""
    k = int(vertices.shape[0])
    heads = np.arange(k) if heads is None else np.asarray(heads)
    ntri = int(np.asarray(triangles).shape[0])
    if k == 0:
        img = None if colors is None else np.zeros((h, w, colors.shape[1]), np.uint8)
        none = np.full((h, w), -1, np.int32)
        return img, np.full((h, w), -1e8, np.float32), none, none.copy()
    v, t, c = union_mesh(vertices, triangles, colors)
    img, depth, u = raster_model.rasterize(v, t, c, h, w)
    cover = u >= 0
    tri = np.where(cover, u % ntri, -1).astype(np.int32)
    head = np.where(cover, heads[np.where(cover, u // ntri, 0)], -1).astype(np.int32)
    return img, depth, tri, head


def render_frames(vertices: np.ndarray, triangles: np.ndarray, colors: Optional[np.ndarray], frame_of_head: np.ndarray,
                  n_frames: int, h: int, w: int):
    """B heads [B,nv,3] into ``n_frames`` frames by ``frame_of_head`` [B] (entries outside [0, n_frames) draw nothing) ->
    (images [F,h,w,c] or None, depth [F,h,w], tri_index [F,h,w], head_index [F,h,w]); head_index holds head numbers b."""
    fo = np.asarray(frame_of_head)
    per = []
    for f in range(n_frames):
        heads = np.flatnonzero(fo == f)
        per.append(render_frame(vertices[heads], triangles, colors, h, w, heads))
    img = None if colors is None else np.stack([p[0] for p in per]) if per else None
    return (img,) + tuple(np.stack([p[i] for p in per]) for i in (1, 2, 3))
