"""Exact numpy model of the reference's z-buffer rasteriser (Sim3DR/lib/rasterize_kernel.cpp `_rasterize`, alpha = 1), used
to check what the reference does not return: the winning triangle of every pixel (``tri_index`` of dad3d_rasterize_batch).

Arithmetic: every float32 operation in the reference's order (``get_point_weight`` :52-82, the depth and colour sums of
``_rasterize``), one numpy float32 operation each, so each is rounded like the reference's SSE code (no FMA).

Order: the reference visits triangles in index order and lets triangle i take pixel p when its depth is strictly greater
than the buffer.  The buffer starts at ``depth0`` and only grows, so the last triangle to take p is the FIRST one (lowest
index) whose depth equals the maximum over the triangles with depth > depth0[p]; equality is float equality, so -0 and +0
tie.  The model computes every (triangle, pixel) candidate of the bounding boxes at once and applies that rule per pixel.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

F = np.float32


def point_weights(px, py, p0x, p0y, p1x, p1y, p2x, p2y):
    """get_point_weight, elementwise over float32 arrays."""
    v0x, v0y = p2x - p0x, p2y - p0y
    v1x, v1y = p1x - p0x, p1y - p0y
    v2x, v2y = px - p0x, py - p0y
    dot00 = v0x * v0x + v0y * v0y
    dot01 = v0x * v1x + v0y * v1y
    dot02 = v0x * v2x + v0y * v2y
    dot11 = v1x * v1x + v1y * v1y
    dot12 = v1x * v2x + v1y * v2y
    den = dot00 * dot11 - dot01 * dot01
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = np.where(den == 0, F(0), F(1) / np.where(den == 0, F(1), den)).astype(F)
        u = (dot11 * dot02 - dot01 * dot12) * inv
        v = (dot00 * dot12 - dot01 * dot02) * inv
        w0 = (F(1) - u) - v
    return w0, v, u


def rasterize(vertices: np.ndarray, triangles: np.ndarray, colors: Optional[np.ndarray], h: int, w: int,
              image: Optional[np.ndarray] = None, depth0: Optional[np.ndarray] = None,
              reverse: bool = False) -> Tuple[Optional[np.ndarray], np.ndarray, np.ndarray]:
    """One head.  vertices [nv,3], triangles [ntri,3], colors [nv,c] or None; image [h,w,c] uint8 (zeros if None) and
    depth0 [h,w] (-1e8 if None) are the initial buffers.  Returns (image, depth, tri_index): the reference's image and depth
    buffer after the loop, and per pixel the triangle that wrote it last (-1: none), in depth-buffer rows."""
    v = np.ascontiguousarray(vertices, F)
    t = np.ascontiguousarray(triangles, np.int64).reshape(-1, 3)
    depth = np.full((h, w), -1e8, F) if depth0 is None else np.array(depth0, F, copy=True)
    c = 0 if colors is None else colors.shape[1]
    img = None
    if colors is not None:
        img = np.zeros((h, w, c), np.uint8) if image is None else np.array(image, np.uint8, copy=True)
    tri_index = np.full((h, w), -1, np.int32)
    if t.shape[0] == 0:
        return img, depth, tri_index
    px, py, pz = (v[t, k] for k in range(3))                          # [ntri,3] each
    with np.errstate(invalid="ignore"):
        x_min = np.maximum(np.ceil(px.min(1)).astype(np.int64), 0)
        x_max = np.minimum(np.floor(px.max(1)).astype(np.int64), w - 1)
        y_min = np.maximum(np.ceil(py.min(1)).astype(np.int64), 0)
        y_max = np.minimum(np.floor(py.max(1)).astype(np.int64), h - 1)
    bw, bh = x_max - x_min + 1, y_max - y_min + 1
    n = np.where((bw > 0) & (bh > 0), bw * bh, 0)
    tri = np.repeat(np.arange(t.shape[0]), n)
    off = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
    x = x_min[tri] + off % bw[tri]
    y = y_min[tri] + off // bw[tri]

    def weights(tri, x, y):
        return point_weights(x.astype(F), y.astype(F), px[tri, 0], py[tri, 0], px[tri, 1], py[tri, 1], px[tri, 2],
                             py[tri, 2])

    w0, w1, w2 = weights(tri, x, y)
    d = (w0 * pz[tri, 0] + w1 * pz[tri, 1]) + w2 * pz[tri, 2]
    pix = y * w + x
    keep = (w2 > 0) & (w1 > 0) & (w0 > 0) & (d > depth.reshape(-1)[pix])
    tri, x, y, d, pix = tri[keep], x[keep], y[keep], d[keep], pix[keep]
    if tri.size == 0:
        return img, depth, tri_index
    order = np.lexsort((tri, pix))                                    # by pixel, then ascending triangle index
    tri, x, y, d, pix = tri[order], x[order], y[order], d[order], pix[order]
    new_pix = np.r_[True, pix[1:] != pix[:-1]]
    group = np.cumsum(new_pix) - 1
    dmax = np.maximum.reduceat(d, np.flatnonzero(new_pix))
    cand = np.flatnonzero(d == dmax[group])
    first = cand[np.r_[True, group[cand][1:] != group[cand][:-1]]]    # the lowest-index maximal candidate of each pixel
    tri, x, y, d, pix = tri[first], x[first], y[first], d[first], pix[first]
    tri_index.reshape(-1)[pix] = tri
    w0, w1, w2 = weights(tri, x, y)
    depth.reshape(-1)[pix] = (w0 * pz[tri, 0] + w1 * pz[tri, 1]) + w2 * pz[tri, 2]
    if img is not None:
        col = np.ascontiguousarray(colors, F)
        yo = (h - 1 - y) if reverse else y
        for k in range(c):
            pc = (w0 * col[t[tri, 0], k] + w1 * col[t[tri, 1], k]) + w2 * col[t[tri, 2], k]
            old = img[yo, x, k].astype(F)
            val = (F(1) - F(1)) * old + (F(1) * F(255)) * pc
            img[yo, x, k] = val.astype(np.int32).astype(np.uint8)
    return img, depth, tri_index
