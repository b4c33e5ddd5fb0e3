"""Exact integer model of the demo's head and face wireframes (demo_utils.draw_mesh, lines 50-65), as csrc/wireframe.cu
draws them into whole frames.

``draw_mesh`` draws every edge of ``{subset}_edges.npy`` in file order with ``cv2.line(img, p, q, EDGE_COLOR, 1,
cv2.LINE_AA)``.  For a 3-channel uint8 image cv2 (4.13.0) takes ``LineAA`` (drawing.cpp); this module restates it, and
tests/test_wireframe_model_cpu.py pins it against the binary:

- the end points are shifted to 16.16 fixed point and clipped to the image by ``clipLine`` on ``Size2l``
  (:func:`tests.overlay_model.clip_line`, int64 with fp64 divisions);
- the walk takes one step per pixel along the major axis, from the first end to one past the second, and at each step
  stamps the three pixels across the minor axis around the line;
- each stamp's coverage ``a`` (0..255) is the filter table at the line's sub-pixel distance, scaled by the slope
  correction, and at the first two and last two steps by the end-point table;
- each stamped pixel is blended ``x += ((c - x) * a + 127) >> 8`` twice per channel (``a = 0`` leaves it unchanged).

A walk visits a pixel at most once, so in a frame the blends of one pixel come in (box, edge) order.  Integer expressions
keep C semantics (``_tdiv`` truncates toward zero; ``>>`` on negative values is the arithmetic shift of both languages).
"""
from __future__ import annotations

from typing import List, NamedTuple, Optional, Tuple

import numpy as np

from tests.overlay_model import XY_ONE, XY_SHIFT, _tdiv, clip_line, int_points

EDGE_COLOR = (39, 48, 218)                                 # demo_utils.EDGE_COLOR
WIREFRAME_KINDS = ("head_mesh", "face_mesh")
SUBSET_VERTICES = {"head_mesh": "flame_indices_face_w_ears", "face_mesh": "flame_indices_face"}

SLOPE_CORR = (181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
              203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254)
FILTER = (168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
          254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
          158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
          40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5)
_FILTER = np.array(FILTER, dtype=np.int64)


class Walk(NamedTuple):
    """One clipped LineAA walk: step k = 0..count visits major coordinate ``m0 + k`` with the minor position
    ``minor0 + k * step`` (16.16); ``x_major`` says which axis is the major one; ``ep`` is the end-point table."""
    x_major: bool
    m0: int
    count: int
    minor0: int
    step: int
    ep: Tuple[int, ...]


def end_point_table(i: int, j: int, slope: int) -> Tuple[int, ...]:
    """LineAA's ep_table from the 4-bit end fractions i, j (multiples of 8 in 0..0x78) and the corrected slope."""
    t0 = slope << 7
    t1 = ((0x78 - i) | 4) * slope
    t2 = (j | 4) * slope
    e13 = ((((j - i) & 0x78) | 4) * slope >> 8) & 0x1ff
    return (0, e13, (t1 >> 8) & 0x1ff, e13, ((((j - i) + 0x80) | 4) * slope >> 8) & 0x1ff, ((t1 + t0) >> 8) & 0x1ff,
            (t2 >> 8) & 0x1ff, ((t2 + t0) >> 8) & 0x1ff, slope)


def line_walk(w: int, h: int, p1, p2, clip: bool = True) -> Optional[Walk]:
    """LineAA's set-up for integer end points p1, p2 in a w x h image: None when clipLine leaves nothing."""
    x1, y1 = int(p1[0]) << XY_SHIFT, int(p1[1]) << XY_SHIFT
    x2, y2 = int(p2[0]) << XY_SHIFT, int(p2[1]) << XY_SHIFT
    if clip:
        ok, (x1, y1), (x2, y2) = clip_line(w << XY_SHIFT, h << XY_SHIFT, (x1, y1), (x2, y2))
        if not ok:
            return None
    dx, dy = x2 - x1, y2 - y1
    j = -1 if dx < 0 else 0
    ax = (dx ^ j) - j
    i = -1 if dy < 0 else 0
    ay = (dy ^ i) - i
    x_major = ax > ay
    if x_major:
        dy = (dy ^ j) - j
        if j:
            x1, x2, y1, y2 = x2, x1, y2, y1
        step = _tdiv(dy << XY_SHIFT, ax | 1)
        x2 += XY_ONE
        count = (x2 >> XY_SHIFT) - (x1 >> XY_SHIFT)
        f = -(x1 & (XY_ONE - 1))
        y1 += ((step * f) >> XY_SHIFT) + (XY_ONE >> 1)
        m0, minor0, e1, e2 = x1 >> XY_SHIFT, y1, x1, x2
    else:
        dx = (dx ^ i) - i
        if i:
            x1, x2, y1, y2 = x2, x1, y2, y1
        step = _tdiv(dx << XY_SHIFT, ay | 1)
        y2 += XY_ONE
        count = (y2 >> XY_SHIFT) - (y1 >> XY_SHIFT)
        f = -(y1 & (XY_ONE - 1))
        x1 += ((step * f) >> XY_SHIFT) + (XY_ONE >> 1)
        m0, minor0, e1, e2 = y1 >> XY_SHIFT, x1, y1, y2
    slope = (step >> (XY_SHIFT - 5)) & 0x3f
    slope ^= 0x3f if step < 0 else 0
    slope = 0x100 if slope & 0x20 else SLOPE_CORR[slope]
    ii = (e1 >> (XY_SHIFT - 7)) & 0x78
    jj = (e2 >> (XY_SHIFT - 7)) & 0x78
    return Walk(x_major, m0, count, minor0, step, end_point_table(ii, jj, slope))


def walk_stamps(walk: Walk, w: int, h: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(x, y, a) int64 of every pixel the walk blends, inside the w x h image, in drawing order."""
    k = np.arange(walk.count + 1, dtype=np.int64)
    major = walk.m0 + k
    minor = walk.minor0 + k * walk.step
    e = np.minimum(k, 2) * 3 + np.minimum(walk.count - k, 2)
    ep = np.array(walk.ep, dtype=np.int64)[e]
    dist = (minor >> (XY_SHIFT - 5)) & 31
    base = (minor >> XY_SHIFT) - 1
    filt = np.stack([_FILTER[dist + 32], _FILTER[dist], _FILTER[63 - dist]], axis=1)
    a = (ep[:, None] * filt >> 8) & 0xff
    mi = base[:, None] + np.arange(3)[None, :]
    ma = np.broadcast_to(major[:, None], mi.shape)
    x, y = (ma, mi) if walk.x_major else (mi, ma)
    keep = (x >= 0) & (x < w) & (y >= 0) & (y < h)
    return x[keep], y[keep], a[keep]


def line_aa_stamps(w: int, h: int, p1, p2) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    walk = line_walk(w, h, p1, p2)
    if walk is None:
        e = np.zeros(0, dtype=np.int64)
        return e, e, e
    return walk_stamps(walk, w, h)


def blend(x: np.ndarray, c: int, a: np.ndarray, twice: bool = True, half: int = 127) -> np.ndarray:
    """LineAA's ICV_PUT_POINT on one channel: ``x += ((c - x) * a + 127) >> 8``, applied twice."""
    x = x.astype(np.int64)
    for _ in range(2 if twice else 1):
        x = x + (((c - x) * a + half) >> 8)
    return x


def apply_stamps(img: np.ndarray, xs: np.ndarray, ys: np.ndarray, a: np.ndarray, color=EDGE_COLOR,
                 twice: bool = True, half: int = 127) -> None:
    """Blend the stamps into ``img`` [H,W,3] uint8 in the order given (the order matters only within one pixel)."""
    if not len(xs):
        return
    H, W = img.shape[:2]
    pix = ys * W + xs
    order = np.argsort(pix, kind="stable")
    ps = pix[order]
    start = np.r_[0, np.flatnonzero(np.diff(ps)) + 1]
    rank = np.arange(len(ps)) - np.repeat(start, np.diff(np.r_[start, len(ps)]))
    flat = img.reshape(-1, 3)
    for r in range(int(rank.max()) + 1):                  # one pixel per stamp in each rank: blend the ranks in order
        sel = order[rank == r]
        p = pix[sel]
        for ch in range(3):
            flat[p, ch] = blend(flat[p, ch], color[ch], a[sel], twice, half).astype(np.uint8)


def line_aa(img: np.ndarray, p1, p2, color=EDGE_COLOR) -> None:
    """cv2.line(img, p1, p2, color, 1, cv2.LINE_AA) on a 3-channel uint8 image."""
    H, W = img.shape[:2]
    apply_stamps(img, *line_aa_stamps(W, H, p1, p2), color=color)


# ----------------------------------------------------------------------------------------------------- edge tables
def mesh_edges(faces: np.ndarray, vertices: np.ndarray) -> np.ndarray:
    """The sorted unique (i < j) edges of the triangles ``faces`` with both ends in ``vertices`` -- row for row the
    reference's ``{subset}_edges.npy`` for the FLAME faces and the subset's vertex list."""
    f = np.asarray(faces, dtype=np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    e = np.unique(np.sort(e, axis=1), axis=0)
    keep = np.isin(e, np.asarray(vertices, dtype=np.int64)).all(axis=1)
    return e[keep]


def subset_edges(static, kind: str, vertex_key: Optional[str] = None) -> np.ndarray:
    return mesh_edges(static["faces"], static[vertex_key or SUBSET_VERTICES[kind]])


# ----------------------------------------------------------------------------------------------------- whole frames
def mesh_stamps(projected: np.ndarray, edges: np.ndarray, w: int, h: int,
                clip: bool = True) -> Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
    """Every stamp of draw_mesh for one head [N, >=2] into a w x h image, in edge order; None when an end point of an
    edge is not finite or does not fit int32 after truncation (cv2 raises, and draw_mesh has no output)."""
    xy, ok = int_points(projected)
    used = np.unique(edges)
    if not ok[used].all():
        return None
    pts = xy.tolist()
    xs, ys, as_ = [], [], []
    for a, b in edges:
        walk = line_walk(w, h, pts[a], pts[b], clip=clip)
        if walk is None:
            continue
        x, y, al = walk_stamps(walk, w, h)
        xs.append(x), ys.append(y), as_.append(al)
    if not xs:
        e = np.zeros(0, dtype=np.int64)
        return e, e, e
    return np.concatenate(xs), np.concatenate(ys), np.concatenate(as_)


def draw_mesh(img: np.ndarray, projected: np.ndarray, edges: np.ndarray, **kw) -> None:
    """demo_utils.draw_mesh's drawing on one image, in place (the returned ``mesh_vis``)."""
    H, W = img.shape[:2]
    twice, half = kw.pop("twice", True), kw.pop("half", 127)
    st = mesh_stamps(projected, edges, W, H, **kw)
    if st is not None:
        apply_stamps(img, *st, twice=twice, half=half)


def wireframe_frames(frames: np.ndarray, frame_of: np.ndarray, valid: np.ndarray, projected: np.ndarray,
                     edges: np.ndarray, box_order: Optional[List[int]] = None, **kw) -> np.ndarray:
    """"frame_<kind>" for every frame: a copy of ``frames`` with draw_mesh of each valid box's head (projected
    [R, N, >=2]) folded in, in box order."""
    out = frames.copy()
    for r in (range(len(valid)) if box_order is None else box_order):
        if valid[r]:
            draw_mesh(out[int(frame_of[r])], projected[r], edges, **kw)
    return out


def template_head(static, x: float, y: float, size: float, ncomp: int = 2) -> np.ndarray:
    """[N, ncomp] fp32: the FLAME template seen from the front (image y down), its face-with-ears part scaled to ``size``
    pixels and placed with its top-left corner at (x, y) -- a head-shaped wireframe for tests and timings."""
    v = np.asarray(static["v_template"], dtype=np.float64).copy()
    v[:, 1] = -v[:, 1]
    sub = v[np.asarray(static["flame_indices_face_w_ears"])]
    lo, hi = sub[:, :2].min(0), sub[:, :2].max(0)
    out = np.zeros((len(v), ncomp), dtype=np.float32)
    out[:, :2] = (v[:, :2] - lo) / (hi - lo).max() * size + [x, y]
    if ncomp == 3:
        out[:, 2] = v[:, 2] * size
    return out
