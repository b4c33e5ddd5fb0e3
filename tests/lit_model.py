"""Exact numpy model of the reference's lit render (Sim3DR/lighting.py:37-71, RenderPipeline.__call__ steps 1-5): the
per-vertex light of one head, every float32 operation in the reference's order, with a pluggable power function.

``pow=np.power`` is the reference itself (tests/test_lit_model_cpu.py pins the two bit for bit); ``pow=exact_pow``
(the default) is what the device computes: the correctly rounded float32 x ** e for integer e in [0, 16].  The
3-element sums are written left to right, ``(a0 + a1) + a2``, the order numpy's ``sum(axis=1)`` uses (also pinned).
Images are then the reference rasteriser with the light as colours (tests/raster_model.py, tests/frame_render_model.py)."""
from __future__ import annotations

import math
from typing import Optional

import numpy as np

F = np.float32
DEFAULTS = {"intensity_ambient": 0.3, "intensity_directional": 0.6, "intensity_specular": 0.1, "specular_exp": 5,
            "color_ambient": (1, 1, 1), "color_directional": (1, 1, 1), "light_pos": (0, 0, 5), "view_pos": (0, 0, 5)}


def round_f32(num: int, exp2: int) -> float:
    """num * 2**exp2 (num >= 0 an integer) rounded to the nearest float32, ties to even, with subnormals and overflow."""
    if num == 0:
        return 0.0
    top = num.bit_length() - 1 + exp2                  # exponent of the leading bit
    lsb = max(top - 23, -149)                          # exponent of the last bit a float32 keeps
    shift = lsb - exp2
    if shift <= 0:
        q = num << -shift
    else:
        q, rem = num >> shift, num & ((1 << shift) - 1)
        half = 1 << (shift - 1)
        if rem > half or (rem == half and q & 1):
            q += 1
    if q.bit_length() + lsb > 128:                     # beyond FLT_MAX: rounds to infinity
        return math.inf
    return math.ldexp(q, lsb)


def exact_pow_scalar(x, e: int) -> np.float32:
    """The correctly rounded float32 x ** e of a float32 x, e an integer >= 0, in exact integer arithmetic."""
    x = F(x)
    if e == 0:
        return F(1)
    if not np.isfinite(x) or x == 0:
        r = x
        for _ in range(e - 1):
            r = F(r * x)
        return r
    fr, ex = math.frexp(float(x))
    m, k = int(abs(fr) * (1 << 24)), ex - 24           # |x| = m * 2**k exactly
    mag = round_f32(m ** e, k * e)
    return F(-mag if (x < 0 and e % 2) else mag)


def exact_pow(x: np.ndarray, e: int) -> np.ndarray:
    """exact_pow_scalar over a float32 array (each distinct value once)."""
    x = np.asarray(x, F)
    u, inv = np.unique(x.reshape(-1).view(np.uint32), return_inverse=True)
    vals = np.array([exact_pow_scalar(v, e) for v in u.view(F)], F)
    return vals[inv].reshape(x.shape)


def vertex_normals(v: np.ndarray, t: np.ndarray) -> np.ndarray:
    """_get_normal (rasterize_kernel.cpp:158-215): face normals added to their vertices in triangle order, normalised."""
    v = np.ascontiguousarray(v, F)
    t = np.asarray(t, np.int64).reshape(-1, 3)
    p0, p1, p2 = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    a, b = p1 - p0, p2 - p0
    n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    acc = np.zeros_like(v)
    np.add.at(acc, t.reshape(-1), np.repeat(n, 3, axis=0))          # sequential, in triangle order per vertex
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        det = np.sqrt((acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1]) + acc[:, 2] * acc[:, 2])
        det = np.where(det <= 0, F(1e-6), det).astype(F)
        return (acc / det[:, None]).astype(F)


def _sum3(a: np.ndarray) -> np.ndarray:
    return (a[:, 0] + a[:, 1]) + a[:, 2]


def _norm(a: np.ndarray) -> np.ndarray:
    return a / np.sqrt(_sum3(a * a))[:, None]


def light(vertices: np.ndarray, triangles: np.ndarray, lighting: Optional[dict] = None, pow=exact_pow,
          normals: Optional[np.ndarray] = None) -> np.ndarray:
    """RenderPipeline(**lighting)'s ``light`` [nv,3] float32 for one head (vertices [nv,3] float32, as it receives them)."""
    kw = dict(DEFAULTS)
    kw.update(lighting or {})
    v = np.ascontiguousarray(vertices, F)
    vec = {k: np.asarray(kw[k], F).reshape(1, 3) for k in ("color_ambient", "color_directional", "light_pos", "view_pos")}
    ia, idr, isp = (kw[k] for k in ("intensity_ambient", "intensity_directional", "intensity_specular"))
    n = vertex_normals(v, triangles) if normals is None else normals
    out = np.zeros_like(v)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if ia > 0:
            out = out + F(ia) * vec["color_ambient"]
        vn = v.copy()                                                # norm_vertices (lighting.py:9-14)
        vn = vn - vn.min(0)[None, :]
        vn = vn / vn.max()
        vn = vn * F(2)
        vn = vn - vn.max(0)[None, :] / F(2)
        if idr > 0:
            direction = _norm(vec["light_pos"] - vn)
            cos = _sum3(n * direction)[:, None]
            out = out + F(idr) * (vec["color_directional"] * np.clip(cos, F(0), F(1)))
            if isp > 0:
                v2v = _norm(vec["view_pos"] - vn)
                reflection = F(2) * cos * n - direction
                spe = _sum3(pow(v2v * reflection, kw["specular_exp"]))[:, None]
                spe = np.where(cos != 0, np.clip(spe, F(0), F(1)), np.zeros_like(spe))
                out = out + (F(isp) * vec["color_directional"]) * np.clip(spe, F(0), F(1))
        return np.clip(out, F(0), F(1)).astype(F)
