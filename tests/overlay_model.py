"""Exact numpy model of the demo's landmark and pose overlays (demo_utils.py:22-47, :68-94) and of calculate_rpy
(model_training/model/flame.py:238-264), as csrc/overlay.cu computes them.

The drawing rules restate what cv2 (4.13.0) does for the calls the demo makes; tests/test_overlay_model_cpu.py pins each
rule against the cv2 binary and the whole processors against the unmodified demo_utils.py:

- ``cv2.circle(img, c, r, color, -1)`` (LINE_8, shift 0) is the integer midpoint circle, filled with horizontal spans;
- ``cv2.line`` of thickness 1 is the clipped 8-connected line iterator, walked left to right;
- ``cv2.line`` of thickness t >= 2 is a four-corner polygon in 16-bit fixed point (its outline drawn by the fixed-point
  line, its inside by the convex scan-line fill) plus two filled circles of radius (t + 1) // 2 at the ends;
- ``cv2.arrowedLine`` (tipLength 0.1) is the shaft and two tip segments whose far points are cvRound of fp64 expressions.

Every integer expression keeps C semantics: ``_tdiv`` truncates toward zero where Python's ``//`` floors, and
``>>`` on negative values is the arithmetic shift both languages share.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
POINT_COLOR = (255, 0, 0)                                # demo_utils.POINT_COLOR
ARROW_COLORS = ((0, 0, 255), (0, 255, 0), (255, 0, 0))   # draw_pose's arrows, in drawing order
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
OVERLAY_KINDS = ("68_landmarks", "191_landmarks", "445_landmarks", "pose")
POSE_RECORD_INTS = 32


def _tdiv(a: int, b: int) -> int:
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def cv_round(v: float) -> int:
    """cvRound(double): round half to even (SSE2 cvtsd2si in the default rounding mode)."""
    return int(np.rint(v))


# ----------------------------------------------------------------------------------------------------- filled circle
def circle_spans(r: int) -> List[Tuple[int, int, int]]:
    """(dy, x0, x1) spans of cv2's filled Circle of radius r around (0, 0), in the order Circle visits them."""
    spans = []
    err, dx, dy, plus, minus = 0, r, 0, 1, 2 * r - 1
    while dx >= dy:
        spans += [(-dy, -dx, dx), (dy, -dx, dx), (-dx, -dy, dy), (dx, -dy, dy)]
        dy += 1
        err += plus
        plus += 2
        m = (1 if err <= 0 else 0) - 1
        err -= minus & m
        dx += m
        minus -= m & 2
    return spans


def disk_offsets(r: int) -> np.ndarray:
    """[n, 2] (dx, dy) pixel offsets the filled circle of radius r covers (each once)."""
    s = set()
    for dy, x0, x1 in circle_spans(r):
        s.update((x, dy) for x in range(x0, x1 + 1))
    return np.array(sorted(s), dtype=np.int64).reshape(-1, 2)


def fill_circle(img: np.ndarray, cx: int, cy: int, r: int, color, clip=None) -> None:
    """cv2.circle(img, (cx, cy), r, color, -1) with LINE_8 and no shift; ``clip`` = (w, h) of the drawable area
    (default: the image)."""
    w, h = clip if clip is not None else (img.shape[1], img.shape[0])
    for dy, x0, x1 in circle_spans(r):
        y = cy + dy
        a, b = max(cx + x0, 0), min(cx + x1, w - 1)
        if 0 <= y < h and a <= b:
            img[y, a:b + 1] = color


# ----------------------------------------------------------------------------------------------------- thin lines
def clip_line(w: int, h: int, p1, p2) -> Tuple[bool, Tuple[int, int], Tuple[int, int]]:
    """cv::clipLine over int64 points and a w x h area."""
    if w <= 0 or h <= 0:
        return False, p1, p2
    right, bottom = w - 1, h - 1
    x1, y1 = p1
    x2, y2 = p2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, (x1, y1), (x2, y2)


def line_pixels(w: int, h: int, p1, p2) -> List[Tuple[int, int]]:
    """Pixels of cv2.line(..., thickness=1, LINE_8) in a w x h area: cv::LineIterator(8, leftToRight)."""
    p1, p2 = (int(p1[0]), int(p1[1])), (int(p2[0]), int(p2[1]))
    if not (0 <= p1[0] < w and 0 <= p2[0] < w and 0 <= p1[1] < h and 0 <= p2[1] < h):
        ok, p1, p2 = clip_line(w, h, p1, p2)
        if not ok:
            return []
    dx, dy = p2[0] - p1[0], p2[1] - p1[1]
    sx, sy = 1, 1
    if dx < 0:                                           # leftToRight: walk from the left end
        dx, dy = -dx, -dy
        p1, p2 = p2, p1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
    err = dx - (dy + dy)
    plus, minus = dx + dx, -(dy + dy)
    x, y = p1
    out = []
    for _ in range(dx + 1):
        out.append((x, y))
        step_minor = err < 0
        err += minus + (plus if step_minor else 0)
        if vert:
            y += sy
            if step_minor:
                x += sx
        else:
            x += sx
            if step_minor:
                y += sy
    return out


def line2_pixels(w: int, h: int, p1, p2) -> List[Tuple[int, int]]:
    """Pixels of cv2's fixed-point Line2 (16-bit fraction) in a w x h area: the outline of a thick line's polygon."""
    ok, (x1, y1), (x2, y2) = clip_line(w << XY_SHIFT, h << XY_SHIFT, p1, p2)
    if not ok:
        return []
    dx, dy = x2 - x1, y2 - y1
    j = -1 if dx < 0 else 0
    ax = (dx ^ j) - j
    i = -1 if dy < 0 else 0
    ay = (dy ^ i) - i
    if ax > ay:
        dy = (dy ^ j) - j
        if j:
            x1, x2, y1, y2 = x2, x1, y2, y1
        x_step, y_step = XY_ONE, _tdiv(dy << XY_SHIFT, ax | 1)
        ecount = (x2 - x1) >> XY_SHIFT
    else:
        dx = (dx ^ i) - i
        if i:
            x1, x2, y1, y2 = x2, x1, y2, y1
        x_step, y_step = _tdiv(dx << XY_SHIFT, ay | 1), XY_ONE
        ecount = (y2 - y1) >> XY_SHIFT
    x1 += XY_ONE >> 1
    y1 += XY_ONE >> 1
    out = [((x2 + (XY_ONE >> 1)) >> XY_SHIFT, (y2 + (XY_ONE >> 1)) >> XY_SHIFT)]
    if ax > ay:
        x1 >>= XY_SHIFT
        while ecount >= 0:
            out.append((x1, y1 >> XY_SHIFT))
            x1 += 1
            y1 += y_step
            ecount -= 1
    else:
        y1 >>= XY_SHIFT
        while ecount >= 0:
            out.append((x1 >> XY_SHIFT, y1))
            x1 += x_step
            y1 += 1
            ecount -= 1
    return [(x, y) for x, y in out if 0 <= x < w and 0 <= y < h]


def convex_poly_spans(w: int, h: int, v: Sequence[Tuple[int, int]]) -> List[Tuple[int, int, int]]:
    """(y, x0, x1) spans of cv2's FillConvexPoly scan-line fill (shift 16, LINE_8) in a w x h area, outline excluded."""
    npts = len(v)
    delta = XY_ONE >> 1
    xmin = xmax = v[0][0]
    ymin = ymax = v[0][1]
    imin = 0
    for k, (px, py) in enumerate(v):
        if py < ymin:
            ymin, imin = py, k
        ymax, xmax, xmin = max(ymax, py), max(xmax, px), min(xmin, px)
    xmin, xmax = (xmin + delta) >> XY_SHIFT, (xmax + delta) >> XY_SHIFT
    ymin, ymax = (ymin + delta) >> XY_SHIFT, (ymax + delta) >> XY_SHIFT
    if npts < 3 or xmax < 0 or ymax < 0 or xmin >= w or ymin >= h:
        return []
    ymax = min(ymax, h - 1)
    e_idx, e_di, e_ye, e_x, e_dx = [imin, imin], [1, npts - 1], [ymin, ymin], [-XY_ONE, -XY_ONE], [0, 0]
    edges = npts
    y = ymin
    spans = []
    while True:
        for k in range(2):
            if y >= e_ye[k]:
                idx0, di = e_idx[k], e_di[k]
                idx = idx0 + di
                if idx >= npts:
                    idx -= npts
                while True:                                  # for (; edges-- > 0; )
                    go = edges > 0
                    edges -= 1
                    if not go:
                        break
                    ty = (v[idx][1] + delta) >> XY_SHIFT
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        e_ye[k] = ty
                        e_dx[k] = _tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        e_x[k] = xs
                        e_idx[k] = idx
                        break
                    idx0 = idx
                    idx += di
                    if idx >= npts:
                        idx -= npts
        if edges < 0:
            break
        if y >= 0:
            left, right = (1, 0) if e_x[0] > e_x[1] else (0, 1)
            xx1 = (e_x[left] + delta) >> XY_SHIFT
            xx2 = (e_x[right] + delta) >> XY_SHIFT
            if xx2 >= 0 and xx1 < w:
                spans.append((y, max(xx1, 0), min(xx2, w - 1)))
        e_x[0] += e_dx[0]
        e_x[1] += e_dx[1]
        y += 1
        if y > ymax:
            break
    return spans


def thick_line_pixels(w: int, h: int, p0, p1, t: int) -> set:
    """Pixels of cv2.line(..., thickness=t, LINE_8), t >= 2, in a w x h area: the segment clipped to the area grown
    by t on every side, then ThickLine with both caps."""
    ok, p0, p1 = clip_line(w + 2 * t, h + 2 * t, (int(p0[0]) + t, int(p0[1]) + t), (int(p1[0]) + t, int(p1[1]) + t))
    if not ok:
        return set()
    p0, p1 = (p0[0] - t, p0[1] - t), (p1[0] - t, p1[1] - t)
    P0 = (int(p0[0]) << XY_SHIFT, int(p0[1]) << XY_SHIFT)
    P1 = (int(p1[0]) << XY_SHIFT, int(p1[1]) << XY_SHIFT)
    px = set()
    dx = (P0[0] - P1[0]) / XY_ONE
    dy = (P1[1] - P0[1]) / XY_ONE
    r = dx * dx + dy * dy
    odd = t & 1
    tt = t << (XY_SHIFT - 1)
    if abs(r) > np.finfo(np.float64).eps:
        r = (tt + odd * XY_ONE * 0.5) / math.sqrt(r)
        dpx, dpy = cv_round(dy * r), cv_round(dx * r)
        pt = [(P0[0] + dpx, P0[1] + dpy), (P0[0] - dpx, P0[1] - dpy), (P1[0] - dpx, P1[1] - dpy),
              (P1[0] + dpx, P1[1] + dpy)]
        prev = pt[3]
        for q in pt:                                         # the outline, Line2 from the previous corner
            px.update(line2_pixels(w, h, prev, q))
            prev = q
        for y, a, b in convex_poly_spans(w, h, pt):
            px.update((x, y) for x in range(a, b + 1))
    rad = (tt + (XY_ONE >> 1)) >> XY_SHIFT
    for P in (P0, P1):
        cx, cy = (P[0] + (XY_ONE >> 1)) >> XY_SHIFT, (P[1] + (XY_ONE >> 1)) >> XY_SHIFT
        for ddy, x0, x1 in circle_spans(rad):
            y = cy + ddy
            if 0 <= y < h:
                px.update((x, y) for x in range(max(cx + x0, 0), min(cx + x1, w - 1) + 1))
    return px


def segment_pixels(w: int, h: int, p0, p1, t: int) -> set:
    """cv2.line(img, p0, p1, color, t) with LINE_8 in a w x h area, t >= 1."""
    if t <= 1:
        return set(line_pixels(w, h, p0, p1))
    return thick_line_pixels(w, h, p0, p1, t)


def arrow_tips(p1, p2) -> Tuple[Tuple[int, int], Tuple[int, int], List[float]]:
    """cv2.arrowedLine's two tip points (tipLength 0.1) and the fp64 values that were rounded."""
    tip = math.sqrt(float(p1[0] - p2[0]) ** 2 + float(p1[1] - p2[1]) ** 2) * 0.1
    ang = math.atan2(float(p1[1]) - p2[1], float(p1[0]) - p2[0])
    vals = [p2[0] + tip * math.cos(ang + math.pi / 4), p2[1] + tip * math.sin(ang + math.pi / 4),
            p2[0] + tip * math.cos(ang - math.pi / 4), p2[1] + tip * math.sin(ang - math.pi / 4)]
    r = [cv_round(v) for v in vals]
    return (r[0], r[1]), (r[2], r[3]), vals


def arrow_segments(p1, p2) -> List[Tuple[Tuple[int, int], Tuple[int, int]]]:
    a, b, _ = arrow_tips(p1, p2)
    return [(tuple(p1), tuple(p2)), (a, tuple(p2)), (b, tuple(p2))]


def arrowed_line(img: np.ndarray, p1, p2, color, t: int) -> None:
    h, w = img.shape[:2]
    for a, b in arrow_segments(p1, p2):
        for x, y in segment_pixels(w, h, a, b, t):
            img[y, x] = color


# ----------------------------------------------------------------------------------------------------- calculate_rpy
def _f32(v) -> np.float32:
    return np.float32(v)


def rot_mat_from_6dof(v: np.ndarray) -> np.ndarray:
    """model/utils.py:92-101 in fp32, in torch's CPU operation order: F.normalize is x / max(|x|, 1e-12) with
    |x| = sqrt(fma(x2, x2, fma(x1, x1, x0 * x0))); torch.cross's component i is fma(a_j, b_k, -(a_k * b_j)).  Columns
    b1, b2, b3.  The fma is evaluated as one float64 sum rounded to fp32 (the product is exact in float64)."""
    v = np.asarray(v, dtype=np.float32)
    vx, vy = v[:3], v[3:6]

    def fma(x, y, z):
        return _f32(np.float64(x) * np.float64(y) + np.float64(z))

    def normalize(a):
        n = np.sqrt(fma(a[2], a[2], fma(a[1], a[1], _f32(a[0] * a[0]))), dtype=np.float32)
        n = n if not n < np.float32(1e-12) else np.float32(1e-12)
        return np.array([a[0] / n, a[1] / n, a[2] / n], dtype=np.float32)

    def cross(a, b):
        return np.array([fma(a[1], b[2], -_f32(a[2] * b[1])), fma(a[2], b[0], -_f32(a[0] * b[2])),
                         fma(a[0], b[1], -_f32(a[1] * b[0]))], dtype=np.float32)

    b1 = normalize(vx)
    b3 = normalize(cross(b1, vy))
    b2 = -cross(b1, b3)
    return np.stack((b1, b2, b3), axis=-1).astype(np.float32)


def polar_factor(m: np.ndarray) -> np.ndarray:
    """The orthogonal polar factor U Vt of a nearly orthogonal 3 x 3 matrix, as the kernel computes it: three Newton steps
    X <- (X + X^-T) / 2 in fp64, X^-T = cofactor(X) / det(X).  scipy's from_matrix takes U Vt by SVD whenever the Gram
    matrix is not the identity to 1e-12 (always, for a matrix built from fp32 vectors, which is ~1e-7 off); the two agree
    to ~1e-15."""
    x = [[float(v) for v in row] for row in np.asarray(m, dtype=np.float64)]
    for _ in range(3):
        c = [[x[(i + 1) % 3][(j + 1) % 3] * x[(i + 2) % 3][(j + 2) % 3] - x[(i + 1) % 3][(j + 2) % 3] * x[(i + 2) % 3][(j + 1) % 3]
              for j in range(3)] for i in range(3)]
        det = x[0][0] * c[0][0] + x[0][1] * c[0][1] + x[0][2] * c[0][2]
        x = [[(x[i][j] + c[i][j] / det) * 0.5 for j in range(3)] for i in range(3)]
    return np.array(x, dtype=np.float64)


def quat_from_matrix(m: np.ndarray) -> np.ndarray:
    """scipy 1.18 Rotation.from_matrix's quaternion of an orthogonal matrix (the largest of the diagonal and the trace
    picks the formula), normalised.  :func:`rpy_from_rotation` applies it to :func:`polar_factor` of the matrix."""
    m = np.asarray(m, dtype=np.float64)
    tr = m[0, 0] + m[1, 1] + m[2, 2]
    choice = int(np.argmax([m[0, 0], m[1, 1], m[2, 2], tr]))
    if choice == 0:
        q = [1 - tr + 2 * m[0, 0], m[1, 0] + m[0, 1], m[2, 0] + m[0, 2], m[2, 1] - m[1, 2]]
    elif choice == 1:
        q = [m[1, 0] + m[0, 1], 1 - tr + 2 * m[1, 1], m[2, 1] + m[1, 2], m[0, 2] - m[2, 0]]
    elif choice == 2:
        q = [m[2, 0] + m[0, 2], m[2, 1] + m[1, 2], 1 - tr + 2 * m[2, 2], m[1, 0] - m[0, 1]]
    else:
        q = [m[2, 1] - m[1, 2], m[0, 2] - m[2, 0], m[1, 0] - m[0, 1], 1 + tr]
    q = np.array(q, dtype=np.float64)
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return q / n


def euler_xyz_from_quat(q: np.ndarray) -> np.ndarray:
    """scipy 1.18 as_euler("xyz") (extrinsic; Bernardes & Viollet's quaternion method), radians."""
    a, b, c, d = q[3] - q[1], q[0] + q[2], q[1] + q[3], q[2] - q[0]
    half_sum, half_diff = math.atan2(b, a), math.atan2(d, c)
    mid = 2 * math.atan2(math.hypot(c, d), math.hypot(a, b))
    case1 = abs(mid) <= 1e-7
    case2 = abs(mid - math.pi) <= 1e-7
    if case1:
        first, third = 2 * half_sum, 0.0
    elif case2:
        first, third = -2 * half_diff, 0.0
    else:
        first, third = half_sum - half_diff, half_sum + half_diff
    ang = np.array([first, mid - math.pi / 2, third], dtype=np.float64)
    return np.mod(ang + math.pi, 2 * math.pi) - math.pi


def limit_angle(angle: float, pi: float = 180.0) -> float:
    """flame.py:239-251."""
    if angle < -pi:
        k = -2 * (int(angle / pi) // 2)
        angle = angle + k * pi
    if angle > pi:
        k = 2 * ((int(angle / pi) + 1) // 2)
        angle = angle - k * pi
    return angle


def rpy_from_rotation(rot6: np.ndarray) -> Tuple[float, float, float]:
    """calculate_rpy (flame.py:254-259) on one head's six rotation parameters -> (roll, pitch, yaw) degrees."""
    m = rot_mat_from_6dof(rot6).astype(np.float64)
    ang = euler_xyz_from_quat(quat_from_matrix(polar_factor(m.T))) * (180.0 / np.pi)
    return limit_angle(ang[2]), limit_angle(ang[0] - 180), limit_angle(ang[1])


# ----------------------------------------------------------------------------------------------------- draw_pose
def pose_geometry(rpy, crop_w: int, crop_h: int) -> Dict[str, object]:
    """draw_pose's integers for one box from its (roll, pitch, yaw): centre, the three arrow ends, thickness, and the
    fp64 values truncated to get the ends (for boundary checks)."""
    tdx, tdy = crop_w // 2, crop_h // 2
    roll = rpy[0] * np.pi / 180
    pitch = rpy[1] * np.pi / 180
    yaw = -(rpy[2] * np.pi / 180)
    size = crop_h // 10
    cy, sy, cr, sr, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(roll), math.sin(roll), math.cos(pitch), math.sin(pitch)
    vals = [size * (cy * cr) + tdx, size * (cp * sr + cr * sp * sy) + tdy,
            size * (-cy * sr) + tdx, size * (cp * cr - sp * sy * sr) + tdy,
            size * sy + tdx, size * (-cy * sp) + tdy]
    ends = [(int(vals[0]), int(vals[1])), (int(vals[2]), int(vals[3])), (int(vals[4]), int(vals[5]))]
    return {"centre": (tdx, tdy), "ends": ends, "thickness": int(crop_h * 0.005), "values": vals}


def pose_record(rpy, crop_box, frame: int, valid: bool) -> np.ndarray:
    """The kernel's per-box pose record (include/dad3d.h dad3d_pose_geometry): [draw, frame, x, y, w, h, t, 0,
    cx, cy, then per arrow: end x, end y, tip1 x, tip1 y, tip2 x, tip2 y, then zeros]."""
    x, y, w, h = (int(v) for v in crop_box)
    g = pose_geometry(rpy, w, h)
    rec = np.zeros(POSE_RECORD_INTS, dtype=np.int32)
    rec[:8] = [int(valid and g["thickness"] >= 1), frame, x, y, w, h, g["thickness"], 0]
    rec[8:10] = g["centre"]
    for k, e in enumerate(g["ends"]):
        a, b, _ = arrow_tips(g["centre"], e)
        rec[10 + 6 * k: 16 + 6 * k] = [e[0], e[1], a[0], a[1], b[0], b[1]]
    return rec


def near_boundaries(rpy, crop_w: int, crop_h: int, tol: float = 1e-9) -> int:
    """How many of draw_pose's fp64 values lie within ``tol`` of the integer boundary their conversion cuts at (an
    integer for the truncated ends, a half-integer for the rounded tips)."""
    g = pose_geometry(rpy, crop_w, crop_h)
    n = sum(abs(v - round(v)) < tol and v != round(v) for v in g["values"])
    for e in g["ends"]:
        for v in arrow_tips(g["centre"], e)[2]:
            n += abs(abs(v - math.floor(v)) - 0.5) < tol
    return n


def draw_pose_record(img: np.ndarray, rec: np.ndarray, key: Optional[np.ndarray] = None, box: int = 0) -> None:
    """Raster one pose record into its frame ``img``: clipped to its crop view, and to the frame (records built from crops
    of the same frame size always lie inside it)."""
    if not rec[0]:
        return
    x, y, w, h, t = (int(v) for v in rec[2:7])
    H, W = img.shape[:2]
    c = (int(rec[8]), int(rec[9]))
    for k in range(3):
        e = (int(rec[10 + 6 * k]), int(rec[11 + 6 * k]))
        a = (int(rec[12 + 6 * k]), int(rec[13 + 6 * k]))
        b = (int(rec[14 + 6 * k]), int(rec[15 + 6 * k]))
        for p, q in ((c, e), (a, e), (b, e)):
            for px, py in segment_pixels(w, h, p, q, t):
                if 0 <= x + px < W and 0 <= y + py < H:
                    img[y + py, x + px] = ARROW_COLORS[k]


# ----------------------------------------------------------------------------------------------------- points
def point_radius(H: int, W: int) -> int:
    """draw_points' radius (demo_utils.py:26)."""
    return max(1, int(min(H, W) * 0.005))


def int_points(src: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(x, y) int64 as ``astype(int)`` gives them, and a mask of the points cv2 accepts (finite, within int32)."""
    src = np.asarray(src)
    xy = src[..., :2]
    if src.dtype.kind == "f":
        d = xy.astype(np.float64)
        ok = np.all(np.isfinite(d) & (d > INT32_MIN - 1.0) & (d < INT32_MAX + 1.0), axis=-1)
        with np.errstate(invalid="ignore"):
            xy = np.where(np.isfinite(d), np.trunc(d), 0).astype(np.int64)
    else:
        xy = xy.astype(np.int64)
        ok = np.all((xy >= INT32_MIN) & (xy <= INT32_MAX), axis=-1)
    return xy, ok


def draw_points(img: np.ndarray, pts: np.ndarray, ok: Optional[np.ndarray] = None, color=POINT_COLOR) -> None:
    """draw_points (demo_utils.py:22-29) for int64 points [n, 2] into one frame; points not ``ok`` draw nothing."""
    H, W = img.shape[:2]
    off = disk_offsets(point_radius(H, W))
    pts = np.asarray(pts, dtype=np.int64).reshape(-1, 2)
    if ok is not None:
        pts = pts[np.asarray(ok).reshape(-1)]
    if not len(pts):
        return
    px = pts[:, None, 0] + off[None, :, 0]
    py = pts[:, None, 1] + off[None, :, 1]
    m = (px >= 0) & (px < W) & (py >= 0) & (py < H)
    img[py[m], px[m]] = color


# ----------------------------------------------------------------------------------------------------- whole frames
def overlay_frames(frames: np.ndarray, kind: str, crop_boxes: np.ndarray, frame_of: np.ndarray, valid: np.ndarray,
                   points: Optional[np.ndarray] = None, projected: Optional[np.ndarray] = None,
                   index: Optional[np.ndarray] = None, pose_records: Optional[np.ndarray] = None) -> np.ndarray:
    """"frame_<kind>" for every frame: a copy of ``frames`` with each valid box's overlay drawn in box order."""
    out = frames.copy()
    R = len(crop_boxes)
    for r in range(R):
        if not valid[r]:
            continue
        f = int(frame_of[r])
        if kind == "pose":
            draw_pose_record(out[f], pose_records[r])
            continue
        if kind == "68_landmarks":
            xy, ok = int_points(points[r])
        else:
            xy, ok = int_points(np.asarray(projected[r])[np.asarray(index)])
        draw_points(out[f], xy, ok)
    return out
