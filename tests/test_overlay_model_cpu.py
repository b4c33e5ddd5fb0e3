"""CPU: tests/overlay_model.py pinned to the cv2 binary (4.13.0) and to the reference's own demo_utils.py / calculate_rpy.

These are the rules csrc/overlay.cu restates; tests/test_overlay_gpu.py compares the kernels with this model."""
import math
import os
import random

import numpy as np
import pytest
import torch

from tests import overlay_model as M

cv2 = pytest.importorskip("cv2")

from oracle import ref_harness  # noqa: E402

needs_ref = pytest.mark.skipif(not ref_harness.available(), reason="reference tree not available")
RED = (255, 0, 0)


def _img(w, h):
    return np.zeros((h, w, 3), np.uint8)


def _paint(w, h, pixels):
    img = _img(w, h)
    for x, y in pixels:
        img[y, x] = RED
    return img


def test_cv2_version():
    assert cv2.__version__.startswith("4.13"), cv2.__version__


@pytest.mark.parametrize("r", range(1, 41))
def test_filled_circle_every_offset_near_edges_and_corners(r):
    W, H = 2 * r + 7, 2 * r + 5
    off = M.disk_offsets(r)
    for cx in range(-r - 2, W + r + 2):
        for cy in range(-r - 2, H + r + 2):
            a = _img(W, H)
            cv2.circle(a, (cx, cy), r, RED, -1)
            b = _img(W, H)
            M.draw_points(b, np.array([[cx, cy]]), color=RED) if M.point_radius(H, W) == r else M.fill_circle(b, cx, cy, r, RED)
            assert np.array_equal(a, b), (r, cx, cy)
    # the span recurrence and the offset table agree
    b1, b2 = _img(2 * r + 3, 2 * r + 3), _img(2 * r + 3, 2 * r + 3)
    M.fill_circle(b1, r + 1, r + 1, r, RED)
    b2[off[:, 1] + r + 1, off[:, 0] + r + 1] = RED
    assert np.array_equal(b1, b2)


def test_thin_lines_every_pair_in_a_window_across_the_border():
    W, H = 7, 5
    pts = [(x, y) for x in range(-6, 6) for y in range(-6, 6)]
    for p in pts:
        for q in pts:
            a = _img(W, H)
            cv2.line(a, p, q, RED, 1)
            assert np.array_equal(a, _paint(W, H, M.line_pixels(W, H, p, q))), (p, q)


def test_thin_lines_long_random():
    rng = random.Random(1)
    for _ in range(3000):
        W, H = rng.randint(1, 64), rng.randint(1, 64)
        R = 10 ** rng.randint(1, 6)
        p, q = [(rng.randint(-R, R), rng.randint(-R, R)) for _ in range(2)]
        a = _img(W, H)
        cv2.line(a, p, q, RED, 1)
        assert np.array_equal(a, _paint(W, H, M.line_pixels(W, H, p, q))), (W, H, p, q)


@pytest.mark.parametrize("t", range(2, 13))
def test_thick_lines_exhaustive_small(t):
    W, H = 6, 5
    pts = [(x, y) for x in range(-4, 5, 2) for y in range(-4, 5, 2)] + [(-t - 2, 3), (W + t, -1), (2, H + t + 1)]
    for p in pts:
        for q in pts:
            a = _img(W, H)
            cv2.line(a, p, q, RED, t)
            assert np.array_equal(a, _paint(W, H, M.segment_pixels(W, H, p, q, t))), (p, q, t)


def test_thick_lines_random():
    rng = random.Random(2)
    for _ in range(1500):
        W, H = rng.randint(1, 80), rng.randint(1, 80)
        R = rng.choice([20, 100, 1000])
        p, q = [(rng.randint(-R, R), rng.randint(-R, R)) for _ in range(2)]
        t = rng.randint(2, 12)
        a = _img(W, H)
        cv2.line(a, p, q, RED, t)
        assert np.array_equal(a, _paint(W, H, M.segment_pixels(W, H, p, q, t))), (W, H, p, q, t)


def test_zero_length_thick_line_is_the_cap_circle():
    for t in range(2, 13):
        a, b = _img(40, 40), _img(40, 40)
        cv2.line(a, (20, 20), (20, 20), RED, t)
        M.fill_circle(b, 20, 20, (t + 1) // 2, RED)
        assert np.array_equal(a, b), t


def test_arrowed_lines_random_and_small():
    rng = random.Random(3)
    cases = [((x0, y0), (x1, y1), t) for x0 in (-3, 2, 9) for y0 in (-2, 4) for x1 in (-5, 0, 6, 13) for y1 in (-4, 3, 11)
             for t in (1, 2, 3)]
    cases += [((rng.randint(-40, 120), rng.randint(-40, 120)), (rng.randint(-40, 120), rng.randint(-40, 120)),
               rng.randint(1, 8)) for _ in range(2000)]
    for p, q, t in cases:
        W, H = 64, 48
        a = _img(W, H)
        cv2.arrowedLine(a, p, q, (0, 0, 255), t)
        b = _img(W, H)
        M.arrowed_line(b, p, q, (0, 0, 255), t)
        assert np.array_equal(a, b), (p, q, t)


# ----------------------------------------------------------------------------------------------- against the reference
def _demo_utils():
    ref_harness.activate()
    import demo_utils
    return demo_utils


def _subset_indices(subset):
    ref_harness.activate()
    from model_training.utils import load_indices_from_npy
    d = os.path.join(ref_harness._active_root, "model_training/model/static/face_keypoints", f"keypoints_{subset}")
    out = []
    for f in os.listdir(d):
        out += list(load_indices_from_npy(os.path.join(d, f)))
    return out


@needs_ref
def test_subset_files_are_the_packed_sets():
    from dad_3dheads_b200.flame import load_flame_static
    st = load_flame_static()
    assert set(_subset_indices("191")) == set(st["keypoints_191"].tolist())
    assert set(_subset_indices("445")) == set(st["keypoints_565"].tolist())
    assert set(_subset_indices("445")) != set(st["keypoints_445"].tolist())


def _scene(seed, H=300, W=420, R=6):
    g = np.random.default_rng(seed)
    frame = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    boxes = []
    for r in range(R):
        h = int(g.integers(1, H + 1))
        w = int(g.integers(1, W + 1))
        boxes.append((int(g.integers(0, W - w + 1)), int(g.integers(0, H - h + 1)), w, h))
    points = g.integers(-20, max(H, W) + 20, (R, 68, 2)).astype(np.int64)
    proj = (g.random((R, 5023, 3)) * np.array([W + 40, H + 40, 1]) - 20).astype(np.float32)
    return frame, boxes, points, proj


@needs_ref
@pytest.mark.parametrize("seed", range(3))
def test_landmark_processors_equal_the_model(seed):
    du = _demo_utils()
    from dad_3dheads_b200.flame import load_flame_static
    st = load_flame_static()
    frame, boxes, points, proj = _scene(seed)
    R = len(boxes)
    crop = np.array(boxes)
    valid = np.ones(R, bool)
    valid[1] = False
    proj[2, 7] = np.nan
    for kind, idx in (("68_landmarks", None), ("191_landmarks", st["keypoints_191"]), ("445_landmarks", st["keypoints_565"])):
        want = frame.copy()
        for r in range(R):
            if not valid[r]:
                continue
            if kind == "68_landmarks":
                du.draw_landmarks({"points": points[r]}, want)
            else:
                p = torch.from_numpy(proj[r].copy())
                if r == 2:                                      # cv2 raises on a NaN point: drop that point alone
                    p = p.clone()
                    sub = kind.split("_")[0]
                    keep = [i for i in _subset_indices(sub) if i != 7]
                    pts = p.numpy().astype(int)[keep]
                    du.draw_points(want, pts)
                    continue
                du.draw_3d_landmarks({"projected_vertices": p}, want, kind.split("_")[0])
        got = M.overlay_frames(frame[None], kind, crop, np.zeros(R, int), valid, points=points, projected=proj,
                               index=idx)[0]
        assert np.array_equal(got, want), kind


def _rot_params(g, n):
    p = np.zeros((n, 413), np.float32)
    p[:, 403:409] = g.normal(size=(n, 6)).astype(np.float32)
    return p


@needs_ref
def test_rpy_model_matches_calculate_rpy():
    ref_harness.activate()
    from model_training.model.flame import FLAME_CONSTS, FlameParams, calculate_rpy
    from model_training.model.utils import rot_mat_from_6dof
    g = np.random.default_rng(5)
    params = _rot_params(g, 400)
    for p in params:
        t = torch.from_numpy(p[None].copy())
        fp = FlameParams.from_3dmm(t, FLAME_CONSTS)
        want = calculate_rpy(fp)
        got = M.rpy_from_rotation(p[403:409])
        if abs(want.yaw) < 89:                                           # the middle Euler angle away from gimbal lock
            assert np.allclose(got, (want.roll, want.pitch, want.yaw), atol=1e-9, rtol=0), (got, want)
        else:
            assert np.allclose(got, (want.roll, want.pitch, want.yaw), atol=1e-4, rtol=0), (got, want)
        rm = rot_mat_from_6dof(fp.rotation).numpy()[0]
        mm = M.rot_mat_from_6dof(p[403:409])
        assert np.array_equal(rm.view(np.int32), mm.view(np.int32))          # bit for bit


@needs_ref
@pytest.mark.parametrize("crop_h", [199, 200, 399, 400, 1080])
def test_draw_pose_equals_the_model(crop_h):
    du = _demo_utils()
    g = np.random.default_rng(crop_h)
    H, W = max(crop_h + 40, 300), 1300
    frame = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    R = 4
    boxes = [(int(g.integers(0, W - 300)), int(g.integers(0, H - crop_h + 1)), int(g.integers(150, 300)), crop_h)
             for _ in range(R)]
    boxes[1] = (boxes[0][0] + 30, boxes[0][1], boxes[0][2], crop_h)         # overlapping crops
    params = _rot_params(g, R)
    want = frame.copy()
    recs = []
    for r, (x, y, w, h) in enumerate(boxes):
        rpy = M.rpy_from_rotation(params[r, 403:409])
        assert M.near_boundaries(rpy, w, h) == 0
        recs.append(M.pose_record(rpy, boxes[r], 0, True))
        if int(h * 0.005) >= 1:
            du.draw_pose({"3dmm_params": torch.from_numpy(params[r:r + 1])}, want[y:y + h, x:x + w])
        else:
            with pytest.raises(cv2.error):
                du.draw_pose({"3dmm_params": torch.from_numpy(params[r:r + 1])}, want[y:y + h, x:x + w].copy())
    got = M.overlay_frames(frame[None], "pose", np.array(boxes), np.zeros(R, int), np.ones(R, bool),
                           pose_records=np.stack(recs))[0]
    assert np.array_equal(got, want)


# ----------------------------------------------------------------------------------------------- modelled errors
MUTATIONS = ["radius_plus_one", "line_tie_flipped", "arrow_order_reversed", "round_not_truncate", "no_crop_clip",
             "445_as_445_set"]


@needs_ref
@pytest.mark.parametrize("mutation", MUTATIONS)
def test_every_modelled_error_changes_a_compared_output(mutation, monkeypatch):
    """Each error, put into the model, changes a frame the GPU tests compare."""
    from dad_3dheads_b200.flame import load_flame_static
    st = load_flame_static()
    g = np.random.default_rng(11)
    H, W = 480, 640
    frame = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    boxes = np.array([(10, 10, 620, 460), (300, 50, 330, 300), (500, 100, 24, 260)])   # t 2, 1, and a narrow crop
    R = len(boxes)
    params = _rot_params(g, R)
    proj = (g.random((R, 5023, 2)) * [W, H]).astype(np.float32)
    points = g.integers(0, 480, (R, 68, 2))
    recs = np.stack([M.pose_record(M.rpy_from_rotation(params[r, 403:409]), boxes[r], 0, True) for r in range(R)])

    def run():
        return [M.overlay_frames(frame[None], k, boxes, np.zeros(R, int), np.ones(R, bool), points=points, projected=proj,
                                 index=st["keypoints_565"], pose_records=recs)[0] for k in ("68_landmarks", "445_landmarks",
                                                                                             "pose")]

    base = run()
    if mutation == "radius_plus_one":
        monkeypatch.setattr(M, "point_radius", lambda h, w: max(1, int(min(h, w) * 0.005)) + 1)
    elif mutation == "line_tie_flipped":
        orig = M.segment_pixels
        monkeypatch.setattr(M, "segment_pixels", lambda w, h, p, q, t: set(_line_tie_flipped(w, h, p, q)) if t <= 1 else
                            orig(w, h, p, q, t))
    elif mutation == "arrow_order_reversed":
        monkeypatch.setattr(M, "ARROW_COLORS", M.ARROW_COLORS[::-1])
    elif mutation == "round_not_truncate":
        recs2 = np.stack([_rounded_record(M.rpy_from_rotation(params[r, 403:409]), boxes[r]) for r in range(R)])
        recs[:] = recs2
    elif mutation == "no_crop_clip":
        orig_draw = M.draw_pose_record

        def unclipped(img, rec, key=None, box=0):
            rec = rec.copy()
            Hh, Ww = img.shape[:2]
            x, y = int(rec[2]), int(rec[3])
            rec[8:10] += (x, y)
            rec[10:28] += np.tile([x, y], 9)
            rec[2:6] = (0, 0, Ww, Hh)
            orig_draw(img, rec)
        monkeypatch.setattr(M, "draw_pose_record", unclipped)
    elif mutation == "445_as_445_set":
        st = dict(st)
        st["keypoints_565"] = st["keypoints_445"]
    mutated = run()
    assert any(not np.array_equal(a, b) for a, b in zip(base, mutated)), mutation


def _rounded_record(rpy, box):
    rec = M.pose_record(rpy, box, 0, True)
    g = M.pose_geometry(rpy, int(box[2]), int(box[3]))
    ends = [(int(round(g["values"][2 * k])), int(round(g["values"][2 * k + 1]))) for k in range(3)]
    for k, e in enumerate(ends):
        a, b, _ = M.arrow_tips(g["centre"], e)
        rec[10 + 6 * k: 16 + 6 * k] = [e[0], e[1], a[0], a[1], b[0], b[1]]
    return rec


def _line_tie_flipped(w, h, p, q):
    """line_pixels with the minor step taken on err <= 0 instead of err < 0."""
    ok, p, q = M.clip_line(w, h, p, q)
    if not ok:
        return []
    if q[0] < p[0]:
        p, q = q, p
    dx, dy, sy = q[0] - p[0], q[1] - p[1], 1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
    err, (x, y), out = dx - 2 * dy, p, []
    for _ in range(dx + 1):
        out.append((x, y))
        minor = err <= 0
        err += -2 * dy + (2 * dx if minor else 0)
        if vert:
            y += sy
            x += 1 if minor else 0
        else:
            x += 1
            y += sy if minor else 0
    return out


def test_polar_factor_is_scipys_svd_factor():
    """scipy's from_matrix replaces the fp32-built matrix by U Vt of its SVD; the model's (and the kernel's) Newton steps
    reach the same matrix to the fp64 rounding level, and the raw matrix is ~1e-7 away from it."""
    g = np.random.default_rng(8)
    far = []
    for _ in range(500):
        m = M.rot_mat_from_6dof(g.normal(size=6).astype(np.float32)).astype(np.float64).T
        u, _, vt = np.linalg.svd(m)
        assert np.abs(M.polar_factor(m) - u @ vt).max() < 1e-14
        far.append(np.abs(m - u @ vt).max())
    assert max(far) > 1e-8
