"""Heads from boxes, CPU: the numpy model of the crop geometry and of the read-back (tests/roi_model.py) equals the reference's
own extend_bbox, ensure_bbox_boundaries, _get_paddings, readjust_landmarks_to_the_input_image,
readjust_3dmm_to_the_input_image and HeadMesh.adjust_3dmm_to_paddings bit for bit, and the model's letter-box of a crop equals
the cv2 pipeline on the same crop."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ref_harness as R
from tests import roi_model as M

# (box [x, y, w, h], extend as extend_bbox takes it, frame (H, W)) -- designed cases
CASES = [
    ([100, 50, 80, 120], 0.0, (480, 640)),                         # inside, no extend
    ([100, 50, 80, 120], 0.1, (480, 640)),
    ([100, 50, 81, 121], (0.15, 0.35), (480, 640)),                 # fractional extends, truncation toward zero
    ([100, 50, 81, 121], (0.05, 0.2, 0.3, 0.11), (480, 640)),
    ([100, 50, 81, 121], (-0.2, -0.1, -0.05, -0.3), (480, 640)),    # negative extends
    ([10, 7, 33, 29], (0.4, 0.0, 0.45, 0.0), (480, 640)),           # extended past the left / top edge: shifted, not cut
    ([-30, -20, 90, 70], 0.0, (480, 640)),                          # starts left of / above the frame
    ([600, 450, 90, 70], 0.2, (480, 640)),                          # past the right / bottom edge: cut
    ([700, 10, 50, 50], 0.0, (480, 640)),                           # fully outside: empty crop
    ([10, 500, 50, 50], 0.0, (480, 640)),
    ([-100, 10, 50, 50], 0.0, (480, 640)),                          # left of the frame: shifted into it
    ([0, 0, 640, 480], 0.0, (480, 640)),                            # the whole frame
    ([5, 5, 512, 3], 0.0, (600, 600)),                              # py3round exact half: 3 * 0.5 = 1.5 -> 2
    ([5, 5, 512, 5], 0.0, (600, 600)),                              # 2.5 -> 2
    ([5, 5, 1024, 2], 0.0, (600, 1100)),                            # 0.5 -> 0: invalid (cv2 refuses a 0-pixel side)
    ([5, 5, 256, 256], 0.0, (600, 600)),                            # scale exactly 1
    ([5, 5, 256, 100], 0.0, (600, 600)),                            # scale 1 with padding
    ([3, 4, 1, 7], 0.0, (50, 50)),                                  # one-pixel sides
    ([3, 4, 9, 1], 0.0, (50, 50)),
    ([3, 4, 1, 1], 0.0, (50, 50)),
    ([0, 0, 1000, 1], 0.0, (20, 1000)),                             # 1 x 1000 -> 0.256 -> 0: invalid
    ([11, 3, 333, 517], 0.07, (700, 900)),
]


def _ext4(extend):
    from dad_3dheads_b200.predictor import extend_sides
    return extend_sides(extend)


@pytest.fixture(scope="module")
def ref():
    if not R.available():
        pytest.skip("reference not available")
    R.activate()
    import predictor as ref_predictor
    from model_training.data.utils import ensure_bbox_boundaries, extend_bbox
    return SimpleNamespace(extend_bbox=extend_bbox, ensure=ensure_bbox_boundaries, P=ref_predictor.FaceMeshPredictor)


def _stub(ref):
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG
    return SimpleNamespace(_img_size=256, flame_constants=dict(DEFAULT_CONFIG["constants"]),
                           find_3dmm_idx=ref.P.find_3dmm_idx)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_crop_and_paddings_match_reference(ref, case):
    box, extend, (H, W) = CASES[case]
    want = ref.ensure(ref.extend_bbox(np.array(box), extend), (H, W))
    got = M.crop_box(box, _ext4(extend), H, W)
    assert tuple(int(v) for v in want) == got
    g = M.geometry(got)
    x, y, w, h = got
    if w <= 0 or h <= 0:
        assert not g["valid"]
        return
    import cv2
    pads, scale = ref.P._get_paddings(_stub(ref), {"input_shape": (h, w)})
    nh, nw = round(h * scale), round(w * scale)
    if nh == 0 or nw == 0:                                    # the reference cannot process such a crop either
        with pytest.raises(cv2.error):
            cv2.resize(np.zeros((h, w, 3), np.uint8), dsize=(nw, nh), interpolation=cv2.INTER_LINEAR)
        assert not g["valid"]
        return
    assert g["valid"] and g["scale"] == scale and (g["new_h"], g["new_w"]) == (nh, nw)
    assert (g["post_top"], g["post_left"]) == (pads[0], pads[2])


def test_extend_quirk_shifts_boxes_left_of_the_frame(ref):
    """ensure_bbox_boundaries computes x2 from the clipped x1 plus the original w: the box moves right, keeping its width."""
    assert M.crop_box([-100, 10, 50, 50], (0, 0, 0, 0), 480, 640) == (0, 10, 50, 50)
    assert M.crop_box([10, -7, 50, 50], (0, 0, 0, 0), 480, 640) == (10, 0, 50, 50)


def _readjust_cases():
    g = np.random.default_rng(0)
    out = []
    for case in range(len(CASES)):
        box, extend, (H, W) = CASES[case]
        geo = M.geometry(M.crop_box(box, _ext4(extend), H, W))
        if geo["valid"]:
            out.append(geo)
    for _ in range(40):                                       # random crops
        H, W = int(g.integers(64, 1500)), int(g.integers(64, 2000))
        box = [int(g.integers(-50, W)), int(g.integers(-50, H)), int(g.integers(1, 700)), int(g.integers(1, 700))]
        geo = M.geometry(M.crop_box(box, _ext4(tuple(g.uniform(-0.1, 0.4, 4))), H, W))
        if geo["valid"]:
            out.append(geo)
    return out


def test_readjust_matches_reference(ref):
    """Params: readjust_3dmm_to_the_input_image, translation z zeroed, then adjust_3dmm_to_paddings' translation arithmetic
    with paddings [y, 0, x, 0].  Points: readjust_landmarks_to_the_input_image on clip(lm * 256, 0, 256), then + [x, y].
    Landmarks below 0 and above 256, and parameters over a wide range."""
    R.activate()
    from model_training.head_mesh import HeadMesh
    stub = _stub(ref)
    hm = HeadMesh(image_size=256)
    g = np.random.default_rng(1)
    geos = _readjust_cases()
    assert len(geos) > 30
    for geo in geos:
        p = (g.standard_normal(413) * g.choice([0.01, 1.0, 30.0], 413)).astype(np.float32)
        lms = g.uniform(-0.3, 1.3, (68, 2)).astype(np.float32)
        lms[:4] = [[0.0, 1.0], [1.0, 0.0], [-0.0, 0.5], [0.99999994, 0.5]]
        pads = [geo["post_top"], 0, geo["post_left"], 0]
        # reference, steps 2 and 3
        want_p = ref.P.readjust_3dmm_to_the_input_image(stub, torch.from_numpy(p.copy())[None], pads, geo["scale"])
        want_p[:, M.TRANSLATION_IDX + 2] = 0.0                                    # reprojected_vertices' side effect
        moved = hm.adjust_3dmm_to_paddings(want_p.clone(), [geo["y"], 0, geo["x"], 0])
        want_p[:, M.TRANSLATION_IDX:M.TRANSLATION_IDX + 3] = moved[:, M.TRANSLATION_IDX:M.TRANSLATION_IDX + 3]
        lm = (lms * 256.0).clip(min=0, max=256)
        want_pts = ref.P.readjust_landmarks_to_the_input_image(None, lm, pads, geo["scale"]) + np.array([geo["x"], geo["y"]])
        got_p = M.readjust_params(p, geo)
        got_pts = M.readjust_points(lms, geo)
        assert np.array_equal(got_p.view(np.int32), want_p[0].numpy().view(np.int32)), geo
        assert got_pts.dtype == np.int64 and np.array_equal(got_pts, want_pts), geo


def test_fp64_division_would_differ(ref):
    """The model divides in fp32 by the fp32-rounded scale; an fp64 division differs on some of these cases, so the test
    above pins the dtype sequence rather than passing by accident."""
    g = np.random.default_rng(2)
    diff = 0
    for geo in _readjust_cases():
        t = g.standard_normal(64).astype(np.float32)
        f32 = (t + np.float32(1)) / np.float32(geo["scale"])
        f64 = ((t.astype(np.float64) + 1.0) / geo["scale"]).astype(np.float32)
        diff += int((f32 != f64).sum())
    assert diff > 0


@pytest.mark.parametrize("case", range(len(CASES)))
def test_crop_letterbox_matches_cv2(case):
    """The model's letter-box of a crop (numpy restatement of cv2's resize, read from the frame) equals the cv2 pipeline
    (letterbox_normalise) on frame[y:y+h, x:x+w]; invalid crops give the all-padding image."""
    from dad_3dheads_b200.predictor import letterbox_normalise
    box, extend, (H, W) = CASES[case]
    frame = np.random.default_rng(case).integers(0, 256, (H, W, 3), dtype=np.uint8)
    geo = M.geometry(M.crop_box(box, _ext4(extend), H, W))
    got = M.letterbox(frame, geo)
    if geo["valid"]:
        want = letterbox_normalise(frame[geo["y"]:geo["y"] + geo["h"], geo["x"]:geo["x"] + geo["w"]], 256)
    else:
        want = letterbox_normalise(np.zeros((256, 256, 3), np.uint8), 256)
    assert np.array_equal(got, want)
