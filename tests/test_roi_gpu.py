"""-m gpu: heads from boxes in whole frames (csrc/roi.cu, predict_batch(frames, boxes=...)).

Every ROI's network input is bit-equal to the cv2 letter-box of its crop; the read-back kernel is bit-equal to the CPU model
(tests/roi_model.py, pinned against the reference in test_roi_model_cpu.py) between guard bands; end to end the result is
bit-equal to the composition through the existing code (crops -> predict_batch -> model read-back -> decode), and the graphed
and stream paths replay new boxes, frame indices and frames exactly."""
import os

import numpy as np
import pytest
import torch

from dad_3dheads_b200.encoder_weights import synthetic_state_dict
from tests import roi_model as M

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
S = 256
ROI_DTYPE = np.dtype([(k, "<i4") for k in ("x", "y", "w", "h", "frame", "valid", "new_h", "new_w", "pre_top", "pre_left",
                                           "post_top", "post_left")] + [(k, "<f8") for k in ("scale", "inv_scale_x",
                                                                                            "inv_scale_y")])
SENT_F32 = 0x7FC0BEEF          # NaN payload, as int32
SENT_I64 = 0x7FF8DEADBEEF0000
GUARD = 37


@pytest.fixture(scope="module")
def pred(cuda_device):
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


def _frames(F, H, W, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (F, H, W, 3), dtype=np.uint8))


def _ext4(extend):
    from dad_3dheads_b200.predictor import extend_sides
    return extend_sides(extend)


def _geos(boxes, frame_index, extend, F, H, W):
    out = []
    for r, b in enumerate(np.asarray(boxes).tolist()):
        f = 0 if frame_index is None else int(np.asarray(frame_index)[r])
        g = M.geometry(M.crop_box(b, _ext4(extend), H, W), frame_ok=0 <= f < F)
        g["frame"] = f
        out.append(g)
    return out


def _setup(pred, frames_d, boxes, frame_index, extend):
    """dad3d_roi_setup + dad3d_preprocess_rois on the device -> (records [R] ROI_DTYPE, inputs [R,3,S,S] between guards)."""
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.predictor import _MEAN, _STD
    lib = _lib.load()
    F, H, W = frames_d.shape[:3]
    boxes_d = torch.as_tensor(boxes).to(pred.device, torch.int32).contiguous()
    fi_d = None if frame_index is None else torch.as_tensor(frame_index).to(pred.device, torch.int32).contiguous()
    R = boxes_d.shape[0]
    rois = torch.empty(R, ROI_DTYPE.itemsize, dtype=torch.uint8, device=pred.device)
    n = R * 3 * S * S
    buf = torch.full((n + 2 * GUARD,), SENT_F32, dtype=torch.int32, device=pred.device)
    ext = np.array(_ext4(extend), dtype=np.float64)
    mean = (np.array(_MEAN, dtype=np.float32) * 255.0).astype(np.float32)
    inv = np.reciprocal(np.array(_STD, dtype=np.float32) * 255.0, dtype=np.float32)
    stream = torch.cuda.current_stream(pred.device).cuda_stream
    _lib.check(lib.dad3d_roi_setup(boxes_d.data_ptr(), fi_d.data_ptr() if fi_d is not None else None, R, F, H, W, S,
                                   ext.ctypes.data, rois.data_ptr(), stream), "setup")
    _lib.check(lib.dad3d_preprocess_rois(frames_d.data_ptr(), H, W, rois.data_ptr(), R, S, mean.ctypes.data,
                                         inv.ctypes.data, buf.data_ptr() + 4 * GUARD, stream), "preprocess")
    torch.cuda.synchronize()
    b = buf.cpu()
    assert (b[:GUARD] == SENT_F32).all() and (b[-GUARD:] == SENT_F32).all(), "store outside the output"
    return rois, np.frombuffer(rois.cpu().numpy().tobytes(), ROI_DTYPE), b[GUARD:-GUARD].view(torch.float32).view(R, 3, S, S)


def _check_records(rec, geos):
    for r, g in enumerate(geos):
        for k in ("x", "y", "w", "h", "new_h", "new_w", "pre_top", "pre_left", "post_top", "post_left", "scale"):
            assert rec[k][r] == g[k], (r, k, rec[k][r], g[k])
        assert bool(rec["valid"][r]) == g["valid"], r
        if g["valid"]:
            assert rec["inv_scale_x"][r] == 1.0 / (np.float64(g["new_w"]) / g["w"])
            assert rec["inv_scale_y"][r] == 1.0 / (np.float64(g["new_h"]) / g["h"])


# boxes on three 480 x 640 frames: every edge, clipped and shifted boxes, S x S (no resize), up- and down-scaling
EDGE_BOXES = [[0, 0, 100, 80], [540, 0, 100, 80], [0, 400, 100, 80], [540, 400, 100, 80],     # corners, touching edges
              [-40, 100, 100, 80], [100, -30, 80, 100], [600, 300, 100, 90], [300, 420, 90, 100],  # shifted / cut
              [50, 60, 256, 256], [200, 100, 256, 120], [10, 10, 37, 23], [20, 30, 7, 5],          # S x S, up-scaling
              [0, 0, 640, 480], [5, 3, 611, 455], [123, 45, 1, 9], [77, 88, 13, 1],                # down-scaling, 1-px sides
              [700, 10, 30, 30], [0, 0, 640, 1]]                                                   # outside; 0-px side


@pytest.mark.parametrize("extend", [0.0, 0.1, (0.05, 0.3, -0.1, 0.2)])
def test_preprocess_rois_bit_exact(pred, extend):
    from dad_3dheads_b200.predictor import letterbox_normalise
    F, H, W = 3, 480, 640
    frames = _frames(F, H, W, 1)
    boxes = np.array(EDGE_BOXES, dtype=np.int64)
    fi = np.arange(len(boxes)) % F
    geos = _geos(boxes, fi, extend, F, H, W)
    _, rec, x = _setup(pred, frames.to(pred.device), boxes, fi, extend)
    _check_records(rec, geos)
    assert sum(g["valid"] for g in geos) >= len(boxes) - 3
    fr = frames.numpy()
    for r, g in enumerate(geos):
        got = x[r].numpy()
        assert np.array_equal(got, np.transpose(M.letterbox(fr[fi[r]], g), (2, 0, 1))), (r, g)
        if g["valid"]:
            crop = fr[fi[r], g["y"]:g["y"] + g["h"], g["x"]:g["x"] + g["w"]]
            assert np.array_equal(got, np.transpose(letterbox_normalise(crop, S), (2, 0, 1))), (r, g)
    assert not geos[-1]["valid"] and not geos[-2]["valid"]


def test_preprocess_rois_full_hd_frames(pred):
    """Four 1920 x 1080 frames, boxes on all of them: the frame pitch and the frame offset are 64-bit."""
    F, H, W = 4, 1080, 1920
    frames = _frames(F, H, W, 2)
    g = np.random.default_rng(3)
    boxes = np.stack([g.integers(-100, W, 24), g.integers(-100, H, 24), g.integers(20, 900, 24), g.integers(20, 900, 24)], 1)
    fi = g.integers(0, F, 24)
    geos = _geos(boxes, fi, 0.1, F, H, W)
    _, rec, x = _setup(pred, frames.to(pred.device), boxes, fi, 0.1)
    _check_records(rec, geos)
    fr = frames.numpy()
    for r, geo in enumerate(geos):
        assert np.array_equal(x[r].numpy(), np.transpose(M.letterbox(fr[fi[r]], geo), (2, 0, 1))), r


def test_invalid_frame_index_on_device(pred):
    frames = _frames(2, 100, 120, 4)
    boxes = np.array([[10, 10, 50, 50]] * 4)
    fi = np.array([0, 2, -1, 1])
    _, rec, x = _setup(pred, frames.to(pred.device), boxes, fi, 0.0)
    assert rec["valid"].tolist() == [1, 0, 0, 1]
    pad = np.transpose(M.letterbox(frames.numpy()[0], M.geometry((0, 0, 0, 0))), (2, 0, 1))
    assert np.array_equal(x[1].numpy(), pad) and np.array_equal(x[2].numpy(), pad)
    assert rec["scale"][1] == 1.0 and rec["post_top"][1] == 0 and rec["new_h"][1] == 0


def test_readjust_bit_exact_with_guard_bands(pred):
    from dad_3dheads_b200 import _lib
    lib = _lib.load()
    F, H, W = 2, 700, 900
    g = np.random.default_rng(5)
    R = 300
    boxes = np.stack([g.integers(-50, W, R), g.integers(-50, H, R), g.integers(1, 700, R), g.integers(1, 700, R)], 1)
    fi = g.integers(0, F + 1, R)                                             # some out of range: invalid rows
    frames_d = _frames(F, H, W, 6).to(pred.device)
    rois, rec, _ = _setup(pred, frames_d, boxes, fi, (0.1, 0.2))
    geos = _geos(boxes, fi, (0.1, 0.2), F, H, W)
    _check_records(rec, geos)
    params = (g.standard_normal((R, 413)) * g.choice([0.01, 1.0, 30.0], (R, 413))).astype(np.float32)
    lms = g.uniform(-0.3, 1.3, (R, 68, 2)).astype(np.float32)
    p_d, l_d = torch.from_numpy(params).to(pred.device), torch.from_numpy(lms).to(pred.device)
    pbuf = torch.full((R * 413 + 2 * GUARD,), SENT_F32, dtype=torch.int32, device=pred.device)
    qbuf = torch.full((R * 136 + 2 * GUARD,), SENT_I64, dtype=torch.int64, device=pred.device)
    stream = torch.cuda.current_stream(pred.device).cuda_stream
    _lib.check(lib.dad3d_readjust_rois(p_d.data_ptr(), l_d.data_ptr(), rois.data_ptr(), R, 413, 68, M.SCALE_IDX,
                                       M.TRANSLATION_IDX, S, pbuf.data_ptr() + 4 * GUARD, qbuf.data_ptr() + 8 * GUARD,
                                       stream), "readjust")
    pb, qb = pbuf.cpu(), qbuf.cpu()
    for b, sent in ((pb, SENT_F32), (qb, SENT_I64)):
        assert (b[:GUARD] == sent).all() and (b[-GUARD:] == sent).all(), "store outside the output"
    got_p = pb[GUARD:-GUARD].view(R, 413).numpy()
    got_q = qb[GUARD:-GUARD].view(R, 68, 2).numpy()
    for r, geo in enumerate(geos):
        assert np.array_equal(got_p[r], M.readjust_params(params[r], geo).view(np.int32)), r
        assert np.array_equal(got_q[r], M.readjust_points(lms[r], geo)), r


def _composition(pred, frames, boxes, fi, extend, fast_decode):
    """The same heads through the existing code: crops on the host -> predict_batch(list of crops) at the same R -> the CPU
    model of the read-back -> head_mesh.decode."""
    F, H, W = frames.shape[:3]
    geos = _geos(boxes, fi, extend, F, H, W)
    fr = frames.numpy()
    crops = [fr[f, g["y"]:g["y"] + g["h"], g["x"]:g["x"] + g["w"]] for f, g in zip(fi, geos)]
    base = pred.predict_batch(crops, landmark_subset=None, fast_decode=fast_decode)
    raw = base["3dmm_params"].cpu().numpy()
    lms = (base["points"].cpu() / 256.0).numpy()                      # points = lms * 256: exact
    params = np.stack([M.readjust_params(raw[r], g) for r, g in enumerate(geos)])
    points = np.stack([M.readjust_points(lms[r], g) for r, g in enumerate(geos)])
    p_d = torch.from_numpy(params).to(pred.device)
    v3, proj = pred.head_mesh.decode(p_d, to_2d=True, hilo=not fast_decode)
    lm445 = proj[:, pred._landmark_index("445")]
    return {"3dmm_params": p_d, "points": torch.from_numpy(points), "3d_vertices": v3, "projected_vertices": proj,
            "landmarks_445": lm445}, geos


def _valid_boxes(F, H, W, R, seed):
    g = np.random.default_rng(seed)
    boxes = np.stack([g.integers(-60, W - 80, R), g.integers(-60, H - 80, R), g.integers(40, 500, R),
                      g.integers(40, 500, R)], 1)
    return boxes, g.integers(0, F, R)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm()).item()


def test_end_to_end_equals_composition(pred):
    F, H, W, R = 3, 600, 800, 9
    frames = _frames(F, H, W, 7)
    boxes, fi = _valid_boxes(F, H, W, R, 8)
    want, geos = _composition(pred, frames, boxes, fi, (0.1, 0.15), fast_decode=False)
    got = pred.predict_batch(frames, boxes=torch.from_numpy(boxes), frame_index=torch.from_numpy(fi), extend=(0.1, 0.15),
                             fast_decode=False)
    assert got["points"].dtype == torch.int64 and got["crop_boxes"].dtype == torch.int32 and got["valid"].dtype == torch.bool
    assert got["valid"].all()
    assert got["crop_boxes"].cpu().tolist() == [[g["x"], g["y"], g["w"], g["h"]] for g in geos]
    for k in ("3dmm_params", "points", "3d_vertices", "projected_vertices", "landmarks_445"):
        assert torch.equal(got[k].cpu(), want[k].cpu()), k
    assert (got["3dmm_params"][:, M.TRANSLATION_IDX + 2] == 0).all()
    fast = pred.predict_batch(frames, boxes=boxes, frame_index=fi, extend=(0.1, 0.15))       # default fast decode
    assert torch.equal(fast["3dmm_params"], got["3dmm_params"]) and torch.equal(fast["points"], got["points"])
    for k in ("3d_vertices", "projected_vertices"):
        assert _rel(fast[k], want[k]) < 5e-5, k


def test_against_live_reference_on_pasted_demo_head(pred):
    """The demo head (954 x 766) pasted at an offset into a larger frame, its box extended by 10 %: within the tolerances of
    test_single_image_call_matches_reference_semantics of the reference's own crop + __call__ + move into the frame."""
    import cv2
    from oracle import ref_harness as R
    if not R.available():
        pytest.skip("reference not available")
    img = cv2.cvtColor(cv2.imread(os.path.join(GOLDEN, "demo_head_1.jpeg")), cv2.COLOR_BGR2RGB)
    frame = np.random.default_rng(9).integers(0, 256, (1300, 1500, 3), dtype=np.uint8)
    oy, ox = 211, 377
    frame[oy:oy + img.shape[0], ox:ox + img.shape[1]] = img
    box = [ox + 60, oy + 90, 640, 820]
    ref = R.predictor(synthetic_state_dict(0))
    from model_training.data.utils import ensure_bbox_boundaries, extend_bbox
    x, y, w, h = (int(v) for v in ensure_bbox_boundaries(extend_bbox(np.array(box), 0.1), frame.shape[:2]))
    want = ref(frame[y:y + h, x:x + w])
    want_p = want["3dmm_params"].clone()
    want_p[:, M.TRANSLATION_IDX:M.TRANSLATION_IDX + 2] += torch.tensor([[x, y]], dtype=torch.float32) * 2 / 256
    want_proj = want["projected_vertices"].double() + torch.tensor([x, y], dtype=torch.float64)
    want_pts = want["points"] + np.array([x, y])
    got = pred.predict_batch(torch.from_numpy(frame[None]), boxes=torch.tensor([box]), extend=0.1)
    assert got["crop_boxes"].cpu().tolist() == [[x, y, w, h]]
    assert _rel(got["3dmm_params"], want_p) < 5e-5
    assert (got["projected_vertices"].cpu().double() - want_proj).abs().max() < 0.25
    assert np.abs(got["points"][0].cpu().numpy() - want_pts).max() <= 1


def test_invalid_rois_do_not_disturb_neighbours(pred):
    F, H, W = 2, 400, 700
    frames = _frames(F, H, W, 10)
    boxes, fi = _valid_boxes(F, H, W, 8, 11)
    bad = boxes.copy()
    bad_fi = fi.copy()
    bad[1] = [750, 10, 30, 30]                 # outside: empty crop
    bad[4] = [0, 0, 700, 1]                    # 700 x 1 -> a 0-pixel side
    bad_fi[6] = 2                              # frame out of range (device frame index)
    good = pred.predict_batch(frames, boxes=boxes, frame_index=fi)
    good = {k: v.clone() for k, v in good.items()}
    got = pred.predict_batch(frames.to(pred.device), boxes=torch.from_numpy(bad).to(pred.device),
                             frame_index=torch.from_numpy(bad_fi).to(pred.device))
    assert got["valid"].cpu().tolist() == [True, False, True, True, False, True, False, True]
    keep = [0, 2, 3, 5, 7]
    for k, v in got.items():
        if v.is_floating_point():
            assert torch.isfinite(v).all(), k
        if k != "valid":
            assert torch.equal(v[keep], good[k][keep]), k


def test_sub_batch_reproduces_rows(pred):
    F, H, W = 3, 500, 700
    frames = _frames(F, H, W, 12)
    boxes, fi = _valid_boxes(F, H, W, 16, 13)
    full = {k: v.clone() for k, v in pred.predict_batch(frames, boxes=boxes, frame_index=fi).items()}
    sub = pred.predict_batch(frames, boxes=boxes[5:11], frame_index=fi[5:11])
    for k in full:
        assert torch.equal(full[k][5:11], sub[k]), k


def test_device_boxes_need_no_host_synchronisation(pred):
    F, H, W = 2, 480, 640
    frames = _frames(F, H, W, 14).to(pred.device)
    boxes, fi = _valid_boxes(F, H, W, 6, 15)
    boxes_d = torch.from_numpy(boxes).to(pred.device)
    fi_d = torch.from_numpy(fi).to(pred.device)
    want = {k: v.clone() for k, v in pred.predict_batch(frames, boxes=boxes_d, frame_index=fi_d).items()}   # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = pred.predict_batch(frames, boxes=boxes_d, frame_index=fi_d)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in want:
        assert torch.equal(got[k], want[k]), k


def _steps(F, H, W, R):
    """Three consecutive steps whose frames, boxes and frame indices all change."""
    out = []
    for i in range(3):
        boxes, fi = _valid_boxes(F, H, W, R, 20 + i)
        if i == 1:
            boxes[2] = [900, 900, 10, 10]          # an invalid ROI in the middle step
        out.append((_frames(F, H, W, 30 + i), torch.from_numpy(boxes), torch.from_numpy(fi)))
    return out


def test_graphed_equals_eager(pred):
    F, H, W, R = 3, 360, 480, 5
    steps = _steps(F, H, W, R)
    want = [{k: v.clone() for k, v in pred.predict_batch(fr, boxes=b, frame_index=f, extend=0.1).items()}
            for fr, b, f in steps]
    for (fr, b, f), w in zip(steps, want):
        got = pred.predict_batch_graphed(fr, boxes=b, frame_index=f, extend=0.1)
        torch.cuda.synchronize()
        for k in w:
            assert torch.equal(got[k], w[k]), k
    assert not want[1]["valid"][2] and want[0]["valid"].all()


def test_stream_equals_eager(pred):
    F, H, W, R = 3, 360, 480, 5
    steps = _steps(F, H, W, R)
    want = [{k: v.clone().cpu() for k, v in pred.predict_batch(fr, boxes=b, frame_index=f, extend=0.1).items()}
            for fr, b, f in steps]
    keys = ("3dmm_params", "points", "projected_vertices", "landmarks_445", "crop_boxes", "valid")
    st = pred.open_stream((F, H, W, 3), rois=R, extend=0.1, keys=keys, depth=2)
    got = []
    for fr, b, f in steps:
        if st._inflight == st.depth:
            got.append({k: v.clone() for k, v in st.collect().items()})
        st.submit(fr.pin_memory(), boxes=b, frame_index=f)
    while st._inflight:
        got.append({k: v.clone() for k, v in st.collect().items()})
    assert len(got) == 3
    for i in range(3):
        for k in keys:
            assert torch.equal(got[i][k], want[i][k]), (i, k)


def test_invalid_arguments_raise_before_any_launch(pred):
    from dad_3dheads_b200 import _lib
    frames = _frames(2, 64, 80, 16)
    boxes = torch.tensor([[1, 2, 30, 40], [5, 6, 20, 10]])
    before = _lib.launch_count()
    bad = [dict(boxes=boxes.float()), dict(boxes=boxes[0]), dict(boxes=boxes[:, :3]),
           dict(boxes=boxes, frame_index=torch.tensor([0, 2])), dict(boxes=boxes, frame_index=torch.tensor([-1, 0])),
           dict(boxes=boxes, frame_index=torch.tensor([0])), dict(boxes=boxes, frame_index=torch.tensor([0.0, 1.0])),
           dict(boxes=torch.zeros(65536, 4, dtype=torch.int32)), dict(boxes=boxes, extend=(0.1, 0.2, 0.3)),
           dict(boxes=boxes, to_2d=False, render="pncc")]
    for kw in bad:
        with pytest.raises(ValueError):
            pred.predict_batch(frames, **kw)
    for f in (frames.float(), frames[0], frames[..., :2]):
        with pytest.raises(ValueError):
            pred.predict_batch(f, boxes=boxes)
    with pytest.raises(ValueError):
        pred.predict_batch_graphed(frames, boxes=boxes, to_2d=False, render="depth")
    with pytest.raises(ValueError):
        pred.predict_batch_graphed(frames, boxes=boxes, frame_index=torch.tensor([0, 5]))
    assert _lib.launch_count() == before
    empty = pred.predict_batch(frames, boxes=torch.zeros(0, 4, dtype=torch.int64))
    assert empty["3dmm_params"].shape == (0, 413) and empty["points"].shape == (0, 68, 2)
    assert empty["valid"].shape == (0,) and empty["crop_boxes"].shape == (0, 4)


def test_submission_with_boxes_is_in_frame_pixels(pred):
    from dad_3dheads_b200.submission import SubmissionWriter
    from oracle.flame_oracle import load_static
    from oracle.predictor_oracle import PredictorOracle
    from tests.test_submission_gpu import _oracle_68
    st = load_static()
    F, H, W = 3, 500, 700
    frames = _frames(F, H, W, 17)
    boxes = np.array([[100, 50, 300, 360], [-20, 200, 250, 200], [450, 100, 300, 330]])
    sub = SubmissionWriter(pred).predict(frames, ["a", "b", "c"], boxes=torch.from_numpy(boxes), extend=0.05)
    orc = PredictorOracle(synthetic_state_dict(0), dtype=torch.float64)
    fr = frames.numpy()
    for i, (key, geo) in enumerate(zip("abc", _geos(boxes, np.arange(F), 0.05, F, H, W))):
        want = orc(fr[i, geo["y"]:geo["y"] + geo["h"], geo["x"]:geo["x"] + geo["w"]])
        proj = want["projected_vertices"][0].double() + torch.tensor([geo["x"], geo["y"]], dtype=torch.float64)
        lm2 = _oracle_68(proj, st)
        got2 = torch.tensor(sub[key]["68_landmarks_2d"], dtype=torch.float64)
        assert got2.shape == (68, 2) and (got2 - lm2).abs().max() < 0.1, (key, (got2 - lm2).abs().max())
