"""-m gpu: the demo's landmark and pose overlays and per-head rpy (csrc/overlay.cu, predict_batch(overlay=, rpy=)).

Every frame of every kind is compared byte for byte with tests/overlay_model.py (pinned to cv2 and to the unmodified
demo_utils.py by tests/test_overlay_model_cpu.py), evaluated on this call's own device outputs."""
import os

import numpy as np
import pytest
import torch

from tests import overlay_model as M
from tests.test_demo_unchanged_gpu import _run_demo, demo_home  # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
KINDS = M.OVERLAY_KINDS
RI = 403                                                   # FlameParams.from_3dmm's rotation slice, released layout


def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def pred():
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


def _frames(F, H, W, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (F, H, W, 3), dtype=np.uint8))


def _scene(F, H, W, seed):
    """Boxes overlapping, at and past the frame border, pose crops of 199 / 200 / 400 px and the whole frame, and two
    invalid boxes (frame index out of range, empty crop)."""
    g = np.random.default_rng(seed)
    boxes, fidx = [], []
    for h in (199, 200, 400, min(H, 1080)):
        if h <= H:
            boxes.append((int(g.integers(0, max(1, W - 300))), int(g.integers(0, H - h + 1)), min(W, 300), h))
            fidx.append(int(g.integers(0, F)))
    boxes.append((0, 0, W, H)); fidx.append(0)
    boxes.append((boxes[0][0] + 40, boxes[0][1] + 10, 300, 220)); fidx.append(fidx[0])          # overlaps box 0
    boxes.append((W - 50, H - 60, 200, 200)); fidx.append(F - 1)                                # past the corner
    boxes.append((-30, -40, 120, 150)); fidx.append(0)                                          # past the origin
    boxes.append((10, 10, 100, 100)); fidx.append(F)                                            # invalid frame
    boxes.append((W, 5, 40, 40)); fidx.append(0)                                                # empty crop
    for _ in range(6):
        w, h = int(g.integers(20, W)), int(g.integers(20, H))
        boxes.append((int(g.integers(-w // 2, W)), int(g.integers(-h // 2, H)), w, h)); fidx.append(int(g.integers(0, F)))
    # on the device: a host frame index out of range is refused before launch, a device one makes the box invalid
    return torch.tensor(boxes, dtype=torch.int32), torch.tensor(fidx, dtype=torch.int32).to(_dev())


def _model_frames(frames, out, kinds, static):
    crop = out["crop_boxes"].cpu().numpy()
    valid = out["valid"].cpu().numpy()
    fidx = out["_frame_index"]
    rpy = out["rpy"].cpu().numpy()
    recs = np.stack([M.pose_record(rpy[r], crop[r], int(fidx[r]), bool(valid[r])) for r in range(len(crop))])
    res = {}
    for k in kinds:
        idx = {"191_landmarks": static["keypoints_191"], "445_landmarks": static["keypoints_565"]}.get(k)
        res[k] = M.overlay_frames(frames, k, crop, fidx, valid, points=out["points"].cpu().numpy(),
                                  projected=out["projected_vertices"].cpu().numpy(), index=idx, pose_records=recs)
    near = sum(M.near_boundaries(rpy[r], int(crop[r, 2]), int(crop[r, 3])) for r in range(len(crop)) if valid[r])
    return res, near


@pytest.mark.parametrize("F,H,W,to_2d", [(3, 333, 517, True), (2, 1080, 1920, False), (1, 201, 199, True)])
def test_frames_equal_the_model(pred, flame_static, F, H, W, to_2d):
    frames = _frames(F, H, W, H)
    keep = frames.clone()
    boxes, fidx = _scene(F, H, W, W)
    dev_frames = frames.to(_dev())
    out = pred.predict_batch(dev_frames, boxes=boxes, frame_index=fidx, to_2d=to_2d, overlay=KINDS, rpy=True)
    torch.cuda.synchronize()
    assert torch.equal(dev_frames.cpu(), keep)                              # the input frames are never written
    out["_frame_index"] = fidx.cpu().numpy()
    want, near = _model_frames(frames.numpy(), out, KINDS, flame_static)
    assert near == 0
    ref = _reference_frames(frames.numpy(), out)
    for k in KINDS:
        got = out[f"frame_{k}"].cpu().numpy()
        assert got.shape == (F, H, W, 3) and got.dtype == np.uint8
        bad = np.argwhere((got != want[k]).any(-1))
        assert len(bad) == 0, (k, len(bad), bad[:5].tolist())
        assert not np.array_equal(got, frames.numpy()), k                  # something was drawn
        if ref is not None:
            bad = np.argwhere((got != ref[k]).any(-1))
            assert len(bad) == 0, ("demo_utils", k, len(bad), bad[:5].tolist())


def _reference_frames(frames, out):
    """The contract itself: demo_utils.py's own processors applied per valid box, in box order, to copies of the frames,
    with this call's predictions (the pose into the crop view; crops under 200 px are skipped, where cv2 refuses)."""
    from oracle import ref_harness as RH
    if not RH.available():
        return None
    RH.activate()
    import demo_utils
    crop, valid, fidx = out["crop_boxes"].cpu().numpy(), out["valid"].cpu().numpy(), out["_frame_index"]
    points, proj, params = out["points"].cpu().numpy(), out["projected_vertices"].cpu(), out["3dmm_params"].cpu()
    res = {k: frames.copy() for k in KINDS}
    for r in range(len(crop)):
        if not valid[r]:
            continue
        f = int(fidx[r])
        x, y, w, h = (int(v) for v in crop[r])
        demo_utils.draw_landmarks({"points": points[r]}, res["68_landmarks"][f])
        demo_utils.draw_3d_landmarks({"projected_vertices": proj[r]}, res["191_landmarks"][f], "191")
        demo_utils.draw_3d_landmarks({"projected_vertices": proj[r]}, res["445_landmarks"][f], "445")
        if int(h * 0.005) >= 1:
            demo_utils.draw_pose({"3dmm_params": params[r:r + 1]}, res["pose"][f][y:y + h, x:x + w])
    return res


def test_non_finite_and_far_heads_in_whole_frames(pred, flame_static):
    """Heads whose vertices are NaN, infinite or beyond int32 after truncation, drawn with the others into whole frames
    through the overlay functions: exactly the points cv2 accepts are drawn."""
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200 import overlay as O
    F, H, W = 2, 480, 640
    frames = _frames(F, H, W, 12)
    boxes, fidx = _scene(F, H, W, 13)
    out = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, to_2d=False)
    proj = out["projected_vertices"].clone()
    proj[0] = float("nan")                                                 # a whole head
    proj[1, ::7, 0] = float("inf")
    proj[1, ::11, 1] = -float("inf")
    proj[2, ::5, 0] = 3e9
    proj[2, ::3, 1] = -2147483904.0
    proj[3, ::2] = float("nan")
    R = int(boxes.shape[0])
    rois = torch.empty(R, 72, dtype=torch.uint8, device=_dev())
    ext = np.zeros(4)
    bd = boxes.to(_dev())
    _lib.check(_lib.load().dad3d_roi_setup(bd.data_ptr(), fidx.data_ptr(), R, F, H, W, 256, ext.ctypes.data, rois.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream), "roi_setup")
    assert torch.equal(rois.view(torch.int32)[:, :4], out["crop_boxes"])
    idx = pred._landmark_index("565")
    img = frames.to(_dev())
    O.draw_points(img, proj.contiguous(), rois, idx)
    torch.cuda.synchronize()
    want = M.overlay_frames(frames.numpy(), "445_landmarks", out["crop_boxes"].cpu().numpy(), fidx.cpu().numpy(),
                            out["valid"].cpu().numpy(), projected=proj.cpu().numpy(), index=flame_static["keypoints_565"])
    assert np.array_equal(img.cpu().numpy(), want)


def test_demo_py_outputs_agree(pred, demo_home, tmp_path):
    """The unmodified demo.py's four overlay outputs on its own demo image (its predictor runs the per-image path, whose
    parameters differ from this call's by encoder rounding): the pixels that differ are a small share of those drawn,
    as in tests/test_demo_unchanged_gpu.py."""
    import cv2
    from oracle import ref_harness as RH
    img = cv2.cvtColor(cv2.imread(os.path.join(RH.root(), "images", "demo_heads", "1.jpeg")), cv2.COLOR_BGR2RGB)
    H, W = img.shape[:2]
    out = pred.predict_batch(torch.from_numpy(img[None].copy()), boxes=torch.tensor([[0, 0, W, H]]), overlay=KINDS)
    torch.cuda.synchronize()
    for k in KINDS:
        _run_demo(demo_home, tmp_path, k)
        want = cv2.cvtColor(cv2.imread(str(tmp_path / f"1_{k}.png")), cv2.COLOR_BGR2RGB)
        got = out[f"frame_{k}"][0].cpu().numpy()
        drawn = ((want != img).any(-1) | (got != img).any(-1)).sum()
        assert drawn > 0, k
        assert (got != want).any(-1).sum() < 0.03 * drawn, (k, int((got != want).any(-1).sum()), int(drawn))


def test_existing_outputs_unchanged_and_no_box_rpy(pred):
    frames = _frames(2, 300, 400, 1)
    boxes, fidx = _scene(2, 300, 400, 2)
    base = pred.predict_batch(frames, boxes=boxes, frame_index=fidx)
    more = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, overlay=KINDS, rpy=True)
    for k, v in base.items():
        assert torch.equal(v, more[k]), k
    x = torch.randn(3, 3, 256, 256, generator=torch.Generator().manual_seed(4))
    a = pred.predict_batch(x)
    b = pred.predict_batch(x, rpy=True)
    for k, v in a.items():
        assert torch.equal(v, b[k]), k
    want = np.array([M.rpy_from_rotation(p[RI:RI + 6]) for p in b["3dmm_params"].cpu().numpy()])
    assert np.allclose(b["rpy"].cpu().numpy(), want, atol=1e-9, rtol=0)
    with pytest.raises(ValueError):
        pred.predict_batch(x, overlay=("pose",))
    with pytest.raises(ValueError):
        pred.predict_batch(frames, boxes=boxes, overlay=("mesh",))


def test_graphed_and_stream_equal_eager(pred):
    F, H, W = 2, 420, 640
    kinds = ("68_landmarks", "445_landmarks", "pose")
    for seed in (5, 6):                                                    # a second box set replays the same graph
        frames = _frames(F, H, W, seed)
        boxes, fidx = _scene(F, H, W, seed)
        eager = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, overlay=kinds, rpy=True)
        eager = {k: v.clone() for k, v in eager.items()}
        g = pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fidx, overlay=kinds, rpy=True)
        for k in ("rpy",) + tuple(f"frame_{k}" for k in kinds):
            assert torch.equal(g[k], eager[k]), (seed, k)
    keys = ("rpy", "frame_pose", "frame_445_landmarks")
    st = pred.open_stream((F, H, W, 3), rois=int(boxes.shape[0]), overlay=kinds, rpy=True, keys=keys)
    st.submit(frames, boxes=boxes, frame_index=fidx)
    res = st.collect()
    for k in keys:
        assert torch.equal(res[k], eager[k].cpu()), k


def test_rpy_against_calculate_rpy(pred):
    from oracle import ref_harness as RH
    if not RH.available():
        pytest.skip("reference not available")
    RH.activate()
    from model_training.model.flame import FLAME_CONSTS, FlameParams, calculate_rpy
    from model_training.model.utils import rot_mat_from_6dof
    from scipy.spatial.transform import Rotation
    from dad_3dheads_b200 import overlay as O
    g = np.random.default_rng(7)
    p = np.zeros((600, 413), np.float32)
    p[:, RI:RI + 6] = g.normal(size=(600, 6)).astype(np.float32)
    for i in range(500, 600):                                              # near gimbal lock: the middle angle near 90
        ang = [g.uniform(-180, 180), 90.0 + (-1) ** i * 10.0 ** g.uniform(-9, -1), g.uniform(-180, 180)]
        m = Rotation.from_euler("xyz", ang, degrees=True).as_matrix().T        # R, whose transpose gives these angles
        p[i, RI:RI + 3], p[i, RI + 3:RI + 6] = m[:, 0], m[:, 1]
    pd = torch.from_numpy(p).to(_dev())
    rpy, _ = O.pose_geometry(pd, RI)
    rpy = rpy.cpu().numpy()
    rot = O.rotation_matrices(pd, RI).cpu().numpy()
    for i in range(600):
        fp = FlameParams.from_3dmm(torch.from_numpy(p[i:i + 1]), FLAME_CONSTS)
        rm = rot_mat_from_6dof(fp.rotation).numpy()[0]
        assert np.array_equal(rm.view(np.int32), rot[i].view(np.int32)), i             # the device's fp32 rotation
        assert np.array_equal(rm.view(np.int32), M.rot_mat_from_6dof(p[i, RI:RI + 6]).view(np.int32))
        want = calculate_rpy(fp)
        w = np.array([want.roll, want.pitch, want.yaw])
        mid = abs(w[2])                                                   # the middle (second) Euler angle
        back = Rotation.from_euler("xyz", [rpy[i, 1] + 180, rpy[i, 2], rpy[i, 0]], degrees=True).as_matrix()
        assert np.linalg.norm(back - rm.T.astype(np.float64)) < 1e-5, i
        if mid < 89:
            assert np.allclose(rpy[i], w, atol=1e-9, rtol=0), (i, rpy[i] - w)


def _guarded(n, dtype, fill):
    """A device buffer of n elements between sentinel bands of 64 elements on each side."""
    buf = torch.full((n + 128,), fill, dtype=dtype, device=_dev())
    return buf, buf[64:64 + n]


def test_cabi_guarded_records_points_and_pose():
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.overlay import point_radius
    lib = _lib.load()
    s = torch.cuda.current_stream().cuda_stream
    g = np.random.default_rng(3)
    F, H, W = 2, 257, 389
    boxes = torch.tensor([[0, 0, W, H], [20, 15, 300, 200], [100, 40, 250, 210], [5, 5, 50, 199], [0, 0, 9, 9]],
                         dtype=torch.int32, device=_dev())
    fidx = torch.tensor([0, 1, 1, 0, 7], dtype=torch.int32, device=_dev())
    R = int(boxes.shape[0])
    rois = torch.empty(R, 72, dtype=torch.uint8, device=_dev())
    ext = np.zeros(4)
    _lib.check(lib.dad3d_roi_setup(boxes.data_ptr(), fidx.data_ptr(), R, F, H, W, 256, ext.ctypes.data, rois.data_ptr(), s),
               "roi_setup")
    params = torch.from_numpy(g.normal(size=(R, 413)).astype(np.float32)).to(_dev())
    rbuf, rpy = _guarded(R * 3, torch.float64, -7.0)
    pbuf, pose = _guarded(R * 32, torch.int32, -7)
    obuf, rot = _guarded(R * 9, torch.float32, -7.0)
    _lib.check(lib.dad3d_pose_geometry(params.data_ptr(), R, 413, RI, rois.data_ptr(), rpy.data_ptr(), pose.data_ptr(),
                                       rot.data_ptr(), s),
               "pose_geometry")
    torch.cuda.synchronize()
    for b in (rbuf, pbuf, obuf):
        assert torch.all(b[:64] == -7) and torch.all(b[-64:] == -7)
    fields = rois.view(torch.int32).cpu().numpy()
    rpy_h = rpy.view(R, 3).cpu().numpy()
    rec = pose.view(R, 32).cpu().numpy()
    rot_h = rot.view(R, 3, 3).cpu().numpy()
    for r in range(R):
        assert np.array_equal(rot_h[r].view(np.int32), M.rot_mat_from_6dof(params[r, RI:RI + 6].cpu().numpy()).view(np.int32))
    for r in range(R):
        assert M.near_boundaries(rpy_h[r], fields[r, 2], fields[r, 3]) == 0
        want = M.pose_record(rpy_h[r], fields[r, :4], fields[r, 4], bool(fields[r, 5]))
        if not want[0]:
            assert rec[r, 0] == 0
            continue
        assert np.array_equal(rec[r], want), r
    # points: fp32 with NaN, inf, beyond int32 and negative; int64 beyond int32; drawn into a guarded frame buffer
    frames0 = _frames(F, H, W, 8).numpy()
    n = F * H * W * 3
    for is_float in (1, 0):
        if is_float:
            src = (g.random((R, 40, 3)) * [W + 60, H + 60, 1] - 30).astype(np.float32)
            src[1, 3, 0], src[1, 4, 1], src[2, 5, 0], src[2, 6, 1] = np.nan, np.inf, 3e9, -2147483904.0
            src[0, :, :2] = -src[0, :, :2]
        else:
            src = g.integers(-30, max(H, W) + 30, (R, 40, 2)).astype(np.int64)
            src[1, 3, 0], src[2, 4, 1] = 2 ** 31, -(2 ** 31) - 1
        idx = torch.tensor([0, 3, 4, 5, 6, 7, 39, 12, 12, 40, -1], dtype=torch.int64, device=_dev())
        fbuf, fr = _guarded(n, torch.uint8, 77)
        fr.copy_(torch.from_numpy(frames0).reshape(-1).to(_dev()))
        srcd = torch.from_numpy(src).to(_dev())
        color = np.array(M.POINT_COLOR, np.uint8)
        _lib.check(lib.dad3d_overlay_points(srcd.data_ptr(), is_float, R, 40, src.shape[2], idx.data_ptr(), int(idx.shape[0]),
                                            rois.data_ptr(), point_radius(H, W), color.ctypes.data, fr.data_ptr(), F, H, W, s),
                   "overlay_points")
        torch.cuda.synchronize()
        assert torch.all(fbuf[:64] == 77) and torch.all(fbuf[-64:] == 77)
        want = frames0.copy()
        ix = idx.cpu().numpy()
        for r in range(R):
            if not fields[r, 5]:
                continue
            sel = src[r][ix[(ix >= 0) & (ix < 40)]]
            xy, ok = M.int_points(sel)
            M.draw_points(want[fields[r, 4]], xy, ok)
        assert np.array_equal(fr.view(F, H, W, 3).cpu().numpy(), want), is_float
    # pose raster into a guarded frame buffer
    fbuf, fr = _guarded(n, torch.uint8, 77)
    fr.copy_(torch.from_numpy(frames0).reshape(-1).to(_dev()))
    key = torch.empty(F * H * W, dtype=torch.int32, device=_dev())
    _lib.check(lib.dad3d_overlay_pose(pose.data_ptr(), R, key.data_ptr(), fr.data_ptr(), F, H, W, s), "overlay_pose")
    torch.cuda.synchronize()
    assert torch.all(fbuf[:64] == 77) and torch.all(fbuf[-64:] == 77)
    want = frames0.copy()
    for r in range(R):
        if rec[r, 0]:
            M.draw_pose_record(want[rec[r, 1]], rec[r])
    assert np.array_equal(fr.view(F, H, W, 3).cpu().numpy(), want)
    # records whose crops reach past the frame (edited, or built for a larger frame): clipped to the frame as well
    moved = rec.copy()
    moved[:, 2] = [W - 40, -60, W - 10, 3, 0][:R]
    moved[:, 3] = [H - 50, -30, 5, H - 20, 0][:R]
    fbuf, fr = _guarded(n, torch.uint8, 77)
    fr.copy_(torch.from_numpy(frames0).reshape(-1).to(_dev()))
    md = torch.from_numpy(moved).to(_dev())
    _lib.check(lib.dad3d_overlay_pose(md.data_ptr(), R, key.data_ptr(), fr.data_ptr(), F, H, W, s), "overlay_pose")
    torch.cuda.synchronize()
    assert torch.all(fbuf[:64] == 77) and torch.all(fbuf[-64:] == 77)
    want = frames0.copy()
    for r in range(R):
        if moved[r, 0]:
            M.draw_pose_record(want[moved[r, 1]], moved[r])
    assert np.array_equal(fr.view(F, H, W, 3).cpu().numpy(), want)
    assert not np.array_equal(want, frames0)


def test_demo_image_equals_demo_utils(pred, flame_static):
    """The demo image as one box [0, 0, W, H]: the reference's own processors on this call's predictions."""
    import cv2
    from oracle import ref_harness as RH
    if not RH.available():
        pytest.skip("reference not available")
    RH.activate()
    import demo_utils
    img = cv2.cvtColor(cv2.imread(os.path.join(GOLDEN, "demo_head_1.jpeg")), cv2.COLOR_BGR2RGB)
    H, W = img.shape[:2]
    frames = torch.from_numpy(img[None].copy())
    out = pred.predict_batch(frames, boxes=torch.tensor([[0, 0, W, H]]), overlay=KINDS, rpy=True)
    torch.cuda.synchronize()
    pts = out["points"][0].cpu().numpy()
    proj = out["projected_vertices"][0:1].cpu()
    params = out["3dmm_params"][0:1].cpu()
    want = {"68_landmarks": demo_utils.draw_landmarks({"points": pts}, img.copy()),
            "191_landmarks": demo_utils.draw_3d_landmarks({"projected_vertices": proj}, img.copy(), "191"),
            "445_landmarks": demo_utils.draw_3d_landmarks({"projected_vertices": proj}, img.copy(), "445"),
            "pose": demo_utils.draw_pose({"3dmm_params": params}, img.copy())}
    assert M.near_boundaries(out["rpy"][0].cpu().numpy(), W, H) == 0
    for k in KINDS:
        assert np.array_equal(out[f"frame_{k}"][0].cpu().numpy(), want[k]), k
