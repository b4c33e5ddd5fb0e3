"""-m gpu: the demo's head and face wireframes (csrc/overlay.cu dad3d_overlay_mesh, predict_batch(overlay=("head_mesh",
"face_mesh"))).

Every frame is compared byte for byte with tests/wireframe_model.py (pinned to cv2 and to the unmodified
demo_utils.draw_mesh by tests/test_wireframe_model_cpu.py) and, where the reference is built, with demo_utils.draw_mesh
applied per box, on this call's own device outputs."""
import os

import numpy as np
import pytest
import torch

from tests import wireframe_model as M
from tests.test_demo_unchanged_gpu import _run_demo, demo_home  # noqa: F401  (fixture)
from tests.test_overlay_gpu import _dev, _frames, _scene

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
KINDS = M.WIREFRAME_KINDS


@pytest.fixture(scope="module")
def pred():
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


def _rois(boxes, fidx, F, H, W):
    from dad_3dheads_b200 import _lib
    R = int(boxes.shape[0])
    rois = torch.empty(R, 72, dtype=torch.uint8, device=_dev())
    ext = np.zeros(4)
    bd = boxes.to(_dev(), torch.int32).contiguous()
    fd = fidx.to(_dev(), torch.int32).contiguous()
    _lib.check(_lib.load().dad3d_roi_setup(bd.data_ptr(), fd.data_ptr(), R, F, H, W, 256, ext.ctypes.data, rois.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream), "roi_setup")
    return rois


def _reference(frames, proj, fidx, valid, kind):
    """demo_utils.draw_mesh applied per valid box, in box order; a box where cv2 raises leaves its frame as it was."""
    import cv2
    from oracle import ref_harness as RH
    if not RH.available():
        return None
    RH.activate()
    import demo_utils
    out = frames.copy()
    for r in range(len(valid)):
        if not valid[r]:
            continue
        f = int(fidx[r])
        try:
            out[f] = demo_utils.draw_mesh({"projected_vertices": torch.from_numpy(proj[r:r + 1, :, :2].copy())}, out[f],
                                          "head" if kind == "head_mesh" else "face")
        except cv2.error:
            pass
    return out


def _check(got, want, what):
    bad = np.argwhere((got != want).any(-1))
    assert len(bad) == 0, (what, len(bad), bad[:5].tolist())


@pytest.mark.parametrize("F,H,W,to_2d", [(3, 333, 517, True), (2, 1080, 1920, False), (1, 201, 199, True)])
def test_frames_equal_the_model_and_draw_mesh(pred, flame_static, F, H, W, to_2d):
    frames = _frames(F, H, W, H + 1)
    keep = frames.clone()
    boxes, fidx = _scene(F, H, W, W + 1)
    dev_frames = frames.to(_dev())
    out = pred.predict_batch(dev_frames, boxes=boxes, frame_index=fidx, to_2d=to_2d, overlay=KINDS)
    torch.cuda.synchronize()
    assert torch.equal(dev_frames.cpu(), keep)                              # the input frames are never written
    proj = out["projected_vertices"].cpu().numpy()
    valid, fi = out["valid"].cpu().numpy(), fidx.cpu().numpy()
    for k in KINDS:
        got = out[f"frame_{k}"].cpu().numpy()
        assert got.shape == (F, H, W, 3) and got.dtype == np.uint8
        _check(got, M.wireframe_frames(frames.numpy(), fi, valid, proj, M.subset_edges(flame_static, k)), k)
        assert not np.array_equal(got, frames.numpy()), k
        ref = _reference(frames.numpy(), proj, fi, valid, k)
        if ref is not None:
            _check(got, ref, ("demo_utils", k))


def _template_scene(static, F, H, W, sizes, seed, ncomp=2):
    g = np.random.default_rng(seed)
    heads, boxes, fidx = [], [], []
    for s in sizes:
        x, y = (g.uniform(*sorted((-0.2 * s, n - 0.8 * s))) for n in (W, H))
        heads.append(M.template_head(static, x, y, s, ncomp))
        boxes.append((0, 0, W, H))
        fidx.append(int(g.integers(0, F)))
    return np.stack(heads), torch.tensor(boxes, dtype=torch.int32), torch.tensor(fidx, dtype=torch.int32)


def _draw(frames, heads, rois, edges):
    from dad_3dheads_b200 import overlay as O
    img = torch.from_numpy(frames).to(_dev())
    O.draw_mesh(img, torch.from_numpy(heads).to(_dev()).contiguous(), rois,
                torch.from_numpy(edges.astype(np.int32)).to(_dev()))
    torch.cuda.synchronize()
    return img.cpu().numpy()


@pytest.mark.parametrize("sizes", [(12, 20, 25, 30, 60, 60), (900, 1500, 2400), (150, 400, 250, 3000, 40)])
def test_small_and_frame_sized_heads(flame_static, sizes):
    """Template heads from a few pixels (every pixel blended dozens of times) to far beyond the frame."""
    F, H, W = 2, 540, 961
    frames = _frames(F, H, W, len(sizes)).numpy()
    heads, boxes, fidx = _template_scene(flame_static, F, H, W, sizes, sum(sizes), ncomp=3)
    rois = _rois(boxes, fidx, F, H, W)
    valid = np.ones(len(sizes), bool)
    for k in KINDS:
        e = M.subset_edges(flame_static, k)
        got = _draw(frames, heads, rois, e)
        _check(got, M.wireframe_frames(frames, fidx.numpy(), valid, heads, e), (k, sizes))
        ref = _reference(frames, heads, fidx.numpy(), valid, k)
        if ref is not None:
            _check(got, ref, ("demo_utils", k, sizes))


def test_non_finite_and_far_heads(flame_static):
    """NaN, infinite and beyond-int32 vertices blank exactly the boxes whose subset reaches them; one head is bad only on
    an ear vertex, which blanks head_mesh and leaves face_mesh."""
    F, H, W = 2, 480, 640
    frames = _frames(F, H, W, 21).numpy()
    heads, boxes, fidx = _template_scene(flame_static, F, H, W, (200, 220, 240, 260, 280, 300, 320), 22)
    ear = np.setdiff1d(np.unique(M.subset_edges(flame_static, "head_mesh")),
                       np.unique(M.subset_edges(flame_static, "face_mesh")))
    face = np.unique(M.subset_edges(flame_static, "face_mesh"))
    heads[0] = np.nan
    heads[1, face[::7], 0] = np.inf
    heads[2, face[::5], 1] = 3e9
    heads[3, face[10], 0] = -2147483904.0
    heads[4, ear[3], 1] = np.nan                                          # outside the face subset only
    heads[5, face[4], 0] = -2147483648.5                                  # truncates to INT32_MIN: cv2 accepts it
    rois = _rois(boxes, fidx, F, H, W)
    valid = np.ones(len(heads), bool)
    drawn = {}
    for k in KINDS:
        e = M.subset_edges(flame_static, k)
        got = _draw(frames, heads, rois, e)
        _check(got, M.wireframe_frames(frames, fidx.numpy(), valid, heads, e), k)
        ref = _reference(frames, heads, fidx.numpy(), valid, k)
        if ref is not None:
            _check(got, ref, ("demo_utils", k))
        drawn[k] = [M.mesh_stamps(heads[r], e, W, H) is not None for r in range(len(heads))]
    assert drawn["head_mesh"] == [False, False, False, False, False, True, True]
    assert drawn["face_mesh"] == [False, False, False, False, True, True, True]


def _guarded(n, dtype, fill):
    buf = torch.full((n + 128,), fill, dtype=dtype, device=_dev())
    return buf, buf[64:64 + n]


def test_cabi_guarded(flame_static):
    from dad_3dheads_b200 import _lib
    lib = _lib.load()
    s = torch.cuda.current_stream().cuda_stream
    F, H, W = 2, 257, 389
    boxes = torch.tensor([[0, 0, W, H], [20, 15, 300, 200], [100, 40, 250, 210], [0, 0, 9, 9]], dtype=torch.int32)
    fidx = torch.tensor([0, 1, 1, 7], dtype=torch.int32)                  # the last record is invalid
    rois = _rois(boxes, fidx, F, H, W)
    R = 4
    heads = np.stack([M.template_head(flame_static, x, y, sz, 3) for x, y, sz in
                      ((-30, -20, 200), (W - 150, H - 120, 300), (40, 30, 120), (10, 10, 100))])
    e = M.subset_edges(flame_static, "face_mesh")
    bad = e.copy()
    bad[5, 1] = heads.shape[1]                                             # an index past the head: box draws nothing
    frames0 = _frames(F, H, W, 3).numpy()
    n = F * H * W * 3
    hd = torch.from_numpy(heads).to(_dev())
    color = np.array(M.EDGE_COLOR, np.uint8)
    for edges, draws in ((e, True), (bad, False)):
        ed = torch.from_numpy(edges.astype(np.int32)).to(_dev())
        fbuf, fr = _guarded(n, torch.uint8, 77)
        fr.copy_(torch.from_numpy(frames0).reshape(-1).to(_dev()))
        wbuf, ws = _guarded(R * 5, torch.int32, -7)
        _lib.check(lib.dad3d_overlay_mesh(hd.data_ptr(), R, heads.shape[1], 3, ed.data_ptr(), int(ed.shape[0]),
                                          rois.data_ptr(), color.ctypes.data, ws.data_ptr(), fr.data_ptr(), F, H, W, s),
                   "overlay_mesh")
        torch.cuda.synchronize()
        for b, v in ((fbuf, 77), (wbuf, -7)):
            assert torch.all(b[:64] == v) and torch.all(b[-64:] == v)
        wsh = ws.view(R, 5).cpu().numpy()
        assert wsh[3, 0] == -1
        got = fr.view(F, H, W, 3).cpu().numpy()
        if draws:
            want = M.wireframe_frames(frames0, fidx.numpy() % F, [True, True, True, False], heads, e)
            assert np.array_equal(got, want)
            assert list(wsh[:3, 0]) == [0, 1, 1]
        else:
            assert np.array_equal(got, frames0) and np.all(wsh[:, 0] == -1)
    p = hd.data_ptr()
    args = dict(v=p, R=R, nv=heads.shape[1], c=3, e=p, E=10, roi=rois.data_ptr(), col=color.ctypes.data, ws=p, fr=p, F=F,
                H=H, W=W)
    for k, v in (("v", None), ("e", None), ("roi", None), ("col", None), ("ws", None), ("fr", None), ("c", 4), ("c", 1),
                 ("nv", 0), ("R", -1), ("E", -1), ("H", 0), ("W", -3), ("F", 0)):
        a = dict(args, **{k: v})
        rc = lib.dad3d_overlay_mesh(a["v"], a["R"], a["nv"], a["c"], a["e"], a["E"], a["roi"], a["col"], a["ws"], a["fr"],
                                    a["F"], a["H"], a["W"], s)
        assert rc != 0, k
    assert lib.dad3d_overlay_mesh(None, 0, 1, 2, None, 5, None, None, None, None, 1, 1, 1, s) == 0     # R = 0: nothing


def test_graphed_and_stream_equal_eager_and_others_unchanged(pred):
    F, H, W = 2, 420, 640
    others = ("68_landmarks", "pose")
    for seed in (5, 6):                                                    # a second box set replays the same graph
        frames = _frames(F, H, W, seed)
        boxes, fidx = _scene(F, H, W, seed)
        base = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, overlay=others)
        base = {k: v.clone() for k, v in base.items()}
        eager = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, overlay=others + KINDS)
        eager = {k: v.clone() for k, v in eager.items()}
        for k, v in base.items():
            assert torch.equal(v, eager[k]), k                             # the existing outputs are unchanged
        g = pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fidx, overlay=others + KINDS)
        for k in eager:
            assert torch.equal(g[k], eager[k]), (seed, k)
    keys = ("frame_head_mesh", "frame_face_mesh", "frame_pose")
    st = pred.open_stream((F, H, W, 3), rois=int(boxes.shape[0]), overlay=others + KINDS, keys=keys)
    st.submit(frames, boxes=boxes, frame_index=fidx)
    res = st.collect()
    for k in keys:
        assert torch.equal(res[k], eager[k].cpu()), k


def test_demo_py_outputs_agree(pred, demo_home, tmp_path):
    """The unmodified demo.py's head_mesh / face_mesh on its own demo image (its predictor runs the per-image path, whose
    vertices differ from this call's by encoder rounding): the pixels that differ are a small share of those drawn."""
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
