"""-m gpu: several heads drawn into whole frames (dad3d_rasterize_frames, rasterizer.rasterize_batch(image_of_head=),
PnccRenderer.render_frames, predict_batch(boxes=, frame_render=)).

Per frame, image and depth are compared bit for bit with the reference's own C++ rasteriser (oracle/_ref/libsim3dr_ref.so)
called once per head in head order with carried buffers, and tri_index / head_index with tests/frame_render_model.py
(pinned to that library by tests/test_frame_render_model_cpu.py)."""
import itertools
import os

import numpy as np
import pytest
import torch

from tests import frame_render_model as FM
from tests import raster_model
from tests import roi_model as M
from tests.test_frame_render_model_cpu import carried
from tests.test_raster_model_cpu import REF_SO, ref_rasterize, ties_mesh, zero_sign_mesh

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not os.path.isfile(REF_SO), reason="oracle/_ref/libsim3dr_ref.so not built")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
ALL = ("pncc", "depth", "tri_index", "head_index")


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _static():
    from dad_3dheads_b200.rasterizer import load_render_static
    st = load_render_static()
    return st["faces_wo_ears"], st["ncc_colors"]


def _base_heads(n, seed):
    """n decoded FLAME heads in 256 x 256 pixels, z negated (depth: larger wins), centred near the origin."""
    from oracle.flame_oracle import FlameOracle, load_static, sample_params
    p = sample_params(n, seed=seed)
    p[:, 409:411] = 0.0
    p[:, 412] = 1.0
    v = FlameOracle(load_static(), image_size=256).reprojected_vertices(p, to_2d=False).numpy().astype(np.float32)
    v[..., 2] *= -1
    v[..., :2] -= 128.0
    return v


def _place(v, scale, x, y, z=0.0):
    """A head scaled (about 128 * scale pixels wide) and moved, in float32."""
    s = np.float32(scale)
    return (v * s + np.array([x, y, z], np.float32)).astype(np.float32)


def _designed_scene(H, W, seed):
    """Heads and their frames (4 frames): separated depths in both head orders, an exact duplicate, heads partly and fully
    outside the frame, overlapping crowds, a frame without heads, and map entries -1 and 4 (nothing drawn)."""
    g = np.random.default_rng(seed)
    base = _base_heads(6, seed)
    s = min(H, W) / 400.0                                  # heads of 150-400 px at either size
    heads, frames = [], []

    def add(v, f):
        heads.append(v)
        frames.append(f)
    near, far = _place(base[0], 2 * s, W * 0.3, H * 0.5, 300.0), _place(base[1], 2.2 * s, W * 0.33, H * 0.52, -300.0)
    add(far, 0)                                            # frame 0: far first, near second
    add(near, 0)
    add(near, 2)                                           # frame 2: near first
    add(far, 2)
    dup = _place(base[2], 1.5 * s, W * 0.7, H * 0.4)
    add(dup, 0)                                            # exact duplicate: the first one wins
    add(dup, 0)
    add(_place(base[3], 2.5 * s, -20.0, H * 0.5), 0)       # partly left of the frame
    add(_place(base[4], 2 * s, W + 400.0, H * 0.5), 2)     # fully outside
    add(_place(base[5], 1.2 * s, W * 0.5, H - 10.0), 2)    # partly below
    add(_place(base[0], 2 * s, W * 0.5, H * 0.5), -1)      # never drawn
    add(_place(base[1], 2 * s, W * 0.5, H * 0.5), 4)       # == n_images: never drawn
    for k in range(8):                                     # frame 3: an overlapping crowd
        add(_place(base[k % 6], g.uniform(1.2, 3.0) * s, g.uniform(0.2, 0.8) * W, g.uniform(0.2, 0.8) * H,
                   g.uniform(-100, 100)), 3)
    return np.stack(heads), np.array(frames, np.int32), 4


def _check_frames(verts, tris, colors, fo, n, H, W, out, image_name="image"):
    """Each frame of ``out`` against the carried reference (image, depth) and the model (tri_index, head_index)."""
    for f in range(n):
        members = np.flatnonzero(fo == f)
        want_img, want_depth = carried(verts[members], tris, colors, H, W)
        _, _, want_tri, want_head = FM.render_frame(verts[members], tris, None, H, W, members)
        if image_name in out:
            assert np.array_equal(out[image_name][f].cpu().numpy(), want_img), f"frame {f}: image"
        if "depth" in out:
            assert np.array_equal(out["depth"][f].cpu().numpy().view(np.uint32), want_depth.view(np.uint32)), f"frame {f}"
        assert np.array_equal(out["tri_index"][f].cpu().numpy(), want_tri), f"frame {f}: tri_index"
        assert np.array_equal(out["head_index"][f].cpu().numpy(), want_head), f"frame {f}: head_index"


@needs_ref
@pytest.mark.parametrize("H,W,negate_z", [(480, 640, False), (1080, 1920, True)])
def test_designed_frames_bit_exact(cuda_device, H, W, negate_z):
    from dad_3dheads_b200.rasterizer import rasterize_batch
    verts, fo, n = _designed_scene(H, W, 3)
    faces, colors = _static()
    vin = verts.copy()
    if negate_z:
        vin[..., 2] *= -1
    out = rasterize_batch(_t(vin), _t(faces), _t(colors), height=H, width=W, negate_z=negate_z, image_of_head=_t(fo),
                          num_images=n)
    assert set(out) == {"image", "depth", "tri_index", "head_index"} and out["image"].shape == (n, H, W, 3)
    _check_frames(verts, faces, colors, fo, n, H, W, out)
    head = out["head_index"].cpu().numpy()
    h0, h2 = set(np.unique(head[0])), set(np.unique(head[2]))
    assert {-1, 1, 4, 6} <= h0 and 5 not in h0             # the near head, the first duplicate, the partly-out head
    assert {-1, 2, 8} <= h2 and 7 not in h2                # nothing from the head outside the frame
    assert (head[1] == -1).all() and len(set(np.unique(head[3]))) > 4
    assert not np.isin([9, 10], head).any()                # map entries -1 and n_images draw nothing


@needs_ref
@pytest.mark.parametrize("mesh", [ties_mesh, zero_sign_mesh])
def test_ties_across_heads(cuda_device, mesh):
    """Coplanar duplicates, degenerate triangles and -0/+0 depth ties inside and across heads: per image, the lower
    (head, triangle) pair wins; also the -0/+0 tie between whole heads in both orders."""
    from dad_3dheads_b200.rasterizer import rasterize_batch
    v, t = mesh()
    flip = v.copy()
    flip[:, 2] = -flip[:, 2]                               # -0 <-> +0, and other depths mirrored
    heads = np.stack([v, flip, v, v + np.float32([1, 0, 0]), flip, v])
    fo = np.array([0, 0, 1, 1, 2, 2], np.int32)
    colors = np.random.default_rng(0).random((v.shape[0], 3)).astype(np.float32)
    out = rasterize_batch(_t(heads), _t(t), _t(colors), height=32, width=32, image_of_head=_t(fo), num_images=3)
    _check_frames(heads, t, colors, fo, 3, 32, 32, out)


@needs_ref
def test_map_independence(cuda_device):
    """A frame's maps do not change when heads mapped to other frames are added, removed or remapped."""
    from dad_3dheads_b200.rasterizer import rasterize_batch
    verts, fo, n = _designed_scene(480, 640, 5)
    faces, colors = _static()
    tv, tf, tc = _t(verts), _t(faces), _t(colors)
    full = rasterize_batch(tv, tf, tc, height=480, width=640, image_of_head=_t(fo), num_images=n)
    other = fo.copy()
    other[fo != 0] = np.where(np.arange((fo != 0).sum()) % 2 == 0, -1, 7)[: (fo != 0).sum()]
    alone = rasterize_batch(tv, tf, tc, height=480, width=640, image_of_head=_t(other), num_images=n)
    for k in full:
        assert torch.equal(full[k][0], alone[k][0]), k
    assert (alone["head_index"][1:] == -1).all()
    keep = np.flatnonzero(fo == 0)                         # the same frame from a batch of only its heads: same maps
    sub = rasterize_batch(_t(verts[keep]), tf, tc, height=480, width=640,
                          image_of_head=_t(np.zeros(len(keep), np.int32)), num_images=1)
    remapped = torch.where(sub["head_index"][0] >= 0, _t(keep.astype(np.int32))[sub["head_index"][0].long()],
                           sub["head_index"][0])
    assert torch.equal(remapped, full["head_index"][0])
    for k in ("image", "depth", "tri_index"):
        assert torch.equal(sub[k][0], full[k][0]), k


def _lib():
    from dad_3dheads_b200 import _lib
    return _lib


@pytest.mark.parametrize("B,n", [(1, 1), (5, 3), (17, 4)])
def test_guarded_stores_and_null_outputs(cuda_device, B, n):
    """Outputs between sentinel-filled guard bands, with an initial depth buffer and background image: guards unchanged,
    every index written, and every subset of null outputs leaves the requested ones identical."""
    L = _lib()
    lib = L.load()
    dev = _dev()
    g = np.random.default_rng(B + n)
    nv, h, w, c = 60, 24, 29, 3
    base = np.c_[g.uniform(-4, 30, (nv, 2)), g.integers(-3, 4, nv)].astype(np.float32)
    tris = g.integers(0, nv, (150, 3)).astype(np.int32)
    verts = base[None] + np.c_[g.integers(-3, 4, (B, 2)), np.zeros(B)].astype(np.float32)[:, None]
    fo = g.integers(-1, n + 1, B).astype(np.int32)
    fo[0] = 0
    colors = g.random((nv, c)).astype(np.float32)
    bg = g.integers(0, 256, (n, h, w, c), dtype=np.uint8)
    depth0 = np.where(g.random((n, h, w)) < 0.3, g.uniform(-2, 2, (n, h, w)), -1e8).astype(np.float32)
    G = 4096
    tv, tt, tc, tm = _t(verts), _t(tris), _t(colors), _t(fo)
    key = torch.empty(n * h * w, dtype=torch.int64, device=dev)
    n_img, n_px = n * h * w * c, n * h * w

    def run(want, d0=depth0):
        img = torch.full((2 * G + n_img,), 0xA5, dtype=torch.uint8, device=dev)
        dep = torch.full((2 * G + n_px,), 7.5, dtype=torch.float32, device=dev)
        tri = torch.full((2 * G + n_px,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
        hed = torch.full((2 * G + n_px,), 0x3C3C3C3C, dtype=torch.int32, device=dev)
        img[G:G + n_img] = _t(bg.reshape(-1))
        dep[G:G + n_px] = _t(d0.reshape(-1))
        ptr = lambda buf, k, m: buf[G:G + m].data_ptr() if k in want else None   # noqa: E731
        L.check(lib.dad3d_rasterize_frames(tv.data_ptr(), nv, B, tt.data_ptr(), tris.shape[0], tc.data_ptr(), c,
                                           tm.data_ptr(), n, h, w, 0, ptr(img, "image", n_img), ptr(dep, "depth", n_px),
                                           ptr(tri, "tri_index", n_px), ptr(hed, "head_index", n_px), key.data_ptr(),
                                           torch.cuda.current_stream(dev).cuda_stream), "rasterize_frames")
        for buf, fill in ((img, 0xA5), (dep, 7.5), (tri, 0x5A5A5A5A), (hed, 0x3C3C3C3C)):
            assert bool((buf[:G] == fill).all()) and bool((buf[-G:] == fill).all())
        return (img[G:G + n_img].view(n, h, w, c), dep[G:G + n_px].view(n, h, w), tri[G:G + n_px].view(n, h, w),
                hed[G:G + n_px].view(n, h, w))

    names = ("image", "depth", "tri_index", "head_index")
    img, dep, tri, hed = run(set(names))
    for f in range(n):
        members = np.flatnonzero(fo == f)
        uv, ut, uc = FM.union_mesh(verts[members], tris, colors)
        if os.path.isfile(REF_SO):
            want_img, want_depth = ref_rasterize(uv, ut, uc, bg[f], depth0=depth0[f])
        else:
            want_img, want_depth = raster_model.rasterize(uv, ut, uc, h, w, bg[f], depth0[f])[:2]
        _, _, u = raster_model.rasterize(uv, ut, None, h, w, depth0=depth0[f])
        assert np.array_equal(img[f].cpu().numpy(), want_img), f
        assert np.array_equal(dep[f].cpu().numpy().view(np.uint32), want_depth.view(np.uint32)), f
        assert np.array_equal(tri[f].cpu().numpy(), np.where(u >= 0, u % tris.shape[0], -1)), f
        want_head = np.where(u >= 0, members[np.maximum(u, 0) // tris.shape[0]], -1) if len(members) else u
        assert np.array_equal(hed[f].cpu().numpy(), want_head), f
    assert bool((tri >= 0).any()) and bool((tri < 0).any())
    flat = np.full_like(depth0, -1e8)                      # without a depth buffer the z-test threshold is -1e8
    full = dict(zip(names, run(set(names), flat)))
    for r in range(4):
        for want in itertools.combinations(names, r):
            part = dict(zip(names, run(set(want), flat)))
            for k in want:
                assert torch.equal(part[k], full[k]), (want, k)


def test_empty_batches_and_invalid_arguments(cuda_device):
    L = _lib()
    lib = L.load()
    dev = _dev()
    s = torch.cuda.current_stream(dev).cuda_stream
    v = torch.zeros(2, 3, 3, device=dev)
    t = torch.tensor([[0, 1, 2]], dtype=torch.int32, device=dev)
    col = torch.zeros(3, 3, device=dev)
    fo = torch.zeros(2, dtype=torch.int32, device=dev)
    key = torch.empty(3 * 64, dtype=torch.int64, device=dev)
    tri = torch.full((3, 8, 8), 5, dtype=torch.int32, device=dev)
    hed = torch.full((3, 8, 8), 5, dtype=torch.int32, device=dev)
    dep = torch.full((3, 8, 8), 3.0, device=dev)
    torch.cuda.synchronize()
    before = L.launch_count()
    for batch, ntri in ((0, 1), (2, 0)):                    # nothing drawn: indices -1, depth untouched, no launch
        tri.fill_(5), hed.fill_(5)
        L.check(lib.dad3d_rasterize_frames(v.data_ptr(), 3, batch, t.data_ptr(), ntri, None, 1, fo.data_ptr(), 3, 8, 8, 0,
                                           None, dep.data_ptr(), tri.data_ptr(), hed.data_ptr(), key.data_ptr(), s), "")
        assert bool((tri == -1).all()) and bool((hed == -1).all()) and bool((dep == 3.0).all())
    good = [v.data_ptr(), 3, 2, t.data_ptr(), 1, col.data_ptr(), 3, fo.data_ptr(), 3, 8, 8, 0, None, None, tri.data_ptr(),
            hed.data_ptr(), key.data_ptr(), s]
    bad = [(2, -1), (1, 0), (4, -1), (8, -1), (9, 0), (10, 0), (6, 0), (0, None), (3, None), (7, None), (16, None)]
    for i, val in bad:
        args = list(good)
        args[i] = val
        assert lib.dad3d_rasterize_frames(*args) == -1, (i, val)
        assert b"invalid argument" in lib.dad3d_last_error()
    args = list(good)
    args[9], args[10] = 65536, 32768                       # h * w = 2^31
    assert lib.dad3d_rasterize_frames(*args) == -1
    img = torch.empty(3 * 64 * 3, dtype=torch.uint8, device=dev)
    args = list(good)
    args[5], args[12] = None, img.data_ptr()               # an image needs colours
    assert lib.dad3d_rasterize_frames(*args) == -1
    for batch, ntri in ((65536, 65536), (65537, 65535), (1 << 30, 4)):    # batch * ntri > 2^32 - 2: the pair overflows
        args = list(good)
        args[2], args[4] = batch, ntri
        assert lib.dad3d_rasterize_frames(*args) == -1, (batch, ntri)
        assert b"2^32" in lib.dad3d_last_error()
    assert L.launch_count() == before
    L.check(lib.dad3d_rasterize_frames(*good), "valid call")
    assert L.launch_count() == before + 2
    from dad_3dheads_b200.rasterizer import rasterize_batch
    for kw in (dict(image_of_head=fo), dict(num_images=3), dict(image_of_head=fo[:1], num_images=3),
               dict(image_of_head=fo.long(), num_images=3), dict(image_of_head=fo, num_images=3, reverse=True)):
        with pytest.raises(ValueError):
            rasterize_batch(v, t, col, height=8, width=8, **kw)


# ------------------------------------------------------------------------------------------------- predictor
@pytest.fixture(scope="module")
def pred(cuda_device):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


def _frames(F, H, W, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (F, H, W, 3), dtype=np.uint8))


def _boxes(F, H, W, R, seed):
    """R head boxes of 150-400 px on F frames, with overlapping boxes, exact duplicates and invalid ones."""
    g = np.random.default_rng(seed)
    side = g.integers(150, 400, R)
    boxes = np.stack([g.integers(-50, W - 100, R), g.integers(-50, H - 100, R), side, (side * g.uniform(1.0, 1.3, R))], 1)
    boxes = boxes.astype(np.int64)
    fi = g.integers(0, F, R)
    if R >= 8:
        boxes[3], fi[3] = boxes[1], fi[1]                  # duplicate
        boxes[5] = boxes[4] + [40, 30, 0, 0]               # overlapping
        fi[5] = fi[4]
        boxes[6] = [W + 10, 10, 100, 100]                  # outside the frame: invalid
        boxes[7] = [0, 0, W, 1]                            # a 0-pixel side: invalid
    return torch.from_numpy(boxes), torch.from_numpy(fi)


def _frame_map(out, fi):
    return torch.where(out["valid"], fi.to(out["valid"].device, torch.int32), -1).to(torch.int32)


@needs_ref
def test_end_to_end_equals_renderer_and_reference(pred):
    """4 frames of 1920 x 1080, 64 boxes: predict_batch's frame maps equal PnccRenderer.render_frames on its own projected
    vertices and frame map, and the reference (pncc() / the C++ rasteriser) on the union of those vertices."""
    from dad_3dheads_b200.rasterizer import PnccRenderer
    F, H, W, R = 4, 1080, 1920, 64
    frames = _frames(F, H, W, 40)
    boxes, fi = _boxes(F, H, W, R, 41)
    got = pred.predict_batch(frames, boxes=boxes, frame_index=fi, extend=0.1, to_2d=False, frame_render=ALL)
    plain = pred.predict_batch(frames, boxes=boxes, frame_index=fi, extend=0.1, to_2d=False)
    assert set(got) == set(plain) | {f"frame_{k}" for k in ALL}
    for k in plain:
        assert torch.equal(got[k], plain[k]), k
    assert got["frame_pncc"].shape == (F, H, W, 3) and got["frame_pncc"].dtype == torch.uint8
    assert got["frame_depth"].dtype == torch.float32 and got["frame_head_index"].dtype == torch.int32
    valid = got["valid"].cpu().numpy()
    assert not valid[6] and not valid[7] and valid.sum() >= R - 4
    fmap = _frame_map(got, fi)
    want = PnccRenderer(_dev()).render_frames(got["projected_vertices"], fmap, F, (H, W))
    for k in ALL:
        assert torch.equal(got[f"frame_{k}"], want[k]), k
    faces, colors = _static()
    v = got["projected_vertices"].cpu().numpy().copy()
    v[..., 2] *= -1                                        # pncc_estimator.py:88
    out = {"image": got["frame_pncc"], "depth": got["frame_depth"], "tri_index": got["frame_tri_index"],
           "head_index": got["frame_head_index"]}
    _check_frames(v, faces, colors, fmap.cpu().numpy(), F, H, W, out)
    head = got["frame_head_index"].cpu().numpy()
    assert not np.isin([3, 6, 7], head).any()              # the later duplicate and the invalid boxes never show
    assert len(np.unique(head)) > 2
    from oracle import ref_harness
    if ref_harness.available():                            # and the reference's pncc() itself on the union mesh
        import importlib
        ref_harness.activate()
        pe = importlib.import_module("inference.pncc_estimator")
        est = pe.PNCCEstimator()
        fm = fmap.cpu().numpy()
        for f in range(F):
            uv, ut, _ = FM.union_mesh(v[fm == f], np.asarray(est.faces_wo_back_remapped), None)
            ut = ut.astype(np.int32)                       # the rasteriser takes int32 triangles
            uc = np.tile(est.colors, ((fm == f).sum(), 1))
            ref = pe.pncc(np.zeros((H, W, 3), np.uint8), uv, ut, uc, with_bg_flag=False)
            assert np.array_equal(got["frame_pncc"][f].cpu().numpy(), ref), f


def test_against_live_reference_on_pasted_demo_head(pred):
    """The demo head pasted into a larger frame: frame_pncc against the reference's PNCCEstimator on the frame-space
    parameters of its own crop + __call__ + move.  Parameters and vertices differ by encoder and decode rounding, so the
    maps are compared by coverage IoU and mean colour difference on the commonly covered pixels."""
    import cv2
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from oracle import ref_harness as RH
    if not RH.available():
        pytest.skip("reference not available")
    img = cv2.cvtColor(cv2.imread(os.path.join(GOLDEN, "demo_head_1.jpeg")), cv2.COLOR_BGR2RGB)
    frame = np.random.default_rng(9).integers(0, 256, (1300, 1500, 3), dtype=np.uint8)
    oy, ox = 211, 377
    frame[oy:oy + img.shape[0], ox:ox + img.shape[1]] = img
    box = [ox + 60, oy + 90, 640, 820]
    ref = RH.predictor(synthetic_state_dict(0))
    from model_training.data.utils import ensure_bbox_boundaries, extend_bbox
    import importlib
    pe = importlib.import_module("inference.pncc_estimator")
    x, y, w, h = (int(v) for v in ensure_bbox_boundaries(extend_bbox(np.array(box), 0.1), frame.shape[:2]))
    want = ref(frame[y:y + h, x:x + w])
    p = want["3dmm_params"].clone()
    p[:, M.TRANSLATION_IDX:M.TRANSLATION_IDX + 2] += torch.tensor([[x, y]], dtype=torch.float32) * 2 / 256
    want_img = pe.PNCCEstimator()(frame, {"3dmm_params": p})
    got = pred.predict_batch(torch.from_numpy(frame[None]), boxes=torch.tensor([box]), extend=0.1, to_2d=False,
                             fast_decode=False, frame_render=ALL)
    # the reference's coverage: its own vertices through its rasteriser's depth buffer
    est = pe.PNCCEstimator()
    vref, _ = est._transform_3dmm_to_3d_face_polygons(p, est.head_mesh.flame)
    _, ref_depth = ref_rasterize(vref, np.asarray(est.faces_wo_back_remapped), est.colors.astype(np.float32),
                                 np.zeros(frame.shape, np.uint8)) if os.path.isfile(REF_SO) else (None, None)
    ref_cover = (ref_depth != np.float32(-1e8)) if ref_depth is not None else want_img.any(-1)
    cover = got["frame_head_index"][0].cpu().numpy() >= 0
    iou = (cover & ref_cover).sum() / (cover | ref_cover).sum()
    both = cover & ref_cover
    diff = np.abs(got["frame_pncc"][0].cpu().numpy()[both].astype(np.int32) - want_img[both].astype(np.int32)).mean()
    print(f"live reference: coverage IoU {iou:.5f} ({cover.sum()} vs {ref_cover.sum()} px), mean |dcolour| {diff:.4f}")
    assert cover.sum() > 1000
    assert iou >= 0.99 and diff <= 1.0, (iou, diff)
    # the documented overlay: with_background=True is the black-background render over the frame where a head covers
    want_overlay = pe.PNCCEstimator()(frame, {"3dmm_params": p}, with_background=True)
    assert np.array_equal(want_overlay, np.where(ref_cover[..., None], want_img, frame))
    overlay = torch.where(got["frame_head_index"][..., None] >= 0, got["frame_pncc"], torch.from_numpy(frame[None]).to(_dev()))
    assert np.array_equal(overlay[0].cpu().numpy()[~cover], frame[~cover])


def _steps(F, H, W, R):
    """Three consecutive steps whose frames, boxes, frame indices and validity change."""
    out = []
    for i in range(3):
        boxes, fi = _boxes(F, H, W, R, 50 + i)
        if i == 1:
            boxes[2] = torch.tensor([W + 5, 5, 50, 50])   # an invalid box in the middle step
        out.append((_frames(F, H, W, 60 + i), boxes, fi))
    return out


def test_graphed_and_stream_equal_eager(pred):
    F, H, W, R = 3, 480, 640, 10
    steps = _steps(F, H, W, R)
    kw = dict(extend=0.1, to_2d=False, frame_render=ALL)
    want = [{k: v.clone() for k, v in pred.predict_batch(fr, boxes=b, frame_index=f, **kw).items()} for fr, b, f in steps]
    assert not want[1]["valid"][2] and want[0]["valid"][2]
    assert all(len(torch.unique(w["frame_head_index"])) > 2 for w in want)
    for (fr, b, f), w in zip(steps, want):
        got = pred.predict_batch_graphed(fr, boxes=b, frame_index=f, **kw)
        torch.cuda.synchronize()
        assert set(got) == set(w)
        for k in w:
            assert torch.equal(got[k], w[k]), k
    plain = pred.predict_batch_graphed(steps[0][0], boxes=steps[0][1], frame_index=steps[0][2], extend=0.1, to_2d=False)
    assert "frame_pncc" not in plain                       # frame_render is part of the graph key
    keys = ("3dmm_params", "valid") + tuple(f"frame_{k}" for k in ALL)
    st = pred.open_stream((F, H, W, 3), rois=R, keys=keys, depth=2, **kw)
    got = []
    for fr, b, f in steps:
        if st._inflight == st.depth:
            got.append({k: v.clone() for k, v in st.collect().items()})
        st.submit(fr.pin_memory(), boxes=b, frame_index=f)
    while st._inflight:
        got.append({k: v.clone() for k, v in st.collect().items()})
    for i in range(3):
        for k in keys:
            assert torch.equal(got[i][k], want[i][k].cpu()), (i, k)


def test_device_boxes_need_no_host_synchronisation(pred):
    F, H, W, R = 2, 480, 640, 8
    frames = _frames(F, H, W, 70).to(pred.device)
    boxes, fi = _boxes(F, H, W, R, 71)
    boxes_d, fi_d = boxes.to(pred.device), fi.to(pred.device)
    kw = dict(boxes=boxes_d, frame_index=fi_d, to_2d=False, frame_render=ALL)
    want = {k: v.clone() for k, v in pred.predict_batch(frames, **kw).items()}       # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = pred.predict_batch(frames, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    empty = pred.predict_batch(frames, boxes=torch.zeros(0, 4, dtype=torch.int64), to_2d=False, frame_render=ALL)
    assert (empty["frame_head_index"] == -1).all() and (empty["frame_pncc"] == 0).all()
    assert (empty["frame_depth"] == -1e8).all() and empty["frame_tri_index"].shape == (F, H, W)


def test_invalid_arguments_raise_before_any_launch(pred):
    from dad_3dheads_b200 import _lib
    frames = _frames(2, 64, 80, 16)
    boxes = torch.tensor([[1, 2, 30, 40], [5, 6, 20, 10]])
    x = torch.zeros(1, 3, 256, 256)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for kw in (dict(to_2d=False, frame_render="pncc"),                                 # without boxes
               dict(boxes=boxes, frame_render=ALL),                                    # to_2d=True
               dict(boxes=boxes, to_2d=False, frame_render=("pncc", "normals"))):      # unknown map
        with pytest.raises(ValueError):
            pred.predict_batch(x if "boxes" not in kw else frames, **kw)
        with pytest.raises(ValueError):
            pred.predict_batch_graphed(x if "boxes" not in kw else frames, **kw)
    with pytest.raises(ValueError):
        pred.open_stream((2, 64, 80, 3), to_2d=False, frame_render="pncc")             # a stream without rois
    with pytest.raises(ValueError):
        pred.predict_batch(frames, boxes=boxes, to_2d=False, render="pncc", frame_render="pncc")
    assert _lib.launch_count() == before
