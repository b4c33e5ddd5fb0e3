"""-m gpu: the batched rasteriser (dad3d_rasterize_batch, rasterizer.rasterize_batch / PnccRenderer) and its use in
FaceMeshPredictor.predict_batch(render=...).  Every head is compared bit for bit with the reference's own C++ rasteriser
(oracle/_ref/libsim3dr_ref.so) for image and depth, and with tests/raster_model.py (pinned to that library by
tests/test_raster_model_cpu.py) for the winning triangle."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch

from tests import raster_model
from tests.test_raster_model_cpu import REF_SO, ref_rasterize, ties_mesh, zero_sign_mesh

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not os.path.isfile(REF_SO), reason="oracle/_ref/libsim3dr_ref.so not built")


def _faces():
    from dad_3dheads_b200.flame import load_flame_static
    return load_flame_static()["faces"].astype(np.int32)


def _heads(size):
    """Six decoded heads (fp32, z as decoded: callers negate it) with varied translation and scale: two ordinary ones, one
    partly off the image, one fully off it, a tiny one and a large rotated one."""
    from oracle.flame_oracle import FlameOracle, load_static, sample_params
    p = sample_params(6, seed=11)
    p[:, 409:411] *= 0.3
    p[:, 412] = torch.tensor([2.0, 1.0, 2.0, 2.0, -0.9, 4.0])
    p[2, 409] = 0.9                                       # right half off the image
    p[3, 409:411] = torch.tensor([4.0, -4.0])             # entirely outside
    v = FlameOracle(load_static(), image_size=size).reprojected_vertices(p, to_2d=False).numpy().astype(np.float32)
    return v


def _negated(v):
    v = v.copy()
    v[..., 2] *= -1
    return v


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _check_heads(v_negated, faces, colors, bg, out, reverse):
    """Each head of ``out`` against the reference library (image, depth) and the model (tri_index)."""
    h, w = bg.shape[1:3]
    for b in range(v_negated.shape[0]):
        want_img, want_depth = ref_rasterize(v_negated[b], faces, colors, bg[b], reverse)
        _, _, want_tri = raster_model.rasterize(v_negated[b], faces, None, h, w)
        assert np.array_equal(out["image"][b].cpu().numpy(), want_img), f"head {b}: image"
        assert np.array_equal(out["depth"][b].cpu().numpy().view(np.uint32), want_depth.view(np.uint32)), f"head {b}: depth"
        assert np.array_equal(out["tri_index"][b].cpu().numpy(), want_tri), f"head {b}: tri_index"


@needs_ref
@pytest.mark.parametrize("h,w,c,reverse,negate_z", [(256, 256, 3, False, True), (256, 256, 1, True, False),
                                                     (200, 317, 3, True, True), (200, 317, 1, False, False)])
def test_each_head_bit_exact(cuda_device, h, w, c, reverse, negate_z):
    from dad_3dheads_b200.rasterizer import rasterize_batch
    v = _heads(256)
    faces = _faces()
    g = np.random.default_rng(h + c)
    colors = g.random((v.shape[1], c)).astype(np.float32)
    bg = g.integers(0, 256, (v.shape[0], h, w, c), dtype=np.uint8)
    vin = v if negate_z else _negated(v)
    out = rasterize_batch(_t(vin), _t(faces), _t(colors), height=h, width=w, image=_t(bg), reverse=reverse,
                          negate_z=negate_z)
    _check_heads(_negated(v), faces, colors, bg, out, reverse)
    cover = [(out["tri_index"][b] >= 0).float().mean().item() for b in range(v.shape[0])]
    assert cover[3] == 0 and 0 < cover[4] < 0.01 and min(cover[0], cover[2]) > 0.02, cover
    # negate_z equals rendering explicitly negated vertices, bit for bit
    other = rasterize_batch(_t(_negated(vin)), _t(faces), _t(colors), height=h, width=w, image=_t(bg), reverse=reverse,
                            negate_z=not negate_z)
    for k in out:
        assert torch.equal(out[k], other[k]), k


@needs_ref
@pytest.mark.parametrize("mesh", [ties_mesh, zero_sign_mesh])
def test_ties_and_degenerate_triangles_across_heads(cuda_device, mesh):
    """Coplanar duplicates (lowest index wins), zero-area and off-image triangles, and -0/+0 depth ties, repeated over heads
    with per-head integer offsets (which keep every tie exact)."""
    from dad_3dheads_b200.rasterizer import rasterize_batch
    v, t = mesh()
    B = 7
    off = np.array([[b % 3, -(b % 2), 0] for b in range(B)], np.float32)
    vb = v[None] + off[:, None]
    colors = np.random.default_rng(0).random((v.shape[0], 3)).astype(np.float32)
    bg = np.random.default_rng(1).integers(0, 256, (B, 32, 32, 3), dtype=np.uint8)
    out = rasterize_batch(_t(vb), _t(t), _t(colors), height=32, width=32, image=_t(bg))
    _check_heads(vb, t, colors, bg, out, False)


@needs_ref
def test_batch_independence(cuda_device):
    from dad_3dheads_b200.rasterizer import rasterize_batch
    v = _negated(_heads(256))
    order = [0, 1, 0, 5, 2, 0, 4, 5]                      # identical heads at different positions
    vb, faces = _t(v[order]), _t(_faces())
    colors = _t(np.random.default_rng(2).random((v.shape[1], 3)).astype(np.float32))
    out = rasterize_batch(vb, faces, colors, height=256, width=256)
    for b in range(len(order)):
        one = rasterize_batch(vb[b:b + 1], faces, colors, height=256, width=256)
        for k in out:
            assert torch.equal(out[k][b], one[k][0]), (b, k)
    for b, a in itertools.combinations(range(len(order)), 2):
        if order[a] == order[b]:
            for k in out:
                assert torch.equal(out[k][a], out[k][b]), (a, b, k)


def test_batch_beyond_the_grid_y_limit(cuda_device):
    """70 001 heads of a 4-vertex mesh on 4x4 images: heads past 65 535 loop over grid y and are rendered like the rest."""
    from dad_3dheads_b200.rasterizer import rasterize_batch
    quad = np.array([[0.2, 0.1, 1], [3.6, 0.3, 2], [0.1, 3.7, 3], [3.5, 3.4, 0]], np.float32)
    tris = np.array([[0, 1, 2], [1, 3, 2], [0, 3, 2]], np.int32)
    colors = np.random.default_rng(3).random((4, 2)).astype(np.float32)
    B, kinds = 70001, 35
    kind = np.arange(B) % kinds
    shift = np.stack([(np.arange(kinds) % 5) * 0.3 - 0.6, (np.arange(kinds) // 5) * 0.2 - 0.6, np.arange(kinds) % 3], 1)
    verts = quad[None] + shift[:, None].astype(np.float32)
    out = rasterize_batch(_t(verts[kind]), _t(tris), _t(colors), height=4, width=4)
    want = [raster_model.rasterize(verts[k], tris, colors, 4, 4) for k in range(kinds)]
    kt = torch.from_numpy(kind).to(_dev())
    for i, name in enumerate(("image", "depth", "tri_index")):
        table = _t(np.stack([x[i] for x in want]))
        assert torch.equal(out[name], table[kt]), name
    assert (out["tri_index"][-1] >= 0).any()


def _lib():
    from dad_3dheads_b200 import _lib
    return _lib


@pytest.mark.parametrize("B", [1, 3, 17])
def test_guarded_stores_and_null_outputs(cuda_device, B):
    """Outputs between sentinel-filled guard bands: guards unchanged, every tri_index written, background pixels keep each
    head's own bytes, and any subset of null outputs leaves the requested ones identical."""
    L = _lib()
    lib = L.load()
    dev = _dev()
    g = np.random.default_rng(B)
    nv, h, w, c = 60, 24, 29, 3
    base = np.c_[g.uniform(-4, 30, (nv, 2)), g.integers(-3, 4, nv)].astype(np.float32)
    tris = g.integers(0, nv, (150, 3)).astype(np.int32)
    verts = base[None] + np.c_[g.integers(-3, 4, (B, 2)), np.zeros(B)].astype(np.float32)[:, None]
    colors = g.random((nv, c)).astype(np.float32)
    bg = g.integers(0, 256, (B, h, w, c), dtype=np.uint8)
    depth0 = np.where(g.random((B, h, w)) < 0.3, g.uniform(-2, 2, (B, h, w)), -1e8).astype(np.float32)
    G = 4096
    tv, tt, tc = _t(verts), _t(tris), _t(colors)
    key = torch.empty(B * h * w, dtype=torch.int64, device=dev)
    n_img, n_px = B * h * w * c, B * h * w

    def run(want, d0=depth0):
        img = torch.full((2 * G + n_img,), 0xA5, dtype=torch.uint8, device=dev)
        dep = torch.full((2 * G + n_px,), 7.5, dtype=torch.float32, device=dev)
        tri = torch.full((2 * G + n_px,), 0x5A5A5A5A, dtype=torch.int32, device=dev)
        img[G:G + n_img] = _t(bg.reshape(-1))
        dep[G:G + n_px] = _t(d0.reshape(-1))
        ptr = lambda buf, k, n: buf[G:G + n].data_ptr() if k in want else None   # noqa: E731
        L.check(lib.dad3d_rasterize_batch(tv.data_ptr(), nv, B, tt.data_ptr(), tris.shape[0], tc.data_ptr(), c, h, w, 1, 0,
                                          ptr(img, "image", n_img), ptr(dep, "depth", n_px), ptr(tri, "tri_index", n_px),
                                          key.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "rasterize_batch")
        for buf, fill in ((img, 0xA5), (dep, 7.5), (tri, 0x5A5A5A5A)):
            assert bool((buf[:G] == fill).all()) and bool((buf[-G:] == fill).all())
        return (img[G:G + n_img].view(B, h, w, c), dep[G:G + n_px].view(B, h, w), tri[G:G + n_px].view(B, h, w))

    img, dep, tri = run({"image", "depth", "tri_index"})
    assert bool(((tri >= -1) & (tri < tris.shape[0])).all())
    # per head: image / depth against the reference, tri_index against the model, with this head's own buffers
    for b in range(B):
        want_img, want_depth = ref_rasterize(verts[b], tris, colors, bg[b], reverse=True, depth0=depth0[b]) \
            if os.path.isfile(REF_SO) else raster_model.rasterize(verts[b], tris, colors, h, w, bg[b], depth0[b], True)[:2]
        _, _, want_tri = raster_model.rasterize(verts[b], tris, None, h, w, depth0=depth0[b])
        assert np.array_equal(img[b].cpu().numpy(), want_img), b
        assert np.array_equal(dep[b].cpu().numpy().view(np.uint32), want_depth.view(np.uint32)), b
        assert np.array_equal(tri[b].cpu().numpy(), want_tri), b
        bgpix = np.flip(want_tri < 0, 0)                  # image rows are flipped (reverse = 1)
        assert np.array_equal(img[b].cpu().numpy()[bgpix], bg[b][bgpix]), b
    assert bool((tri >= 0).any()) and bool((tri < 0).any())
    # without a depth buffer the z-test threshold is -1e8, so the subsets are compared on a depth buffer that starts there
    names = ("image", "depth", "tri_index")
    flat = np.full_like(depth0, -1e8)
    full = dict(zip(names, run(set(names), flat)))
    for r in range(3):
        for want in itertools.combinations(names, r):
            part = dict(zip(names, run(set(want), flat)))
            for k in want:
                assert torch.equal(part[k], full[k]), (want, k)


def test_zero_batch_and_zero_triangles(cuda_device):
    L = _lib()
    lib = L.load()
    dev = _dev()
    v = torch.zeros(2, 3, 3, device=dev)
    t = torch.zeros(0, 3, dtype=torch.int32, device=dev)
    key = torch.empty(2 * 8 * 8, dtype=torch.int64, device=dev)
    tri = torch.full((2, 8, 8), 5, dtype=torch.int32, device=dev)
    dep = torch.full((2, 8, 8), 3.0, device=dev)
    s = torch.cuda.current_stream(dev).cuda_stream
    before = L.launch_count()
    L.check(lib.dad3d_rasterize_batch(v.data_ptr(), 3, 0, t.data_ptr(), 0, None, 1, 8, 8, 0, 0, None, dep.data_ptr(),
                                      tri.data_ptr(), key.data_ptr(), s), "batch 0")
    assert bool((tri == 5).all())
    L.check(lib.dad3d_rasterize_batch(v.data_ptr(), 3, 2, t.data_ptr(), 0, None, 1, 8, 8, 0, 0, None, dep.data_ptr(),
                                      tri.data_ptr(), key.data_ptr(), s), "ntri 0")
    assert bool((tri == -1).all()) and bool((dep == 3.0).all())
    assert L.launch_count() == before


def test_invalid_arguments(cuda_device):
    L = _lib()
    lib = L.load()
    dev = _dev()
    v = torch.zeros(1, 3, 3, device=dev)
    t = torch.tensor([[0, 1, 2]], dtype=torch.int32, device=dev)
    col = torch.zeros(3, 3, device=dev)
    key = torch.empty(64, dtype=torch.int64, device=dev)
    out = torch.empty(64, dtype=torch.int32, device=dev)
    s = torch.cuda.current_stream(dev).cuda_stream
    good = [v.data_ptr(), 3, 1, t.data_ptr(), 1, col.data_ptr(), 3, 8, 8, 0, 0, None, None, out.data_ptr(), key.data_ptr(), s]
    L.check(lib.dad3d_rasterize_batch(*good), "valid call")
    torch.cuda.synchronize()
    before = L.launch_count()
    for i, bad in [(2, -1), (7, 65536), (14, None), (0, None), (3, None), (6, 0), (1, 0), (4, -1)]:
        args = list(good)
        args[i] = bad
        if i == 7:
            args[8] = 32768                              # h * w = 2^31
        assert lib.dad3d_rasterize_batch(*args) == -1, (i, bad)
        assert b"invalid argument" in lib.dad3d_last_error()
    img = torch.empty(64 * 3, dtype=torch.uint8, device=dev)
    args = list(good)
    args[5], args[11] = None, img.data_ptr()               # an image needs colours
    assert lib.dad3d_rasterize_batch(*args) == -1
    assert L.launch_count() == before
    from dad_3dheads_b200.rasterizer import rasterize_batch
    with pytest.raises(ValueError):
        rasterize_batch(v, torch.tensor([[0, 1, 3]], dtype=torch.int32, device=dev), height=8, width=8)


@needs_ref
def test_pncc_renderer_equals_reference_pncc(cuda_device):
    """PnccRenderer on decoded heads == the reference's own pncc() (inference/pncc_estimator.py, Sim3DR = its C++ rasteriser)
    with its own faces and colours on the same fp32 vertices, z negated as PNCCEstimator does."""
    from dad_3dheads_b200.head_mesh import HeadMesh
    from dad_3dheads_b200.rasterizer import PnccRenderer
    from oracle import ref_harness
    from oracle.flame_oracle import sample_params
    if not ref_harness.available():
        pytest.skip("reference harness unavailable")
    ref_harness.activate()
    import importlib
    pe = importlib.import_module("inference.pncc_estimator")
    import Sim3DR
    assert "ref_shims" in Sim3DR.__file__
    est = pe.PNCCEstimator()
    p = sample_params(5, seed=21)
    p[:, 409:411] *= 0.3
    p[:, 412] = torch.tensor([2.0, 1.0, 3.0, -0.8, 2.0])
    p[4, 409] = 1.0
    _, proj = HeadMesh(cuda_id=0).decode(p.to(_dev()), to_2d=False)
    out = PnccRenderer(_dev())(proj, 256)
    assert set(out) == {"pncc", "depth", "tri_index"} and out["pncc"].shape == (5, 256, 256, 3)
    faces = np.asarray(est.faces_wo_back_remapped)
    cover = []
    for b in range(5):
        v = proj[b].cpu().numpy().copy()
        v[:, 2] *= -1                                     # pncc_estimator.py:77
        want = pe.pncc(np.zeros((256, 256, 3), np.uint8), v, faces, est.colors, with_bg_flag=False)
        assert np.array_equal(out["pncc"][b].cpu().numpy(), want), b
        _, want_depth = ref_rasterize(v, faces, est.colors.astype(np.float32), np.zeros((256, 256, 3), np.uint8))
        assert np.array_equal(out["depth"][b].cpu().numpy().view(np.uint32), want_depth.view(np.uint32)), b
        _, _, want_tri = raster_model.rasterize(v, faces, None, 256, 256)
        assert np.array_equal(out["tri_index"][b].cpu().numpy(), want_tri), b
        cover.append((want_tri >= 0).mean())
    assert min(cover) > 0 and max(cover) > 0.05, cover


@pytest.fixture(scope="module")
def predictor(cuda_device):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


def test_predict_batch_render(predictor):
    from dad_3dheads_b200.rasterizer import PnccRenderer
    x = torch.randn(4, 3, 256, 256, generator=torch.Generator().manual_seed(5)).to(_dev())
    plain = predictor.predict_batch(x, to_2d=False)
    got = predictor.predict_batch(x, to_2d=False, render=("pncc", "depth", "tri_index"))
    for k, t in plain.items():
        assert torch.equal(got[k], t), k
    want = PnccRenderer(_dev())(got["projected_vertices"], 256)
    for k in ("pncc", "depth", "tri_index"):
        assert torch.equal(got[k], want[k]), k
    only = predictor.predict_batch(x, to_2d=False, render=("tri_index",))
    assert "pncc" not in only and "depth" not in only and torch.equal(only["tri_index"], want["tri_index"])
    with pytest.raises(ValueError):
        predictor.predict_batch(x, to_2d=True, render=("pncc",))
    with pytest.raises(ValueError):
        predictor.predict_batch(x, to_2d=False, render=("normals",))


def test_render_eager_graphed_and_stream_identical(predictor):
    keys = ("pncc", "depth", "tri_index")
    x = torch.randint(0, 256, (3, 300, 240, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6))
    eager = predictor.predict_batch(x.to(_dev()), to_2d=False, render=keys)
    graphed = predictor.predict_batch_graphed(x, to_2d=False, render=keys)
    graphed = {k: t.clone() for k, t in graphed.items()}
    plain = predictor.predict_batch_graphed(x, to_2d=False)
    assert "pncc" not in plain                            # render is part of the graph key
    stream = predictor.open_stream(tuple(x.shape), to_2d=False, render=keys, keys=("3dmm_params",) + keys)
    stream.submit(x.pin_memory())
    res = stream.collect()
    for k in keys:
        assert torch.equal(eager[k], graphed[k]), k
        assert res[k].is_pinned() and torch.equal(res[k], eager[k].cpu()), k
    assert torch.equal(res["3dmm_params"], eager["3dmm_params"].cpu())
