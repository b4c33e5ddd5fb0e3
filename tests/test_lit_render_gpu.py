"""-m gpu: the lit render (dad3d_light_batch, dad3d_render_lit, rasterizer.light_batch / render_lit / LitRenderer,
predict_batch(render=("lit",)) and frame_render=("lit", ...), compat Sim3DR.RenderPipeline).

The light is compared bit for bit with tests/lit_model.py using the correctly rounded power (pinned to the reference's
RenderPipeline by tests/test_lit_model_cpu.py), and images byte for byte with the reference's own C++ rasteriser
(oracle/_ref/libsim3dr_ref.so) given that light as colours."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import lighting_ref
from tests import lit_model as LM
from tests.test_lit_model_cpu import demo_head, designed_meshes, same_bits
from tests.test_raster_model_cpu import REF_SO, ref_rasterize

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not os.path.isfile(REF_SO), reason="oracle/_ref/libsim3dr_ref.so not built")
F = np.float32


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _faces():
    from dad_3dheads_b200.rasterizer import load_render_static
    return np.ascontiguousarray(load_render_static()["faces_wo_ears"][:, [0, 2, 1]])


def _heads(n, seed, scale=1.0, shift=(0.0, 0.0)):
    """n decoded FLAME heads in 256 x 256 pixels (z as decoded: the renderers negate it)."""
    from oracle.flame_oracle import FlameOracle, load_static, sample_params
    p = sample_params(n, seed=seed)
    p[:, 409:411] = 0.0
    p[:, 412] = 1.0
    v = FlameOracle(load_static(), image_size=256).reprojected_vertices(p, to_2d=False).numpy().astype(F)
    c = v[..., :2].mean(1, keepdims=True)
    v[..., :2] = (v[..., :2] - c) * F(scale) + np.asarray(shift, F)
    return np.ascontiguousarray(v, F)


def _neg(v):
    v = np.array(v, F, copy=True)
    v[..., 2] *= -1
    return v


# ------------------------------------------------------------------------------------------------------ light
@pytest.mark.parametrize("name", sorted(designed_meshes()))
def test_light_batch_designed_meshes(cuda_device, name):
    from dad_3dheads_b200.rasterizer import light_batch
    v, t, kw = designed_meshes()[name]
    got = light_batch(_t(v[None]), _t(t), lighting=kw)[0].cpu().numpy()
    assert same_bits(got, LM.light(v, t, kw)), name


def test_light_batch_real_heads_negate_z_and_guard_bands(cuda_device):
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.rasterizer import _adjacency, light_batch, lighting_struct
    v, t = _heads(5, 11, 1.7, (128, 128)), _faces()
    want = np.stack([LM.light(_neg(h), t) for h in v])
    got = light_batch(_t(v), _t(t), negate_z=True).cpu().numpy()
    assert same_bits(got, want)
    assert same_bits(light_batch(_t(_neg(v)), _t(t)).cpu().numpy(), want)
    # the raw entry writes exactly [B,nv,3] between NaN guard bands
    B, nv = v.shape[:2]
    tt = _t(t)
    off, adj = _adjacency(tt, nv)
    buf = torch.full((B * nv * 3 + 2048,), float("nan"), device=_dev())
    lib = _lib.load()
    _lib.check(lib.dad3d_light_batch(_t(v).data_ptr(), nv, B, tt.data_ptr(), off.data_ptr(), adj.data_ptr(), 1,
                                     lighting_struct(None), buf.data_ptr() + 1024 * 4, 0), "dad3d_light_batch")
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert np.isnan(b[:1024]).all() and np.isnan(b[-1024:]).all()
    assert same_bits(b[1024:-1024].reshape(B, nv, 3), want)


def test_light_batch_every_exponent(cuda_device):
    from dad_3dheads_b200.rasterizer import light_batch
    v, t = _heads(2, 12, 1.3, (100, 140)), _faces()
    for e in range(17):
        kw = dict(specular_exp=e, intensity_specular=0.6, view_pos=(0.5, -0.5, 3))
        got = light_batch(_t(v), _t(t), lighting=kw, negate_z=True).cpu().numpy()
        for b in range(2):
            assert same_bits(got[b], LM.light(_neg(v[b]), t, kw)), e


def test_light_batch_past_the_grid_limit(cuda_device):
    """70 000 small heads (more CTAs than one grid dimension takes): every sampled head equals the model."""
    from dad_3dheads_b200.rasterizer import light_batch
    B = 70_000
    g = np.random.default_rng(13)
    base = np.array([[0, 0, 0], [10, 0, 1], [0, 10, 2], [3, 3, 9]], F)
    t = np.array([[0, 1, 2], [0, 3, 1], [1, 3, 2], [2, 3, 0]], np.int32)
    v = (base[None] + g.uniform(-2, 2, (B, 4, 3))).astype(F)
    got = light_batch(_t(v), _t(t)).cpu().numpy()
    for b in np.r_[0, 1, 65_534, 65_535, 65_536, B - 1, g.integers(0, B, 200)]:
        assert same_bits(got[b], LM.light(v[b], t)), b


def test_argument_errors_launch_nothing(cuda_device):
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.rasterizer import LitRenderer, light_batch, lighting_struct, render_lit
    lib = _lib.load()
    v, t = _t(_heads(2, 1)), _t(_faces())
    light_batch(v, t)                                     # warm: bounds check and adjacency of t
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for e in (-1, 17, 2.5, True):
        with pytest.raises(ValueError):
            light_batch(v, t, lighting=dict(specular_exp=e))
        with pytest.raises(ValueError):
            LitRenderer(_dev(), specular_exp=e)
    with pytest.raises(ValueError):
        light_batch(v, t, lighting=dict(intensity_ambient=1e-50))
    with pytest.raises(ValueError):
        light_batch(v, t, lighting=dict(shininess=3))
    with pytest.raises(ValueError):
        render_lit(v, t, height=8, width=8, image_of_head=_t(np.zeros(2, np.int32)))
    L = lighting_struct(None)
    L.specular_exp = 17
    buf = torch.empty(1, device=_dev())
    assert lib.dad3d_light_batch(v.data_ptr(), 5023, 2, t.data_ptr(), buf.data_ptr(), buf.data_ptr(), 0, L, buf.data_ptr(),
                                 None) == -1
    L.specular_exp = 5
    assert lib.dad3d_light_batch(None, 5023, 2, t.data_ptr(), buf.data_ptr(), buf.data_ptr(), 0, L, buf.data_ptr(), None) == -1
    # (head, triangle) pairs beyond 2^32 - 2 with a map; the same sizes without one are accepted by that check
    p = buf.data_ptr()
    assert lib.dad3d_render_lit(p, 3, 70_000, p, 70_000, p, p, 0, L, p, 1, 8, 8, p, p, p, None) == -1
    assert b"2^32" in lib.dad3d_last_error()
    L.specular_exp = 99
    assert lib.dad3d_render_lit(p, 3, 1, p, 1, p, p, 0, L, None, 0, 8, 8, p, p, p, None) == -1
    torch.cuda.synchronize()
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------------------ images
def _want_images(v_neg, t, kw, H, W, bgs=None):
    out = []
    for b, h in enumerate(v_neg):
        bg = np.zeros((H, W, 3), np.uint8) if bgs is None else bgs[b]
        out.append(ref_rasterize(h, t, LM.light(h, t, kw), bg)[0])
    return np.stack(out)


@needs_ref
@pytest.mark.parametrize("H,W", [(256, 256), (200, 317)])
def test_lit_images_at_network_size(cuda_device, H, W):
    from dad_3dheads_b200.rasterizer import LitRenderer, render_lit
    t = _faces()
    v = _heads(4, 21, 2.5, (W / 2, H / 2))
    v[3] = v[2]
    v[1, :, :2] += 90                                     # partly outside
    want = _want_images(_neg(v), t, {}, H, W)
    got = render_lit(_t(v), _t(t), height=H, width=W, negate_z=True).cpu().numpy()
    assert np.array_equal(got, want)
    assert (want.reshape(4, -1, 3).any(-1).sum(1) > 1000).all()
    if H == W:
        r = LitRenderer(_dev())
        assert np.array_equal(r(_t(v), H)["lit"].cpu().numpy(), want)
    kw = dict(intensity_ambient=0.2, specular_exp=9, intensity_specular=0.5, light_pos=(2, 1, 4), color_directional=(1, .5, .2))
    bgs = np.random.default_rng(2).integers(0, 256, (4, H, W, 3), dtype=np.uint8)
    got = render_lit(_t(v), _t(t), height=H, width=W, negate_z=True, lighting=kw, image=_t(bgs)).cpu().numpy()
    assert np.array_equal(got, _want_images(_neg(v), t, kw, H, W, bgs))


def _union_want(v_neg, t, fo, n, H, W, frames=None, kw=None):
    """Per frame: the reference's rasteriser once on the union mesh of its heads (head order), each head's light as its
    colours, drawn over the frame or black."""
    nv = v_neg.shape[1]
    out = []
    for f in range(n):
        heads = np.flatnonzero(fo == f)
        bg = np.zeros((H, W, 3), np.uint8) if frames is None else frames[f]
        if len(heads) == 0:
            out.append(np.array(bg, copy=True))
            continue
        verts = v_neg[heads].reshape(-1, 3)
        tris = (t[None].astype(np.int64) + (np.arange(len(heads)) * nv)[:, None, None]).reshape(-1, 3)
        cols = np.concatenate([LM.light(v_neg[h], t, kw) for h in heads])
        out.append(ref_rasterize(verts, tris, cols, bg)[0])
    return np.stack(out)


@needs_ref
@pytest.mark.parametrize("H,W", [(480, 640), (1080, 1920)])
@pytest.mark.parametrize("with_frames", [False, True])
def test_lit_frames(cuda_device, H, W, with_frames):
    """Overlapping heads in both orders, an exact duplicate, heads mapped to -1 and to F (nothing drawn), a frame
    without heads; over black or over given frames."""
    from dad_3dheads_b200.rasterizer import LitRenderer
    t = _faces()
    n = 12
    g = np.random.default_rng(31)
    v = np.concatenate([_heads(1, 40 + i, g.uniform(0.8, 2.5), (g.uniform(0, W), g.uniform(0, H))) for i in range(n)])
    v[1] = v[0] + np.array([25, 10, 40], F)              # overlaps head 0, nearer after negation? both orders below
    v[2] = v[0] + np.array([-20, 5, -40], F)
    v[5] = v[4]                                          # duplicate: the earlier head wins every tie
    fo = np.array([0, 0, 0, 1, 2, 2, -1, 1, 4, 0, 1, 2], np.int32)
    frames = np.random.default_rng(3).integers(0, 256, (4, H, W, 3), dtype=np.uint8) if with_frames else None
    r = LitRenderer(_dev())
    got = r.render_frames(_t(v), _t(fo), 4, (H, W), frames=_t(frames) if with_frames else None)["lit"].cpu().numpy()
    want = _union_want(_neg(v), t, fo, 4, H, W, frames)
    assert np.array_equal(got, want)
    assert np.array_equal(got[3], frames[3] if with_frames else np.zeros((H, W, 3), np.uint8))


# ------------------------------------------------------------------------------------------------------ predictor
@pytest.fixture(scope="module")
def pred(cuda_device):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


@needs_ref
def test_predict_batch_render_lit_eager_graphed_stream(pred):
    from dad_3dheads_b200.rasterizer import LitRenderer
    x = torch.randn(6, 3, 256, 256, generator=torch.Generator().manual_seed(4)).to(_dev())
    eager = {k: v.clone() for k, v in pred.predict_batch(x, to_2d=False, render=("lit", "pncc")).items()}
    assert eager["lit"].shape == (6, 256, 256, 3) and "pncc" in eager
    only = pred.predict_batch(x, to_2d=False, render="lit")
    assert "pncc" not in only and torch.equal(only["lit"], eager["lit"])
    assert torch.equal(LitRenderer(_dev())(eager["projected_vertices"], 256)["lit"], eager["lit"])
    pv = eager["projected_vertices"].cpu().numpy()
    assert np.array_equal(eager["lit"][:2].cpu().numpy(), _want_images(_neg(pv[:2]), _faces(), {}, 256, 256))
    graphed = pred.predict_batch_graphed(x, to_2d=False, render=("lit", "pncc"))
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(graphed[k], eager[k]), k
    st = pred.open_stream(tuple(x.shape), dtype=torch.float32, to_2d=False, render=("lit",), keys=("lit",))
    st.submit(x.cpu().pin_memory())
    assert torch.equal(st.collect()["lit"], eager["lit"].cpu())


@needs_ref
def test_predict_batch_frame_lit_eager_graphed_stream(pred):
    from tests.test_frame_render_gpu import _frame_map, _steps
    F_, H, W, R = 3, 480, 640, 10
    steps = _steps(F_, H, W, R)
    kw = dict(extend=0.1, to_2d=False, frame_render=("lit", "pncc", "head_index"))
    want = [{k: v.clone() for k, v in pred.predict_batch(fr, boxes=b, frame_index=f, **kw).items()} for fr, b, f in steps]
    for (fr, b, f), w in zip(steps, want):
        assert w["frame_lit"].shape == (F_, H, W, 3)
        fo = _frame_map(w, f).cpu().numpy()
        pv = w["projected_vertices"].cpu().numpy()
        assert np.array_equal(w["frame_lit"].cpu().numpy(), _union_want(_neg(pv), _faces(), fo, F_, H, W, fr.numpy()))
        alone = pred.predict_batch(fr, boxes=b, frame_index=f, extend=0.1, to_2d=False, frame_render="lit")
        assert "frame_pncc" not in alone and torch.equal(alone["frame_lit"], w["frame_lit"])
        got = pred.predict_batch_graphed(fr, boxes=b, frame_index=f, **kw)
        torch.cuda.synchronize()
        assert set(got) == set(w)
        for k in w:
            assert torch.equal(got[k], w[k]), k
    keys = ("valid", "frame_lit", "frame_pncc")
    st = pred.open_stream((F_, H, W, 3), rois=R, keys=keys, depth=2, **kw)
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


# ------------------------------------------------------------------------------------------------------ compat
@needs_ref
@pytest.mark.skipif(not lighting_ref.available(), reason="oracle/_ref lighting.pyc not built")
def test_compat_render_pipeline_against_live_reference(cuda_device):
    import importlib.util
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compat", "Sim3DR")
    spec = importlib.util.spec_from_file_location("_compat_sim3dr", os.path.join(root, "__init__.py"),
                                                  submodule_search_locations=[root])
    compat = importlib.util.module_from_spec(spec)
    import sys
    sys.modules["_compat_sim3dr"] = compat
    spec.loader.exec_module(compat)
    ref = lighting_ref.load()
    v, t = demo_head(), _faces()
    frame = np.random.default_rng(8).integers(0, 256, (640, 420, 3), dtype=np.uint8)
    for kw in ({}, dict(specular_exp=3, intensity_specular=0.5, light_pos=(1, -1, 4))):
        bg_ref, bg_gpu = frame.copy(), frame.copy()
        want = ref.RenderPipeline(**kw)(v, t, bg_ref)
        rp = compat.RenderPipeline(**kw)
        got = rp(v, t, bg_gpu)
        assert got is bg_gpu and want is bg_ref
        light_ref = ref.RenderPipeline(**kw)
        # the pixels whose vertex lights differ between the host power and the correctly rounded one
        host_l, exact_l = LM.light(v, t, kw, pow=lambda a, e: a ** e), LM.light(v, t, kw)
        differ = ~np.all(host_l == exact_l, axis=1)
        _, _, tri = __import__("tests.raster_model", fromlist=["x"]).rasterize(v, t, None, 640, 420)
        touched = np.zeros(tri.shape, bool)
        cov = tri >= 0
        touched[cov] = differ[t[tri[cov]]].any(1)
        d = np.abs(got.astype(np.int32) - want.astype(np.int32)).max(-1)
        print(f"compat vs live reference {kw}: {int(differ.sum())} vertices with a different light, "
              f"{int(touched.sum())} pixels drawn from them, {int((d > 0).sum())} pixels differ, max {int(d.max())} level")
        assert (d[~touched] == 0).all() and d.max() <= 1
        assert light_ref.light_pos.shape == (1, 3) and rp.light_pos.shape == (1, 3)
    rp.update_light_pos((0, 1, 5))
    assert rp.light_pos.tolist() == [[0, 1, 5]]
    # texture: multiplied in place by the light, in its own dtype
    tex = np.random.default_rng(9).uniform(0, 1, v.shape)
    tex_ref = tex.copy()
    a, b = frame.copy(), frame.copy()
    ref.RenderPipeline()(v, t, a, tex_ref)
    compat.RenderPipeline()(v, t, b, tex)
    assert tex.dtype == np.float64 and np.abs(tex - tex_ref).max() <= 1e-7
    assert np.abs(a.astype(int) - b.astype(int)).max() <= 1
