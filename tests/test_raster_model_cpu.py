"""-m "not gpu": tests/raster_model.py against the reference's own C++ rasteriser (Sim3DR/lib/rasterize_kernel.cpp, compiled
unmodified into oracle/_ref/libsim3dr_ref.so).  Image bytes and depth bits must be identical on designed cases before the
model's third output, the winning triangle, is used to check the GPU's tri_index."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import raster_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libsim3dr_ref.so")
pytestmark = pytest.mark.skipif(not os.path.isfile(REF_SO), reason="oracle/_ref/libsim3dr_ref.so not built")


def ref_rasterize(v, t, c, bg, reverse=False, depth0=None):
    lib = C.CDLL(REF_SO)
    lib.sim3dr_ref_rasterize.argtypes = [C.c_void_p] * 5 + [C.c_int] * 4 + [C.c_float, C.c_int]
    h, w, ch = bg.shape
    img = np.array(bg, np.uint8, copy=True)
    depth = np.full((h, w), -1e8, np.float32) if depth0 is None else np.array(depth0, np.float32, copy=True)
    v, t, c = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(t, np.int32), np.ascontiguousarray(c, np.float32)
    lib.sim3dr_ref_rasterize(img.ctypes.data, v.ctypes.data, t.ctypes.data, c.ctypes.data, depth.ctypes.data, t.shape[0], h, w,
                             ch, 1.0, 1 if reverse else 0)
    return img, depth


def ties_mesh():
    """The 15-vertex case of test_rasterizer_gpu.py: coplanar duplicates (lowest index wins), a zero-area triangle, one
    outside the image, and an ordinary one."""
    v = np.array([[2, 2, 5], [30, 3, 5], [4, 28, 5], [2, 2, 5], [30, 3, 5], [4, 28, 5], [10, 10, 1], [10, 10, 1], [10, 10, 1],
                  [-50, -50, 9], [-40, -50, 9], [-50, -40, 9], [5, 5, 7], [20, 6, 2], [6, 22, 9]], np.float32)
    t = np.array([[3, 4, 5], [0, 1, 2], [6, 7, 8], [9, 10, 11], [12, 13, 14]], np.int32)
    return v, t


def zero_sign_mesh():
    """Two overlapping triangles whose depth is -0 (the first) and +0 (the second) everywhere: the reference's strict
    z-test keeps the first."""
    v = np.array([[1, 1, -0.0], [20, 2, -0.0], [3, 20, -0.0], [1, 1, 0.0], [20, 2, 0.0], [3, 20, 0.0]], np.float32)
    return v, np.array([[0, 1, 2], [3, 4, 5]], np.int32)


def random_mesh(seed, nv=60, ntri=120, size=40):
    """Overlapping random triangles, with a few depths made equal so that exact ties occur."""
    g = np.random.default_rng(seed)
    v = np.c_[g.uniform(-5, size + 5, (nv, 2)), g.integers(-3, 4, nv)].astype(np.float32)
    return v, g.integers(0, nv, (ntri, 3)).astype(np.int32)


def flame_head(seed, size):
    from dad_3dheads_b200.flame import load_flame_static
    from oracle.flame_oracle import FlameOracle, sample_params
    st = load_flame_static()
    p = sample_params(1, seed=seed)
    p[:, 409:411] *= 0.3
    p[:, 412] = 2.0                                       # three times the unit scale: a head of about half the image
    v = FlameOracle(st, image_size=size).reprojected_vertices(p, to_2d=False)[0].numpy().astype(np.float32)
    v[:, 2] *= -1
    return v, st["faces"].astype(np.int32)


CASES = {
    "ties": (ties_mesh, 32, 32),
    "zero_sign": (zero_sign_mesh, 24, 24),
    "random0": (lambda: random_mesh(0), 40, 45),
    "random1": (lambda: random_mesh(1, ntri=300), 40, 40),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("c", [1, 3])
def test_model_matches_reference(case, reverse, c):
    make, h, w = CASES[case]
    v, t = make()
    g = np.random.default_rng(len(case) + c)
    col = g.random((v.shape[0], c)).astype(np.float32)
    bg = g.integers(0, 256, (h, w, c), dtype=np.uint8)
    want_img, want_depth = ref_rasterize(v, t, col, bg, reverse)
    img, depth, tri = raster_model.rasterize(v, t, col, h, w, image=bg, reverse=reverse)
    assert np.array_equal(img, want_img)
    assert np.array_equal(depth.view(np.uint32), want_depth.view(np.uint32))
    assert np.array_equal(tri >= 0, want_depth != np.float32(-1e8))


def test_model_winners_on_designed_cases():
    _, _, tri = raster_model.rasterize(*ties_mesh(), None, 32, 32)
    assert set(np.unique(tri)) == {-1, 0, 4}              # triangle 1 duplicates 0 at equal depth and never wins
    _, depth, tri = raster_model.rasterize(*zero_sign_mesh(), None, 24, 24)
    assert set(np.unique(tri)) == {-1, 0} and np.signbit(depth[tri == 0]).all()


def test_model_matches_reference_with_initial_depth():
    v, t = random_mesh(2)
    g = np.random.default_rng(2)
    depth0 = g.uniform(-2, 2, (40, 40)).astype(np.float32)
    col = g.random((v.shape[0], 3)).astype(np.float32)
    want_img, want_depth = ref_rasterize(v, t, col, np.zeros((40, 40, 3), np.uint8), depth0=depth0)
    img, depth, _ = raster_model.rasterize(v, t, col, 40, 40, depth0=depth0)
    assert np.array_equal(img, want_img) and np.array_equal(depth.view(np.uint32), want_depth.view(np.uint32))


@pytest.mark.parametrize("size,reverse", [(256, False), (200, True)])
def test_model_matches_reference_on_a_head(size, reverse):
    v, t = flame_head(3, size)
    col = np.random.default_rng(3).random((v.shape[0], 3)).astype(np.float32)
    want_img, want_depth = ref_rasterize(v, t, col, np.zeros((size, size + 17, 3), np.uint8), reverse)
    img, depth, tri = raster_model.rasterize(v, t, col, size, size + 17, reverse=reverse)
    assert (tri >= 0).mean() > 0.05
    assert np.array_equal(img, want_img) and np.array_equal(depth.view(np.uint32), want_depth.view(np.uint32))
