"""-m "not gpu": tests/frame_render_model.py against the reference's own C++ rasteriser (oracle/_ref/libsim3dr_ref.so).

The union-mesh model of a frame must equal, bit for bit in image and depth, the reference called once per head in head
order with the image and depth buffer carried over (what a caller of the reference writes to draw several heads into one
frame).  Its split of the winning union triangle into (head, triangle) is then checked on designed cases: the nearer head
wins in either order, an exact duplicate goes to the first head, a +-0 depth tie to the earlier head, heads partly or fully
outside the frame, and a frame without heads."""
import os

import numpy as np
import pytest

from tests import frame_render_model as FM
from tests import raster_model
from tests.test_raster_model_cpu import REF_SO, flame_head, random_mesh, ref_rasterize, zero_sign_mesh

pytestmark = pytest.mark.skipif(not os.path.isfile(REF_SO), reason="oracle/_ref/libsim3dr_ref.so not built")


def carried(vertices, triangles, colors, h, w):
    """The reference, once per head in head order, with the image and depth buffer carried from one call to the next."""
    img = np.zeros((h, w, colors.shape[1]), np.uint8)
    depth = None
    for v in vertices:
        img, depth = ref_rasterize(v, triangles, colors, img, depth0=depth)
    if depth is None:
        depth = np.full((h, w), -1e8, np.float32)
    return img, depth


def _shift(v, dx, dy, dz=0.0):
    return (v + np.array([dx, dy, dz], np.float32)).astype(np.float32)


def _check_against_reference(heads, t, h, w, seed=0):
    col = np.random.default_rng(seed).random((heads.shape[1], 3)).astype(np.float32)
    want_img, want_depth = carried(heads, t, col, h, w)
    img, depth, tri, head = FM.render_frame(heads, t, col, h, w)
    assert np.array_equal(img, want_img)
    assert np.array_equal(depth.view(np.uint32), want_depth.view(np.uint32))
    assert np.array_equal(tri >= 0, want_depth != np.float32(-1e8)) and np.array_equal(tri >= 0, head >= 0)
    # the union mesh through the reference in one call is the same computation
    uv, ut, uc = FM.union_mesh(heads, t, col)
    one_img, one_depth = ref_rasterize(uv, ut, uc, np.zeros((h, w, 3), np.uint8))
    assert np.array_equal(one_img, want_img) and np.array_equal(one_depth.view(np.uint32), want_depth.view(np.uint32))
    return tri, head, depth


def test_union_equals_carried_reference_on_random_meshes():
    v, t = random_mesh(4, size=40)
    heads = np.stack([v, _shift(v, 3, -2), _shift(v, -4, 5, 1), v])          # overlapping, integer shifts, a duplicate
    _check_against_reference(heads, t, 44, 47)


@pytest.mark.parametrize("order", [(0, 1), (1, 0)])
def test_nearer_head_wins_in_either_order(order):
    v, t = flame_head(5, 160)
    near, far = _shift(v, 10, 0, 500.0), _shift(v, 0, 0, -500.0)            # depth = z (already negated): larger wins
    pair = [near, far]
    heads = np.stack([pair[i] for i in order])
    tri, head, _ = _check_against_reference(heads, t, 160, 180)
    _, _, tri_near = raster_model.rasterize(near, t, None, 160, 180)
    near_head = order.index(0)
    assert np.array_equal(head[tri_near >= 0], np.full((tri_near >= 0).sum(), near_head))
    assert np.array_equal(tri[tri_near >= 0], tri_near[tri_near >= 0])
    assert (head == 1 - near_head).any()                                    # the far head shows where the near one does not


def test_exact_duplicate_goes_to_the_first_head():
    v, t = flame_head(6, 128)
    heads = np.stack([_shift(v, 20, 0), v, v, _shift(v, -30, 10)])
    tri, head, _ = _check_against_reference(heads, t, 128, 128)
    assert not (head == 2).any() and (head == 1).any()
    _, _, tri_one = raster_model.rasterize(v, t, None, 128, 128)
    only = (tri_one >= 0) & (head != 0) & (head != 3)
    assert np.array_equal(head[only], np.ones(only.sum(), np.int32)) and np.array_equal(tri[only], tri_one[only])


@pytest.mark.parametrize("first_sign", [-0.0, 0.0])
def test_signed_zero_tie_between_heads(first_sign):
    v, t = zero_sign_mesh()
    a = v[:3].copy()
    a[:, 2] = first_sign
    b = v[:3].copy()
    b[:, 2] = -first_sign
    tri, head, depth = _check_against_reference(np.stack([a, b]), t[:1], 24, 24)
    assert set(np.unique(head)) == {-1, 0} and set(np.unique(tri)) == {-1, 0}
    assert np.array_equal(np.signbit(depth[head == 0]), np.full((head == 0).sum(), np.signbit(np.float32(first_sign))))


def test_heads_partly_and_fully_outside_the_frame():
    v, t = flame_head(7, 120)
    heads = np.stack([_shift(v, -60, 0), _shift(v, 500, 30), _shift(v, 40, 70), _shift(v, 0, -400)])
    tri, head, _ = _check_against_reference(heads, t, 120, 150)
    assert set(np.unique(head)) == {-1, 0, 2}


def test_empty_frame():
    v, t = random_mesh(8)
    col = np.random.default_rng(8).random((v.shape[0], 3)).astype(np.float32)
    img, depth, tri, head = FM.render_frame(np.zeros((0,) + v.shape, np.float32), t, col, 20, 30)
    want_img, want_depth = carried(np.zeros((0,) + v.shape, np.float32), t, col, 20, 30)
    assert np.array_equal(img, want_img) and np.array_equal(depth.view(np.uint32), want_depth.view(np.uint32))
    assert (tri == -1).all() and (head == -1).all()


def test_render_frames_groups_heads_by_frame():
    """render_frames: head numbers are global, out-of-range entries draw nothing, and each frame is its own render_frame."""
    v, t = random_mesh(9, size=30)
    heads = np.stack([_shift(v, i % 3, -(i % 2)) for i in range(6)])
    fo = np.array([1, -1, 1, 0, 3, 1])
    col = np.random.default_rng(9).random((v.shape[0], 3)).astype(np.float32)
    img, depth, tri, head = FM.render_frames(heads, t, col, fo, 3, 32, 32)
    assert img.shape == (3, 32, 32, 3) and (head[2] == -1).all() and (tri[2] == -1).all()
    for f, members in ((0, [3]), (1, [0, 2, 5])):
        want = carried(heads[members], t, col, 32, 32)
        assert np.array_equal(img[f], want[0]) and np.array_equal(depth[f].view(np.uint32), want[1].view(np.uint32))
        assert set(np.unique(head[f])) <= {-1, *members}
