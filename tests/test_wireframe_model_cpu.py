"""CPU: tests/wireframe_model.py pinned to the cv2 binary (4.13.0) and to the reference's own demo_utils.draw_mesh.

These are the rules csrc/overlay.cu's wireframe kernels restate; tests/test_wireframe_gpu.py compares the kernels with this
model."""
import numpy as np
import pytest
import torch

from tests import wireframe_model as M

cv2 = pytest.importorskip("cv2")

from oracle import ref_harness  # noqa: E402

needs_ref = pytest.mark.skipif(not ref_harness.available(), reason="reference tree not available")
KINDS = M.WIREFRAME_KINDS


@pytest.fixture(scope="module")
def static():
    from dad_3dheads_b200.flame import load_flame_static
    return load_flame_static()


def _cv2_line(img, p, q, color=M.EDGE_COLOR):
    cv2.line(img, (int(p[0]), int(p[1])), (int(q[0]), int(q[1])), color, 1, cv2.LINE_AA)


def test_cv2_version():
    assert cv2.__version__.startswith("4.13."), cv2.__version__


def test_every_line_in_a_window_across_the_border():
    """Both ends anywhere in a window reaching 3 px past every border and corner of a 7 x 5 image."""
    H, W = 5, 7
    bg = np.random.default_rng(0).integers(0, 256, (H, W, 3), dtype=np.uint8)
    pts = [(x, y) for x in range(-3, W + 3) for y in range(-3, H + 3)]
    bad = []
    for p in pts:
        for q in pts:
            a, b = bg.copy(), bg.copy()
            _cv2_line(a, p, q)
            M.line_aa(b, p, q)
            if not np.array_equal(a, b):
                bad.append((p, q))
    assert not bad, (len(bad), bad[:5])


@pytest.mark.parametrize("reach", [10 ** 6, (1 << 31) - 1])
def test_long_random_lines(reach):
    """Ends out to +-1e6 and close to +-2^31, where clipLine's fp64 divisions decide the first and last pixels."""
    g = np.random.default_rng(reach % 1000)
    for _ in range(400):
        H, W = int(g.integers(1, 200)), int(g.integers(1, 200))
        bg = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
        p = [int(v) for v in g.integers(-reach, reach, 4, endpoint=True)]
        if g.random() < 0.5:                                   # one end inside
            p[0], p[1] = int(g.integers(0, W)), int(g.integers(0, H))
        a, b = bg.copy(), bg.copy()
        _cv2_line(a, p[:2], p[2:])
        M.line_aa(b, p[:2], p[2:])
        assert np.array_equal(a, b), (H, W, p)


def test_overlapping_line_sequences_in_order():
    """2-300 overlapping lines drawn one after the other: the blends of one pixel in drawing order."""
    g = np.random.default_rng(3)
    for n in (2, 3, 7, 40, 300):
        for _ in range(4):
            H, W = int(g.integers(9, 40)), int(g.integers(9, 40))
            bg = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
            lines = g.integers(-8, max(H, W) + 8, (n, 4))
            a = bg.copy()
            for l in lines:
                _cv2_line(a, l[:2], l[2:])
            xs, ys, al = [], [], []
            for l in lines:
                x, y, s = M.line_aa_stamps(W, H, l[:2], l[2:])
                xs.append(x), ys.append(y), al.append(s)
            b = bg.copy()
            M.apply_stamps(b, np.concatenate(xs), np.concatenate(ys), np.concatenate(al))
            assert np.array_equal(a, b), n


def test_double_blend_for_every_background():
    """A touched pixel of a line equals the blend applied twice, for all 256 backgrounds, and never once."""
    for c in (0, 39, 255):
        col = (c, c, c)
        once_ok = 0
        for v in range(256):
            img = np.full((9, 17, 3), v, np.uint8)
            _cv2_line(img, (1, 2), (15, 6), col)
            x, y, a = M.line_aa_stamps(17, 9, (1, 2), (15, 6))
            assert np.array_equal(img[y, x, 0], M.blend(np.full(len(a), v), c, a)), (c, v)
            once = M.blend(np.full(len(a), v), c, a, twice=False)
            once_ok += np.array_equal(img[y, x, 0], once)
        assert once_ok < 256, c


# ----------------------------------------------------------------------------------------------- edge tables
@needs_ref
@pytest.mark.parametrize("kind", KINDS)
def test_derived_edge_tables_are_the_reference_files(static, kind):
    import os
    from dad_3dheads_b200 import overlay as O
    ref_harness.activate()
    sub = "head" if kind == "head_mesh" else "face"
    want = np.load(os.path.join(ref_harness._active_root, "model_training/model/static/flame_indices", f"{sub}_edges.npy"))
    got = M.subset_edges(static, kind)
    assert np.array_equal(got, want)
    assert np.array_equal(O.mesh_edges(static["faces"], static[O.MESH_VERTICES[kind]]), want)
    assert not np.array_equal(M.subset_edges(static, kind, "flame_indices_head"), want)


# ----------------------------------------------------------------------------------------------- against draw_mesh
def _heads(static, H, W, seed, ncomp=2):
    """Template heads of 20, 90 and 300 px, one across the left and top border, one across the right and bottom, and a
    random cloud."""
    g = np.random.default_rng(seed)
    heads = [M.template_head(static, g.uniform(0, W - 20), g.uniform(0, H - 20), 20, ncomp),
             M.template_head(static, g.uniform(0, W / 2), g.uniform(0, H / 2), 90, ncomp),
             M.template_head(static, -60.5, -40.25, 300, ncomp),
             M.template_head(static, W - 70.0, H - 55.0, 160, ncomp)]
    cloud = np.zeros((len(heads[0]), ncomp), np.float32)
    cloud[:, :2] = g.random((len(cloud), 2)) * [W + 80, H + 80] - 40
    heads.append(cloud)
    return np.stack(heads)


def _draw_mesh_ref(du, img, head, kind):
    """demo_utils.draw_mesh on a copy of img; img itself when cv2 raises (draw_mesh has no output)."""
    try:
        return du.draw_mesh({"projected_vertices": torch.from_numpy(head[None, :, :2].copy())}, img,
                            "head" if kind == "head_mesh" else "face")
    except cv2.error:
        return img


@needs_ref
@pytest.mark.parametrize("kind", KINDS)
def test_draw_mesh_equals_the_model(static, kind):
    ref_harness.activate()
    import demo_utils as du
    H, W = 241, 317
    g = np.random.default_rng(5)
    frame = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    heads = _heads(static, H, W, 6)
    heads[1, static["flame_indices_head"][0]] = np.nan        # a vertex outside both subsets: both still draw
    edges = M.subset_edges(static, kind)
    want = frame.copy()
    for r in range(len(heads)):
        want = _draw_mesh_ref(du, want, heads[r], kind)
    got = M.wireframe_frames(frame[None], np.zeros(len(heads), int), np.ones(len(heads), bool), heads, edges)[0]
    assert np.array_equal(got, want)
    assert not np.array_equal(got, frame)


@needs_ref
def test_points_cv2_refuses_blank_only_their_subset(static):
    """A NaN on an ear vertex blanks head_mesh but not face_mesh; beyond int32 blanks both; inf blanks the subset."""
    ref_harness.activate()
    import demo_utils as du
    H, W = 120, 160
    frame = np.random.default_rng(1).integers(0, 256, (H, W, 3), dtype=np.uint8)
    head = M.template_head(static, 10, 5, 100)
    ear = np.setdiff1d(static["flame_indices_face_w_ears"], static["flame_indices_face"])
    ear = int(np.intersect1d(ear, np.unique(M.subset_edges(static, "head_mesh")))[0])
    face = int(np.unique(M.subset_edges(static, "face_mesh"))[0])
    cases = {"ear_nan": (ear, np.nan, (False, True)), "face_inf": (face, np.inf, (False, False)),
             "face_far": (face, 3e9, (False, False)), "face_just_fits": (face, -2147483648.5, (True, True))}
    for name, (v, val, draws) in cases.items():
        h = head.copy()
        h[v, 0] = val
        for kind, d in zip(KINDS, draws):
            want = _draw_mesh_ref(du, frame.copy(), h, kind)
            got = M.wireframe_frames(frame[None], [0], [True], h[None], M.subset_edges(static, kind))[0]
            assert np.array_equal(got, want), (name, kind)
            assert (not np.array_equal(got, frame)) == d, (name, kind)


# ----------------------------------------------------------------------------------------------- modelled errors
MUTATIONS = ("single_blend", "no_half", "reversed_edges", "swapped_boxes", "no_clip", "head_on_flame_indices_head")


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_every_modelled_error_changes_a_compared_frame(static, mutation):
    """Each error, made in the model, changes a frame of the scene the GPU tests compare."""
    H, W = 241, 317
    frames = np.random.default_rng(8).integers(0, 256, (1, H, W, 3), dtype=np.uint8)
    heads = _heads(static, H, W, 9)[:4]                       # the cloud's many blends would saturate the swap away
    R = len(heads)
    edges = M.subset_edges(static, "head_mesh")
    right = M.wireframe_frames(frames, np.zeros(R, int), np.ones(R, bool), heads, edges)
    kw = {}
    order = None
    if mutation == "single_blend":
        kw["twice"] = False
    elif mutation == "no_half":
        kw["half"] = 0
    elif mutation == "reversed_edges":
        edges = edges[::-1]
    elif mutation == "swapped_boxes":
        order = [1, 0] + list(range(2, R))
        heads[1] = M.template_head(static, 5, 5, 60)           # overlapping box 0's head
        heads[0] = M.template_head(static, 8, 3, 60)
        right = M.wireframe_frames(frames, np.zeros(R, int), np.ones(R, bool), heads, edges)
    elif mutation == "no_clip":
        kw["clip"] = False
    else:
        edges = M.subset_edges(static, "head_mesh", "flame_indices_head")
    wrong = M.wireframe_frames(frames, np.zeros(R, int), np.ones(R, bool), heads, edges, box_order=order, **kw)
    assert not np.array_equal(wrong, right), mutation
