"""-m "not gpu": the exact model of csrc/uv_texture.cu (tests/uv_model.py) against the reference's own
``UVTextureCreator._compute_texture_map`` run live on a psbody ``Mesh`` restated in tests/psbody_mesh.py, byte for byte; the restricted table loader; the
faces the kernels use; the restated normals against an independent fp64 computation."""
import os
import pickle

import numpy as np
import pytest

from dad_3dheads_b200.flame import load_flame_static
from dad_3dheads_b200.uv_texture import compact_table, faces_by_vertex, read_table
from oracle import ref_harness as R
from tests import uv_model as M

TABLE = M.reference_table_path()
needs_table = pytest.mark.skipif(TABLE is None, reason="the reference's inference/texture_data.npy is not available")
FACES = load_flame_static()["faces"]


@pytest.fixture(scope="module")
def table():
    return read_table(TABLE)


@pytest.fixture(scope="module")
def compact(table):
    return compact_table(table)


def _model(v, frame, compact):
    S, texel, vids, bary = compact
    row, col = faces_by_vertex(FACES, 5023)
    nz = M.vertex_normals_z(v, FACES, row, col)
    return M.texture(v, nz, frame, texel, vids, bary, S)


@needs_table
@pytest.mark.parametrize("case", ["frontal", "rough_normals", "yaw_plus_85", "yaw_minus_88", "facing_away", "partly_off_image",
                                  "straddles_0", "straddles_W_H", "half_ties", "nonfinite", "huge_fp64", "frame_1x1"])
def test_model_equals_the_live_reference(case, table, compact):
    v, frame = M.designed_heads(FACES, fp64=True)[case]
    want = M.reference_texture_map(frame, v, FACES, table)
    got = _model(v, frame, compact)
    assert want.dtype == np.uint8 and want.shape == (512, 512, 3)
    assert np.array_equal(got, want), (case, int((got != want).any(-1).sum()))
    written = int(want.any(-1).sum())
    if case in ("frontal", "partly_off_image", "straddles_0", "straddles_W_H", "half_ties", "yaw_plus_85"):
        assert written > 1000, written
    if case == "frame_1x1":
        assert written == 0                                          # no pixel is strictly inside (0, 1) x (0, 1)


@needs_table
def test_designed_cases_reach_their_edges(compact):
    """The designed heads exercise what they are named for: exact .5 ties, texels on row/column 0 and W-1 / H-1
    rejected or kept by the strict bound, normals whose value depends on the order of the face sum."""
    S, texel, vids, bary = compact
    heads = M.designed_heads(FACES)
    row, col = faces_by_vertex(FACES, 5023)
    desc = col.copy()
    for i in range(5023):
        desc[row[i]:row[i + 1]] = col[row[i]:row[i + 1]][::-1]
    v = heads["rough_normals"][0]
    assert (M.vertex_normals_z(v, FACES, row, col) != M.vertex_normals_z(v, FACES, row, desc)).sum() > 100
    v = heads["half_ties"][0].astype(np.float64)
    px = (v[vids[:, 0], 0] * bary[:, 0] + v[vids[:, 1], 0] * bary[:, 1]) + v[vids[:, 2], 0] * bary[:, 2]
    assert ((px - np.floor(px)) == 0.5).sum() > 100
    for name, edge in (("straddles_0", 0), ("straddles_W_H", None)):
        v, frame = heads[name]
        H, W = frame.shape[:2]
        v = v.astype(np.float64)
        x = np.rint((v[vids[:, 0], 0] * bary[:, 0] + v[vids[:, 1], 0] * bary[:, 1]) + v[vids[:, 2], 0] * bary[:, 2])
        if edge == 0:
            assert (x == 0).sum() > 0 and (x == 1).sum() > 0
        else:
            assert (x == W).sum() > 0 and (x == W - 1).sum() > 0


def test_rint_bound_equals_astype_int_bound():
    """Comparing the rounded doubles (the kernel) equals the reference's comparisons on ``.astype(int)``, for NaN, the
    infinities, magnitudes >= 2^63 and the values around 0 and W."""
    W = 7
    xs = np.array([np.nan, np.inf, -np.inf, 1e300, -1e300, 2.0 ** 63, -2.0 ** 63, 2.0 ** 64, -0.5, 0.0, 0.49, 0.5, 0.51,
                   1.0, 6.49, 6.5, 6.51, 7.0, 7.5, -1.5])
    r = np.round(xs, 0)
    with np.errstate(invalid="ignore"):
        as_int = r.astype(int)
        kernel = (r > 0) & (r < W)
    assert np.array_equal(kernel, (as_int > 0) & (as_int < W))
    assert np.array_equal(np.rint(xs), r, equal_nan=True)


@needs_table
def test_loader_reads_the_real_file(table, compact):
    S, texel, vids, bary = compact
    assert S == 512 and texel.shape == (237456,) and vids.shape == (237456, 3) and bary.dtype == np.float64
    ids = table["valid_pixel_ids"]
    want = table["y_coords"][ids].astype(int) * S + table["x_coords"][ids].astype(int)
    assert np.array_equal(texel, want)
    assert np.array_equal(vids, table["valid_pixel_3d_faces"].astype(np.int64))
    assert np.array_equal(bary, table["valid_pixel_b_coords"])
    assert np.unique(texel).size == texel.size and vids.max() < 5023


def _save(path, obj):
    arr = np.empty((), dtype=object)
    arr[()] = obj
    np.save(path, arr, allow_pickle=True)                          # writing only: the loader under test never unpickles freely


def _small_table(n=4, S=8):
    x = np.arange(S * S, dtype=np.float64) % S + 0.5
    y = np.arange(S * S, dtype=np.float64) // S + 0.5
    ids = np.arange(n, dtype=np.int64) * 3
    return {"img_size": S, "x_coords": x, "y_coords": y, "valid_pixel_ids": ids,
            "valid_pixel_3d_faces": np.tile(np.array([0, 1, 2], dtype=np.uint32), (n, 1)),
            "valid_pixel_b_coords": np.full((n, 3), 1.0 / 3.0)}


def test_loader_round_trip_and_refusals(tmp_path):
    d = _small_table()
    p = tmp_path / "ok.npy"
    _save(p, d)
    got = read_table(str(p))
    assert all(np.array_equal(got[k], d[k]) for k in d)
    S, texel, vids, bary = compact_table(got)
    assert S == 8 and texel.tolist() == [0, 3, 6, 9 + 0] and vids.dtype == np.int32

    import collections
    bad = tmp_path / "foreign.npy"
    _save(bad, collections.OrderedDict(d))                          # a global outside the dict / ndarray / dtype set
    with pytest.raises(pickle.UnpicklingError, match="not allowed"):
        read_table(str(bad))

    class Evil:
        def __reduce__(self):
            return (os.system, ("echo unsafe",))
    evil = tmp_path / "evil.npy"
    _save(evil, {**d, "x": Evil()})
    with pytest.raises(pickle.UnpicklingError, match="not allowed"):
        read_table(str(evil))
    plain = tmp_path / "plain.npy"
    np.save(plain, np.zeros(3))
    with pytest.raises(ValueError, match="0-d object array"):
        read_table(str(plain))


@pytest.mark.parametrize("edit, match", [
    (lambda d: d["valid_pixel_ids"].__setitem__(1, 0), "duplicate texels"),
    (lambda d: d["x_coords"].__setitem__(3, 8.5), "outside the 8x8 image"),
    (lambda d: d["y_coords"].__setitem__(3, -0.5 - 1.0), "outside the 8x8 image"),
    (lambda d: d["valid_pixel_3d_faces"].__setitem__((2, 1), 5023), "vertex ids outside"),
    (lambda d: d["valid_pixel_ids"].__setitem__(0, 64), "outside x_coords"),
    (lambda d: d.pop("valid_pixel_b_coords"), "missing"),
])
def test_compaction_rejects(edit, match):
    d = _small_table()
    edit(d)
    with pytest.raises(ValueError, match=match):
        compact_table(d)


@pytest.mark.skipif(R.root() is None or not os.path.isfile(os.path.join(R.root() or "", "inference", "generic_model.pkl")),
                    reason="the reference's inference/generic_model.pkl is not available")
def test_packed_faces_are_generic_model_faces():
    from dad_3dheads_b200.flame_assets import load_pickle
    f = np.asarray(load_pickle(os.path.join(R.root(), "inference", "generic_model.pkl"))["f"])
    assert f.shape == FACES.shape and np.array_equal(f.astype(np.int64), FACES.astype(np.int64))


def test_faces_by_vertex_is_the_restated_csr():
    from tests.psbody_mesh import Mesh
    m = Mesh(np.zeros((5023, 3)), FACES)
    csr = m.faces_by_vertex(as_sparse_matrix=True)
    row, col = faces_by_vertex(FACES, 5023)
    assert np.array_equal(csr.indptr, row) and np.array_equal(csr.indices, col)
    assert (csr.data == 1.0).all()


def _icosphere():
    t = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                  [6, 2, 10], [8, 6, 7], [9, 8, 1]])
    return v, f


def test_restated_normals_against_an_independent_fp64_computation():
    """Closed, outward-wound icosahedron (scaled, shifted, one loose vertex): unit normals pointing away from the centre,
    equal to an np.add.at computation within round-off; the model's z equals the restatement's bit for bit."""
    from tests.psbody_mesh import Mesh
    v, f = _icosphere()
    v = np.vstack([v * 3.0 + [1.0, -2.0, 0.5], [[9.0, 9.0, 9.0]]])       # vertex 12 is in no face: normal 0
    n = Mesh(v, f).estimate_vertex_normals()
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    acc = np.zeros_like(v)
    for k in range(3):
        np.add.at(acc, f[:, k], fn)
    lens = np.linalg.norm(acc, axis=1)
    want = acc / np.where(lens == 0, 1.0, lens)[:, None]
    assert np.allclose(n, want, rtol=0, atol=1e-14)
    assert np.allclose(np.linalg.norm(n[:12], axis=1), 1.0, atol=1e-14) and (n[12] == 0).all()
    assert ((n[:12] * (v[:12] - [1.0, -2.0, 0.5])).sum(1) > 0).all()
    row, col = faces_by_vertex(f, 13)
    assert np.array_equal(M.vertex_normals_z(v, f, row, col), n[:, 2])


def test_model_normals_count_a_repeated_vertex_twice():
    """A face that lists a vertex twice adds its normal twice (the CSR's summed entry), in the model as in the restatement."""
    from tests.psbody_mesh import Mesh
    rng = np.random.default_rng(3)
    v = rng.standard_normal((6, 3))
    f = np.array([[0, 1, 2], [2, 3, 2], [3, 4, 5], [0, 5, 1]])
    row, col = faces_by_vertex(f, 6)
    assert np.array_equal(M.vertex_normals_z(v, f, row, col), Mesh(v, f).estimate_vertex_normals()[:, 2])


def test_step_options_uv_texture():
    """predict_batch(uv_texture=) is checked in StepOptions: it needs boxes and to_2d=False; a path is kept as a str."""
    import pathlib
    from dad_3dheads_b200.predictor import StepOptions
    with pytest.raises(ValueError, match="needs boxes.*no-box path"):
        StepOptions(to_2d=False, uv_texture="texture_data.npy")
    with pytest.raises(ValueError, match="to_2d=False"):
        StepOptions(rois=2, uv_texture="texture_data.npy")
    with pytest.raises(ValueError, match="a path to texture_data.npy or a UvTextureTable"):
        StepOptions(rois=2, to_2d=False, uv_texture=3)
    a = StepOptions(rois=2, to_2d=False, uv_texture=pathlib.Path("t/texture_data.npy"))
    assert a.uv_texture == "t/texture_data.npy" and a == StepOptions(rois=2, to_2d=False, uv_texture="t/texture_data.npy")
    assert a != StepOptions(rois=2, to_2d=False) and StepOptions(rois=2, to_2d=False).uv_texture is None
