"""-m gpu: the UV textures of csrc/uv_texture.cu (dad_3dheads_b200.uv_texture, predict_batch(uv_texture=)).

Every texture is compared byte for byte with tests/uv_model.py, which tests/test_uv_model_cpu.py pins to the reference's own
``_compute_texture_map`` on tests/psbody_mesh.py's ``Mesh``, evaluated on this call's own device inputs."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from dad_3dheads_b200.flame import load_flame_static
from dad_3dheads_b200.uv_texture import UvTextureTable, compact_table, faces_by_vertex, read_table, uv_textures
from tests import uv_model as M
from tests.test_demo_unchanged_gpu import ROOT, demo_home  # noqa: F401  (fixture)

TABLE = M.reference_table_path()
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device"),
              pytest.mark.skipif(TABLE is None, reason="the reference's texture_data.npy (oracle/_ref) is not built")]
FACES = load_flame_static()["faces"]


def _dev(i=0):
    return torch.device("cuda", i)


@pytest.fixture(scope="module")
def compact():
    return compact_table(read_table(TABLE))


@pytest.fixture(scope="module")
def table():
    return UvTextureTable.load(TABLE, _dev())


@pytest.fixture(scope="module")
def pred():
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    return FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0))


def _heads(R, F, seed):
    """R fp32 heads over F odd-sized frames: the designed cases first, then decoded heads placed at random; frame indices
    not monotone; head 1 invalid (when R > 1)."""
    g = np.random.default_rng(seed)
    H, W = [(257, 263), (301, 199)][seed % 2]
    frames = g.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    designed = [v for v, _ in M.designed_heads(FACES, seed).values()]
    extra = list(M.flame_heads(R - len(designed), seed + 1)) if R > len(designed) else []
    v = np.stack((designed + extra)[:R]).astype(np.float32)
    for r in range(len(designed), R):
        v[r, :, :2] += g.uniform(-40, 60, 2).astype(np.float32)
    fidx = g.permutation(np.arange(R) % F).astype(np.int32)
    valid = np.ones(R, dtype=bool)
    if R > 1:
        valid[1] = False
    return frames, v, fidx, valid


def _want(frames, v, fidx, valid, compact):
    S, texel, vids, bary = compact
    row, col = faces_by_vertex(FACES, 5023)
    return M.textures(v, frames, fidx, valid, FACES, row, col, texel, vids, bary, S)


@pytest.mark.parametrize("R, F", [(1, 1), (3, 3), (64, 3), (65, 1)])
def test_kernels_equal_the_model(table, compact, R, F):
    frames, v, fidx, valid = _heads(R, F, seed=R + F)
    got = uv_textures(table, torch.from_numpy(frames).to(_dev()), torch.from_numpy(v).to(_dev()),
                      torch.from_numpy(fidx).to(_dev()), torch.from_numpy(valid).to(_dev()))
    want = _want(frames, v, fidx, valid, compact)
    got = got.cpu().numpy()
    for r in range(R):
        assert np.array_equal(got[r], want[r]), (r, int((got[r] != want[r]).any(-1).sum()))
    if R > 1:
        assert not got[1].any()
    assert got.any()


def test_guard_bands_and_out_of_range_frames(table, compact):
    """Through the C ABI: the output between 0xA5 bands that stay untouched; a device frame index outside [0, F) zeroes
    that head; no valid array means every head is valid."""
    R, F = 3, 2
    frames, v, fidx, _ = _heads(R, F, seed=9)
    fidx[2] = F                                                       # out of range on the device: an all-zero texture
    S = table.img_size
    n = R * S * S * 3
    buf = torch.full((n + 2 * 4096,), 0xA5, dtype=torch.uint8, device=_dev())
    ws = torch.empty(int(table.lib.dad3d_uv_workspace_bytes(table.handle, R)), dtype=torch.uint8, device=_dev())
    fr, vd, fi = (torch.from_numpy(a).to(_dev()) for a in (frames, v, fidx))
    _lib.check(table.lib.dad3d_uv_texture(table.handle, vd.data_ptr(), R, None, fr.data_ptr(), F, frames.shape[1],
                                          frames.shape[2], fi.data_ptr(), buf.data_ptr() + 4096, ws.data_ptr(),
                                          ws.numel(), torch.cuda.current_stream().cuda_stream), "dad3d_uv_texture")
    b = buf.cpu().numpy()
    assert (b[:4096] == 0xA5).all() and (b[4096 + n:] == 0xA5).all()
    got = b[4096:4096 + n].reshape(R, S, S, 3)
    want = _want(frames, v, fidx, None, compact)
    assert np.array_equal(got, want) and not got[2].any() and got[0].any()
    # the workspace keeps the normals' z of the heads that ran (head 1 is rough_normals): bit for bit, so a change of
    # summation order shows even where it flips no texel
    nz = ws.view(torch.float64).view(R, 5023).cpu().numpy()
    row, col = faces_by_vertex(FACES, 5023)
    for r in range(2):
        want_nz = M.vertex_normals_z(v[r], FACES, row, col)
        assert np.array_equal(nz[r].view(np.int64), want_nz.view(np.int64)), r


def test_invalid_arguments_are_reported_not_crashed(table):
    lib = table.lib
    d = torch.zeros(16, dtype=torch.uint8, device=_dev())
    p = d.data_ptr()
    ws = torch.empty(int(lib.dad3d_uv_workspace_bytes(table.handle, 1)), dtype=torch.uint8, device=_dev())
    s = torch.cuda.current_stream().cuda_stream
    cases = [
        (None, p, 1, None, p, 1, 4, 4, None, p, ws.data_ptr(), ws.numel()),       # null handle
        (table.handle, p, -1, None, p, 1, 4, 4, None, p, ws.data_ptr(), ws.numel()),
        (table.handle, p, 65536, None, p, 1, 4, 4, None, p, ws.data_ptr(), ws.numel()),
        (table.handle, p, 1, None, p, 0, 4, 4, None, p, ws.data_ptr(), ws.numel()),
        (table.handle, p, 1, None, p, 1, 0, 4, None, p, ws.data_ptr(), ws.numel()),
        (table.handle, None, 1, None, p, 1, 4, 4, None, p, ws.data_ptr(), ws.numel()),
        (table.handle, p, 1, None, p, 1, 4, 4, None, None, ws.data_ptr(), ws.numel()),
        (table.handle, p, 1, None, p, 1, 4, 4, None, p, ws.data_ptr(), ws.numel() - 1),
    ]
    before = _lib.launch_count()
    for args in cases:
        assert lib.dad3d_uv_texture(*args, s) == -1, args
        assert b"invalid argument" in lib.dad3d_last_error()
    assert _lib.launch_count() == before
    assert lib.dad3d_uv_workspace_bytes(None, 1) == 0 and lib.dad3d_uv_workspace_bytes(table.handle, -1) == 0
    # create: duplicate texel, texel outside the image, vertex id out of range, a CSR that is not faces_by_vertex
    faces = np.ascontiguousarray(FACES, dtype=np.int32)
    row, col = faces_by_vertex(faces, 5023)
    good = (np.array([0, 5], np.int32), np.zeros((2, 3), np.int32), np.zeros((2, 3)))

    def create(texel, vids, bary, c):
        h = C.c_void_p()
        rc = lib.dad3d_uv_create(C.byref(h), 8, texel.ctypes.data, vids.ctypes.data, bary.ctypes.data, 2,
                                 faces.ctypes.data, faces.shape[0], row.ctypes.data, c.ctypes.data, 5023, 0)
        if h:
            lib.dad3d_uv_destroy(h)
        return rc, bool(h)

    assert create(*good, col) == (0, True)
    assert create(np.array([5, 5], np.int32), *good[1:], col) == (-1, False)          # duplicate texel
    assert create(np.array([0, 64], np.int32), *good[1:], col) == (-1, False)         # outside the 8x8 image
    assert create(good[0], np.full((2, 3), 5023, np.int32), good[2], col) == (-1, False)
    assert create(*good, col[::-1].copy()) == (-1, False)                             # not faces_by_vertex


def test_launches_no_sync_determinism_and_permutation(table):
    frames, v, fidx, valid = _heads(65, 3, seed=4)
    fr, vd, fi, va = (torch.from_numpy(a).to(_dev()) for a in (frames, v, fidx, valid))
    uv_textures(table, fr, vd[:1].contiguous(), fi[:1].contiguous(), va[:1].contiguous())
    torch.cuda.synchronize()
    counts = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for R in (1, 65):
            before = _lib.launch_count()
            a = uv_textures(table, fr, vd[:R].contiguous(), fi[:R].contiguous(), va[:R].contiguous())
            counts.append(_lib.launch_count() - before)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert counts == [2, 2]
    b = uv_textures(table, fr, vd, fi, va)
    assert torch.equal(a, b)
    perm = torch.from_numpy(np.random.default_rng(1).permutation(65)).to(_dev())
    c = uv_textures(table, fr, vd[perm].contiguous(), fi[perm].contiguous(), va[perm].contiguous())
    assert torch.equal(c, b[perm])


def _scene(F, H, W, seed):
    g = np.random.default_rng(seed)
    boxes = [(int(g.integers(0, W - 200)), int(g.integers(0, H - 200)), int(g.integers(120, 200)),
              int(g.integers(120, 200))) for _ in range(6)]
    boxes += [(0, 0, W, H), (W, 5, 40, 40)]                                # the whole frame; an empty crop (invalid)
    fidx = [int(g.integers(0, F)) for _ in range(7)] + [0]
    return torch.tensor(boxes, dtype=torch.int32), torch.tensor(fidx, dtype=torch.int32).to(_dev())


def test_step_output_equals_uv_textures_and_leaves_the_rest(pred, table):
    F, H, W = 2, 301, 407
    frames = torch.from_numpy(np.random.default_rng(2).integers(0, 256, (F, H, W, 3), dtype=np.uint8))
    boxes, fidx = _scene(F, H, W, 3)
    base = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, to_2d=False)
    out = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, to_2d=False, uv_texture=TABLE)
    assert set(out) == set(base) | {"uv_texture"}
    for k, v in base.items():
        assert torch.equal(v, out[k]), k
    want = uv_textures(table, frames.to(_dev()).contiguous(), out["projected_vertices"].contiguous(), fidx, out["valid"])
    assert torch.equal(out["uv_texture"], want)
    assert not out["valid"][-1] and not out["uv_texture"][-1].any() and out["uv_texture"].any()
    again = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, to_2d=False, uv_texture=table)
    assert torch.equal(again["uv_texture"], want)
    with pytest.raises(ValueError, match="needs boxes"):
        pred.predict_batch(frames, to_2d=False, uv_texture=TABLE)
    with pytest.raises(ValueError, match="to_2d=False"):
        pred.predict_batch(frames, boxes=boxes, frame_index=fidx, uv_texture=TABLE)


def test_graphed_and_stream_equal_eager(pred):
    F, H, W = 2, 360, 480
    for seed in (5, 6):
        frames = torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (F, H, W, 3), dtype=np.uint8))
        boxes, fidx = _scene(F, H, W, seed)
        eager = pred.predict_batch(frames, boxes=boxes, frame_index=fidx, to_2d=False, uv_texture=TABLE)
        eager = {k: v.clone() for k, v in eager.items()}
        g = pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fidx, to_2d=False, uv_texture=TABLE)
        for k in eager:
            assert torch.equal(g[k], eager[k]), (seed, k)
    st = pred.open_stream((F, H, W, 3), rois=int(boxes.shape[0]), to_2d=False, uv_texture=TABLE,
                          keys=("uv_texture", "valid"))
    st.submit(frames, boxes=boxes, frame_index=fidx)
    res = st.collect()
    assert torch.equal(res["uv_texture"], eager["uv_texture"].cpu())


def test_demo_py_uv_texture_equals_the_reference_loop(demo_home, tmp_path):
    """``python demo.py images/demo_heads/1.jpeg <out> uv_texture``, the reference's unchanged demo over compat/: its PNG
    equals the reference's own ``_compute_texture_map`` (on tests/psbody_mesh.py's ``Mesh``) fed the vertices the demo's own predictor
    and HeadMesh give on the same image."""
    import cv2
    from oracle import ref_harness as R
    from tests.test_demo_unchanged_gpu import _run_demo
    _run_demo(demo_home, tmp_path, "uv_texture")
    got = cv2.cvtColor(cv2.imread(str(tmp_path / "1_uv_texture.png")), cv2.COLOR_BGR2RGB)
    ref_root = R.root()
    dump = tmp_path / "demo_vertices.npz"
    code = ("import sys\n"
            "sys.path[:0] = [%r, %r, %r, %r]\n"
            "import numpy as np\n"
            "from predictor import FaceMeshPredictor\n"
            "from pytorch_toolbelt.utils import read_rgb_image\n"
            "from model_training.head_mesh import HeadMesh\n"
            "image = read_rgb_image('images/demo_heads/1.jpeg')\n"
            "p = FaceMeshPredictor.dad_3dnet()(image)\n"
            "v = HeadMesh().reprojected_vertices(params_3dmm=p['3dmm_params'], to_2d=False)[0]\n"
            "np.savez(%r, image=image, v=v.cpu().numpy())\n"
            % (os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "oracle", "ref_shims"), ref_root, str(dump)))
    out = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=600,
                         cwd=ref_root, env=dict(os.environ, HOME=str(demo_home)))
    assert out.returncode == 0, out.stderr[-3000:]
    z = np.load(dump)
    want = M.reference_texture_map(z["image"], z["v"], FACES, read_table(TABLE))
    assert got.shape == want.shape == (512, 512, 3)
    assert np.array_equal(got, want), int((got != want).any(-1).sum())
    assert want.any(-1).sum() > 1000


def test_second_device_follows_the_tensors(compact):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    frames, v, fidx, valid = _heads(3, 2, seed=11)
    t1 = UvTextureTable.load(TABLE, _dev(1))
    with torch.cuda.device(0):
        got = uv_textures(t1, *(torch.from_numpy(a).to(_dev(1)) for a in (frames, v)),
                          *(torch.from_numpy(a).to(_dev(1)) for a in (fidx, valid)))
    assert got.device == _dev(1)
    assert np.array_equal(got.cpu().numpy(), _want(frames, v, fidx, valid, compact))
    with pytest.raises(ValueError, match="table is on"):
        uv_textures(t1, torch.from_numpy(frames).to(_dev(0)), torch.from_numpy(v).to(_dev(0)))
