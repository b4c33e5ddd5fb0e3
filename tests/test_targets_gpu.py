"""-m gpu: FlameBatchBuilder (dad_3dheads_b200.training_data, csrc/targets.cu) against the exact model
(tests/targets_model.py) bit for bit, and against the live reference FlameDataset within the two-tier contract of
tests/test_targets_model_cpu.py."""
import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from dad_3dheads_b200.training_data import (INPUT_BBOX_KEY, TARGET_LANDMARKS_HEATMAP, FlameBatchBuilder, FlameDataset,
                                             collate_records, heatmap_window)
from tests import targets_model as M
from tests.test_targets_model_cpu import (CONFIGS, check_against_reference, dataset_config, edge_cells, lm_tables,
                                          make_dataset, reference_batch)

pytestmark = pytest.mark.gpu


def synthetic_records(B: int, seed: int, crops=None):
    """B host records without files: crops of mixed sizes (long sides 1 to 600 px) at random frame positions, seeded FLAME
    meshes, random poses and pixel-space projections that put the heads around their crops."""
    from oracle.flame_oracle import FlameOracle, sample_params
    from tests.test_targets_model_cpu import _rotation
    rng = np.random.default_rng(seed)
    meshes = FlameOracle().vertices_3d(sample_params(16, seed)).numpy().astype(np.float32)
    recs = []
    for b in range(B):
        w, h = crops[b] if crops is not None and b < len(crops) else (int(rng.integers(20, 600)), int(rng.integers(20, 600)))
        x, y = int(rng.integers(0, 400)), int(rng.integers(0, 400))
        H = y + h + int(rng.integers(0, 300))
        f = rng.uniform(1.5, 3.0) * max(w, h, 64)
        d = f * 0.2 / (rng.uniform(0.5, 1.2) * max(min(w, h), 8))
        u, v = x + w * rng.uniform(0.3, 0.7), y + h * rng.uniform(0.3, 0.7)
        mv = np.eye(4)
        mv[:3, :3] = _rotation(rng)
        mv[:3, 3] = [(u - 300) * d / f, (H - v - 300) * d / f, -d]
        P = np.array([[f, 0, -300, 0], [0, f, -300, 0], [0, 0, -1.0, -0.2], [0, 0, -1.0, 0]])
        recs.append({"image": rng.integers(0, 256, (h, w, 3), dtype=np.uint8), "crop": (x, y, w, h), "frame_height": H,
                     "vertices": meshes[b % len(meshes)], "model_view": mv.astype(np.float32),
                     "projection": P.astype(np.float32), "index": 1000 + b, "filename": f"frame_{b}.png"})
    return recs


def _cpu(out):
    return {k: ([t.cpu() for t in v] if isinstance(v, list) and v and isinstance(v[0], torch.Tensor)
                else v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


def _assert_equal_to_model(out, want):
    for k, w in want.items():
        if k == "landmarks_px":
            continue
        g = out[k]
        if isinstance(w, list):
            assert len(g) == len(w), k
            for a, b in zip(g, w):
                assert (np.array_equal(a.numpy(), b) if isinstance(a, torch.Tensor) else a == b), k
        else:
            a = g.numpy()
            assert a.shape == w.shape, (k, a.shape, w.shape)
            if a.dtype == np.float32:
                assert np.array_equal(a.view(np.int32), np.asarray(w, np.float32).view(np.int32)), k
            else:
                assert np.array_equal(a, w), k


@pytest.mark.parametrize("name", list(CONFIGS))
def test_builder_matches_model_bit_for_bit(tmp_path, cuda_device, name):
    config = dataset_config(str(tmp_path), name)
    edge = [(256, 180), (170, 256), (1, 200), (256, 256), (600, 1), (3, 3)]     # no resize; 1-px sides that letter-box
    packed = collate_records(synthetic_records(300, 5, edge))
    out = _cpu(FlameBatchBuilder(config, cuda_device)(packed))
    torch.cuda.synchronize()
    tri, bary = lm_tables(config)
    _assert_equal_to_model(out, M.build_batch(packed, config, tri, bary))
    assert out["TARGET_2D_LANDMARKS_PRESENCE"].any() and not out["TARGET_2D_LANDMARKS_PRESENCE"].all()


@pytest.mark.parametrize("radius", [5, 2, "pointwise"])
@pytest.mark.parametrize("stride", [2, 3, 4])
def test_heatmap_entry_point_on_edge_cells(cuda_device, radius, stride):
    S = 256 // stride
    r = 1 if radius == "pointwise" else radius
    cells = edge_cells(S, r)
    pts = [((cx + 0.5) * stride, (cy + 0.25) * stride) for cx in cells for cy in cells[::7]]
    pts += [(cx * stride, 255.99998) for cx in (0, S - 1, S)] + [(float("nan"), 3.0), (float("inf"), 3.0)]
    lm = np.array(pts, np.float32)[None]
    pres = np.ones(lm.shape[:2], bool)
    pres[0, ::5] = False
    want = M.heatmaps(lm, pres, S, stride, radius)
    table = torch.from_numpy(heatmap_window(radius)).to(cuda_device)
    lm_d = torch.from_numpy(lm).to(cuda_device)
    pres_d = torch.from_numpy(pres.astype(np.uint8)).to(cuda_device)
    out = torch.full(want.shape, 77, dtype=torch.uint8, device=cuda_device)       # every byte must be written
    lib = _lib.load()
    _lib.check(lib.dad3d_heatmap_targets(lm_d.data_ptr(), pres_d.data_ptr(), lm.shape[1], S, stride, table.data_ptr(), r,
                                         out.data_ptr(), torch.cuda.current_stream().cuda_stream), "dad3d_heatmap_targets")
    assert np.array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_builder_matches_live_reference(tmp_path, cuda_device, name):
    config = dataset_config(str(tmp_path), name)
    data = make_dataset(str(tmp_path), 28, seed=9)
    ref = reference_batch(data, config, seed=13)
    ds = FlameDataset(data, config)
    np.random.seed(13)
    packed = ds.get_collate_fn()([ds[i] for i in range(len(data))])
    out = _cpu(FlameBatchBuilder(config, cuda_device)(packed))
    assert set(out) == set(ref)
    for k, v in ref.items():
        if isinstance(v, torch.Tensor):
            assert out[k].dtype == v.dtype and out[k].shape == v.shape, k
    assert [t.dtype for t in out[INPUT_BBOX_KEY]] == [t.dtype for t in ref[INPUT_BBOX_KEY]]
    check_against_reference(out, ref, config, f"gpu {name}")


def test_properties(tmp_path, cuda_device):
    config = dataset_config(str(tmp_path), "68")
    builder = FlameBatchBuilder(config, cuda_device)
    recs = synthetic_records(64, 8)
    a = _cpu(builder(collate_records(recs)))
    b = _cpu(builder(collate_records(recs)))
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
    perm = np.random.default_rng(0).permutation(len(recs))
    c = _cpu(builder(collate_records([recs[i] for i in perm])))
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(c[k], a[k][torch.from_numpy(perm)]), k
    assert c["IMAGE_FILENAME_KEY"] == [a["IMAGE_FILENAME_KEY"][i] for i in perm]
    for x, y in zip(c[INPUT_BBOX_KEY], a[INPUT_BBOX_KEY]):
        assert torch.equal(x, y[torch.from_numpy(perm)])
    packed = collate_records(recs)
    packed = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in packed.items()}
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        builder(packed)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    counts = []
    for B in (8, 256):
        packed = collate_records(synthetic_records(B, B))
        before = _lib.launch_count()
        builder(packed)
        counts.append(_lib.launch_count() - before)
    torch.cuda.synchronize()
    assert counts[0] == counts[1] == 4, counts


def test_training_path_accepts_builder_targets(tmp_path, cuda_device):
    """The reference's LossModule (train_loss.yaml weights) over dad_3dheads_b200.losses, on the builder's targets after
    KeypointsDataMixin.get_input's conversions (train/mixins.py:45-51)."""
    from tests.test_losses_gpu import _mine
    from oracle import ref_harness as R
    R.activate()
    from model_training.model.flame import uint8_to_float32
    config = dataset_config(str(tmp_path), "68")
    B = 8
    t = FlameBatchBuilder(config, cuda_device)(collate_records(synthetic_records(B, 3)))
    t[TARGET_LANDMARKS_HEATMAP] = uint8_to_float32(t[TARGET_LANDMARKS_HEATMAP])
    t[INPUT_BBOX_KEY] = torch.stack(t[INPUT_BBOX_KEY]).T
    K, module = _mine()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 68, 64, 64, generator=g).to(cuda_device).requires_grad_(True)
    from oracle.flame_oracle import sample_params
    p = sample_params(B, 4).to(cuda_device).requires_grad_(True)
    lm = torch.rand(B, 68, 2, generator=g).to(cuda_device).requires_grad_(True)
    preds = {K.OUTPUT_LANDMARKS_HEATMAP: x, K.OUTPUT_3DMM_PARAMS: p * 1.0, K.OUTPUT_2D_LANDMARKS: lm}
    total, parts = module(preds, t, epoch=0)
    grads = torch.autograd.grad(total, [x, p, lm])
    assert torch.isfinite(total) and all(torch.isfinite(v).all() for v in grads)
    assert t[INPUT_BBOX_KEY].shape == (B, 4)
