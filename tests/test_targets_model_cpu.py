"""-m "not gpu": the exact model of the training-target kernels (tests/targets_model.py) and the host side of
dad_3dheads_b200.training_data, against the live reference FlameDataset (oracle/ref_harness.py, with the keypoint path of
tests/albumentations_keypoints.py) on a synthetic dataset.

Two tiers against the reference, whose 4x4 matmuls run through BLAS sgemm in a host-dependent order:
  * continuous targets within 1e-5 * max(1, |ref|) pixels;
  * presence and heat-map planes equal for every landmark whose reference coordinate is more than 1e-3 px from its presence
    bounds and whose p / stride is more than 1e-4 from an integer; the excluded landmarks are counted, and fewer than 1 %
    may be excluded."""
import json
import os

import cv2
import numpy as np
import pytest
import torch

from dad_3dheads_b200.training_data import (IMAGE_FILENAME_KEY, INPUT_BBOX_KEY, INPUT_IMAGE_KEY, SAMPLE_INDEX_KEY,
                                             TARGET_2D_FULL_LANDMARKS, TARGET_2D_LANDMARKS, TARGET_2D_LANDMARKS_PRESENCE,
                                             TARGET_3D_MODEL_VERTICES, TARGET_LANDMARKS_HEATMAP, FlameDataset, crop_box,
                                             heatmap_window)
from oracle import ref_harness as R
from tests import targets_model as M
from tests.albumentations_keypoints import keypoint_albumentations

FRAMES = [(180, 240), (300, 200), (512, 400), (120, 150), (400, 640), (256, 320), (700, 500)]      # (H, W)
CONFIGS = {
    "68": dict(num_classes=68, stride=4, radius=5, normalize="imagenet", subset="multipie_keypoints"),
    "191": dict(num_classes=191, stride=2, radius="pointwise", normalize="mean", subset="keypoints_191"),
}


def ref_root():
    if not R.available():
        pytest.skip("reference harness not available")
    return R.root()


def dataset_config(root: str, name: str) -> dict:
    c = CONFIGS[name]
    subset = os.path.join(ref_root(), "model_training", "model", "static", "face_keypoints", c["subset"])
    cfg = {"dataset_root": root, "img_size": 256, "stride": c["stride"], "num_classes": c["num_classes"],
           "keypoints": {"2d_subset_name": c["subset"], "2d_subset_path": subset},
           "coder": {"_target_": "model_training.data.coder.HeatmapCoder"},
           "transform": {"normalize": c["normalize"], "resize_mode": "longest_max_size"}}
    if c["radius"] != 5:
        cfg["radius"] = c["radius"]
    return cfg


def _rotation(rng):
    yaw, pitch, roll = np.deg2rad(rng.uniform(-40, 40)), np.deg2rad(rng.uniform(-20, 20)), np.deg2rad(rng.uniform(-20, 20))
    cy, sy, cp, sp, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    Rz = np.array([[cr, -sr, 0], [sr, cr, 0], [0, 0, 1]])
    return Rz @ Rx @ Ry


def make_dataset(root: str, n: int, seed: int = 0):
    """n items over PNG frames of the FRAMES sizes: seeded FLAME meshes, random head poses under a pixel-space perspective
    projection (P @ X / w gives x and height - y), boxes around the projected heads; every fourth head sits on a frame
    border, so boxes cross each border of the frame in turn -> the annotation list."""
    from oracle.flame_oracle import FlameOracle, sample_params
    rng = np.random.default_rng(seed)
    verts = FlameOracle().vertices_3d(sample_params(n, seed)).numpy().astype(np.float32)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    data = []
    for i in range(n):
        H, W = FRAMES[i % len(FRAMES)]
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        img = cv2.GaussianBlur(img, (5, 5), 1.5)
        path = f"images/{i:04d}.png"
        cv2.imwrite(os.path.join(root, path), cv2.cvtColor(img, cv2.COLOR_RGB2BGR))
        f = rng.uniform(1.5, 3.0) * max(H, W)
        frac = rng.uniform(0.25, 0.7)
        d = f * 0.2 / (frac * min(H, W))
        u, v = rng.uniform(0.2, 0.8) * W, rng.uniform(0.2, 0.8) * H
        side = i % 4 if i % 2 == 0 else None
        if side is not None:                       # left, top, right, bottom border in turn
            u, v = [(0.02 * W, v), (u, 0.02 * H), (0.98 * W, v), (u, 0.98 * H)][(i // 2) % 4]
        mv = np.eye(4)
        mv[:3, :3] = _rotation(rng)
        mv[:3, 3] = [(u - W / 2) * d / f, (H / 2 - v) * d / f, -d]
        P = np.array([[f, 0, -W / 2, 0], [0, f, -H / 2, 0], [0, 0, -1.0, -0.2], [0, 0, -1.0, 0]])
        mv32, P32 = mv.astype(np.float32), P.astype(np.float32)
        X = np.concatenate([verts[i], np.ones((verts.shape[1], 1), np.float32)], 1).astype(np.float64) @ mv.T @ P.T
        px, py = X[:, 0] / X[:, 3], H - X[:, 1] / X[:, 3]
        x0, y0, x1, y1 = px.min(), py.min(), px.max(), py.max()
        jit = rng.uniform(-0.05, 0.05, 4) * (x1 - x0)
        bbox = [int(x0 + jit[0]), int(y0 + jit[1]), int(x1 - x0 + jit[2]), int(y1 - y0 + jit[3])]
        anno = f"meshes/{i:04d}.json"
        os.makedirs(os.path.join(root, "meshes"), exist_ok=True)
        with open(os.path.join(root, anno), "w") as fd:
            json.dump({"vertices": verts[i].astype(np.float64).tolist(), "model_view_matrix": mv32.astype(np.float64).tolist(),
                       "projection_matrix": P32.astype(np.float64).tolist()}, fd)
        data.append({"img_path": path, "bbox": bbox, "annotation_path": anno})
    return data


def reference_batch(data, config, seed: int):
    R.activate()
    from model_training.data.flame_dataset import FlameDataset as RefDataset, collate_skip_none
    with keypoint_albumentations():
        ds = RefDataset(data, config)
        np.random.seed(seed)
        return collate_skip_none([ds[i] for i in range(len(data))])


def package_batch(data, config, seed: int):
    ds = FlameDataset(data, config)
    np.random.seed(seed)
    return ds.get_collate_fn()([ds[i] for i in range(len(data))])


def lm_tables(config):
    if config["num_classes"] != 68:
        return None, None
    from dad_3dheads_b200.submission import landmark68_tables
    tri, bary = landmark68_tables()
    return tri.numpy(), bary.numpy()


def check_against_reference(got, ref, config, label: str):
    """The two-tier contract; got: numpy arrays (or tensors) in the builder's layout; ref: the reference's collated dict."""
    np_ = lambda t: t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    assert set(ref) == set(got) - {"landmarks_px"}, (sorted(ref), sorted(got))
    S, stride = config["img_size"], config["stride"]
    assert np.array_equal(np_(got[INPUT_IMAGE_KEY]), ref[INPUT_IMAGE_KEY].numpy()), "images differ"
    assert np.array_equal(np_(got[TARGET_3D_MODEL_VERTICES]), ref[TARGET_3D_MODEL_VERTICES].numpy())
    for a, b in zip(got[INPUT_BBOX_KEY], ref[INPUT_BBOX_KEY]):
        assert np.array_equal(np_(a), b.numpy())
    assert np.array_equal(np_(got[SAMPLE_INDEX_KEY]), ref[SAMPLE_INDEX_KEY].numpy())
    assert list(got[IMAGE_FILENAME_KEY]) == list(ref[IMAGE_FILENAME_KEY])
    worst = 0.0
    for key, scale in ((TARGET_2D_FULL_LANDMARKS, 1.0), (TARGET_2D_LANDMARKS, float(S))):
        a, b = np_(got[key]).astype(np.float64) * scale, ref[key].numpy().astype(np.float64) * scale
        err = np.abs(a - b) / np.maximum(1.0, np.abs(b))
        worst = max(worst, float(err.max()))
        assert err.max() <= 1e-5, (key, float(err.max()))
    # exclusions: reference landmark too close to a presence bound or to a heat-map cell edge
    lm = ref[TARGET_2D_LANDMARKS].numpy().astype(np.float64) * S                       # network pixels
    bbox = np.stack([b.numpy() for b in ref[INPUT_BBOX_KEY]], 1)                       # [B,4]
    w, h = bbox[:, 2:3].astype(np.float64), bbox[:, 3:4].astype(np.float64)
    sc = S / np.maximum(w, h)
    nw, nh = np.rint(w * sc), np.rint(h * sc)
    crop_x = (lm[..., 0] - np.where(nw < S, (S - nw) // 2, 0)) / sc
    crop_y = (lm[..., 1] - np.where(nh < S, (S - nh) // 2, 0)) / sc
    near_bound = np.minimum.reduce([np.abs(crop_x), np.abs(crop_x - w), np.abs(crop_y), np.abs(crop_y - h)]) <= 1e-3
    q = lm / stride
    near_cell = (np.abs(q - np.rint(q)) <= 1e-4).any(-1)
    keep = ~(near_bound | near_cell)
    excluded = int((~keep).sum())
    total = keep.size
    print(f"[{label}] max continuous error {worst:.3e} (relative to max(1, |ref|)); excluded {excluded} of {total} landmarks")
    assert excluded < 0.01 * total
    pres = np_(got[TARGET_2D_LANDMARKS_PRESENCE]).astype(bool)
    assert np.array_equal(pres[keep], ref[TARGET_2D_LANDMARKS_PRESENCE].numpy()[keep])
    hm_got, hm_ref = np_(got[TARGET_LANDMARKS_HEATMAP]), ref[TARGET_LANDMARKS_HEATMAP].numpy()
    assert hm_got.dtype == np.uint8 and hm_got.shape == hm_ref.shape
    assert np.array_equal(hm_got[keep], hm_ref[keep])
    assert ref[TARGET_2D_LANDMARKS_PRESENCE].numpy()[keep].any()
    return worst


@pytest.mark.parametrize("name", list(CONFIGS))
def test_model_matches_live_reference(tmp_path, name):
    config = dataset_config(str(tmp_path), name)
    data = make_dataset(str(tmp_path), 28, seed=7)
    ref = reference_batch(data, config, seed=11)
    packed = package_batch(data, config, seed=11)
    tri, bary = lm_tables(config)
    got = M.build_batch(packed, config, tri, bary)
    for key, want in ref.items():
        if isinstance(want, torch.Tensor):
            assert got[key].shape == tuple(want.shape), key
    check_against_reference(got, ref, config, name)


def test_host_crop_and_offsets_match_reference(tmp_path):
    ref_root()
    R.activate()
    from model_training.data.utils import ensure_bbox_boundaries, extend_bbox
    rng = np.random.default_rng(3)
    for _ in range(2000):
        H, W = (int(v) for v in rng.integers(1, 900, 2))
        bbox = [int(rng.integers(-200, W + 200)), int(rng.integers(-200, H + 200)), int(rng.integers(0, 600)),
                int(rng.integers(0, 600))]
        off = tuple(0.1 * rng.uniform(size=4) + 0.05)
        want = tuple(int(v) for v in ensure_bbox_boundaries(extend_bbox(np.array(bbox), off), (H, W)))
        assert crop_box(bbox, off, (H, W)) == want, (bbox, off, H, W)
    # the datasets draw the same offsets in the same order: same crops, same RNG state afterwards
    config = dataset_config(str(tmp_path), "68")
    data = make_dataset(str(tmp_path), 6, seed=1)
    from model_training.data.flame_dataset import FlameDataset as RefDataset
    from model_training.data.config import INPUT_BBOX_KEY as K
    with keypoint_albumentations():
        ds_ref = RefDataset(data, config)
    ds = FlameDataset(data, config)
    np.random.seed(5)
    ref_boxes = [tuple(int(v) for v in ds_ref._parse_anno(data[i])[K]) for i in range(6)]
    after_ref = np.random.uniform()
    np.random.seed(5)
    boxes = [ds[i]["crop"] for i in range(6)]
    assert boxes == ref_boxes and np.random.uniform() == after_ref


def test_configuration_and_crop_errors(tmp_path):
    config = dataset_config(str(tmp_path), "68")
    for key, value, pattern in (("resize_mode", "resize", "resize_mode 'resize'"), ("normalize", "none", "normalize 'none'")):
        bad = dict(config, transform=dict(config["transform"], **{key: value}))
        with pytest.raises(ValueError, match=pattern):
            FlameDataset([], bad)
    with pytest.raises(ValueError, match="coder._target_ 'my.Coder'"):
        FlameDataset([], dict(config, coder={"_target_": "my.Coder"}))
    with pytest.raises(ValueError, match="num_classes 190"):
        FlameDataset([], dict(dataset_config(str(tmp_path), "191"), num_classes=190))
    os.makedirs(tmp_path / "images")
    cv2.imwrite(str(tmp_path / "images" / "a.png"), np.zeros((700, 200, 3), np.uint8))
    with open(tmp_path / "m.json", "w") as fd:
        json.dump({"vertices": [[0, 0, 0]], "model_view_matrix": np.eye(4).tolist(), "projection_matrix": np.eye(4).tolist()}, fd)
    data = [{"img_path": "images/a.png", "bbox": [250, 10, 40, 40], "annotation_path": "m.json"},      # right of the frame
            {"img_path": "images/a.png", "bbox": [0, 0, 1, 690], "annotation_path": "m.json"}]        # 1 x 700 px
    ds = FlameDataset(data, config)
    with pytest.raises(ValueError, match=r"item 0 \(images/a.png\): the crop .* is empty"):
        ds[0]
    with pytest.raises(ValueError, match=r"item 1 \(images/a.png\): the crop .* letter-boxes to a side of 0 pixels"):
        ds[1]


@pytest.mark.parametrize("subset", ["keypoints_191", "keypoints_445", "multipie_keypoints"])
def test_load_2d_indices_matches_reference(subset):
    root = ref_root()
    R.activate()
    from model_training.utils import load_2d_indices as ref_load
    from dad_3dheads_b200.flame_assets import load_2d_indices
    cfg = {"2d_subset_name": subset, "2d_subset_path": os.path.join(root, "model_training", "model", "static",
                                                                     "face_keypoints", subset)}
    want = ref_load(dict(cfg))
    got = load_2d_indices(dict(cfg))
    assert got == want and (want is None or len(want) in (191, 445))


def edge_cells(S: int, r: int):
    return sorted(set(range(-2 * S - 2 * r - 3, -S + 2 * r + 3)) | set(range(-2 * r - 3, 2 * r + 4))
                  | set(range(S - 2 * r - 3, S + 2 * r + 4)) | {S // 2, 2 * S, 3 * S + 1})


@pytest.mark.parametrize("radius", [5, 2, "pointwise"])
@pytest.mark.parametrize("stride", [2, 3, 4])
def test_heatmap_model_matches_draw_gaussian(radius, stride):
    """Cells at 0, S-1, S, negative values and beyond the radius, and keypoints that reach them through float32 floor
    division: the model equals HeatmapCoder + np.uint8(255 * heatmap) of the reference."""
    ref_root()
    R.activate()
    from model_training.data.coder import HeatmapCoder
    S = 256 // stride
    r = 1 if radius == "pointwise" else radius
    coder = HeatmapCoder({"img_size": 256, "stride": stride, "radius": radius}, 1)
    table = heatmap_window(radius)
    rng = np.random.default_rng(stride)
    cells = edge_cells(S, r)
    points = [np.float32([(cx + 0.5) * stride, (cy + 0.25) * stride]) for cx in cells for cy in (0, S - 1, S // 3)]
    points += [np.float32([rng.uniform(-300, 600), rng.uniform(-300, 600)]) for _ in range(300)]
    points += [np.float32([cx * stride, 255.99998]) for cx in (0, S - 1, S)]       # exact multiples, and a row that rounds
    for p in points:
        want = np.uint8(255.0 * coder(p[None], np.array([True])))[0]
        got = M.heatmap_plane(p, True, S, stride, table, r)
        assert np.array_equal(got, want), (p, stride, radius)
        cx = M.heat_cell(p[0], stride)
        assert cx == int((p // stride)[0])
    assert not M.heatmap_plane(points[0], False, S, stride, table, r).any()


def test_keypoint_albumentations_restores_the_module():
    ref_root()
    R.activate()
    import albumentations as A
    before = {k: getattr(A, k) for k in ("Compose", "LongestMaxSize", "PadIfNeeded", "Normalize", "KeypointParams")}
    with keypoint_albumentations():
        assert A.Compose is not before["Compose"]
    assert {k: getattr(A, k) for k in before} == before
