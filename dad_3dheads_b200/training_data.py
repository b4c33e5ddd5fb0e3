"""The reference's training batches (model_training/data/flame_dataset.py) with the per-item arithmetic on the GPU.

``FlameDataset`` keeps the reference's constructor, ``from_config`` and configuration keys, but ``__getitem__`` does only what
has to happen on the host: it reads the frame and the mesh JSON, draws the crop offset from numpy's global RNG with the
reference's call in the reference's order, computes the crop box and slices the crop.  ``get_collate_fn()`` packs a list of
those records into CPU tensors; it runs in DataLoader workers and never touches CUDA.  ``FlameBatchBuilder`` turns a packed
batch into the dict the reference's ``collate_skip_none`` returns -- same keys, dtypes and shapes -- on the device:
``dad3d_roi_setup`` + ``dad3d_preprocess_rois`` letter-box the crops (csrc/roi.cu, bit-exact with cv2), then
``dad3d_training_targets`` projects the vertices and landmarks and ``dad3d_heatmap_targets`` draws the heat-maps
(csrc/targets.cu).  Nothing in a build synchronises the host, and it launches four kernels whatever the batch size.

The crop box is computed here on the host, in the reference's float64-then-int32 arithmetic, although ``dad3d_roi_setup``
can compute the same box on the device.  The host has to slice the crop anyway, and uploading whole dataset frames instead of
crops would move many times the bytes; the device then sees each crop as a frame of its own, with box (0, 0, w, h) and no
extend.

Arithmetic that differs from the pinned environment, stated once (DESIGN.md §2):
  * numpy 2 / NEP 50: albumentations multiplies a float32 keypoint by a Python-float scale and adds a Python-int pad, which
    now stays float32: fp32(fp32(x * fp32(s)) + pad).  Under the pinned numpy 1.22 both were float64 with one final rounding;
    the two differ by at most about one ulp of the keypoint.  This module follows numpy 2, as the reference runs here.
  * The reference's 4x4 matmuls go through BLAS sgemm, whose summation order and fma use depend on the host CPU.  The kernels
    use one explicit order of single roundings (tests/targets_model.py restates it bit for bit), so against the reference
    the continuous targets agree to float32 round-off, not bit for bit.
"""
from __future__ import annotations

import json
import os
from typing import Any, Dict, List, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .flame_assets import load_2d_indices
from .predictor import ROI_RECORD_BYTES

SAMPLE_INDEX_KEY = "SAMPLE_INDEX_KEY"
IMAGE_FILENAME_KEY = "IMAGE_FILENAME_KEY"
INPUT_IMAGE_KEY = "INPUT_IMAGE_KEY"
INPUT_BBOX_KEY = "INPUT_BBOX_KEY"
TARGET_3D_MODEL_VERTICES = "TARGET_3D_MODEL_VERTICES"
TARGET_2D_FULL_LANDMARKS = "TARGET_2D_FULL_LANDMARKS"
TARGET_2D_LANDMARKS = "TARGET_2D_LANDMARKS"
TARGET_LANDMARKS_HEATMAP = "TARGET_LANDMARKS_HEATMAP"
TARGET_2D_LANDMARKS_PRESENCE = "TARGET_2D_LANDMARKS_PRESENCE"

NORMALIZE = {"imagenet": ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)), "mean": ((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))}
MAX_BATCH = 65535                                    # dad3d_preprocess_rois runs the crops along grid z


def read_as_rgb(path: str) -> np.ndarray:
    """data/utils.py:18-35: the image as HxWx3 uint8 RGB, read with cv2."""
    import cv2
    img = cv2.imread(path, cv2.IMREAD_COLOR)
    if img is None:
        raise IOError(f"cannot read image {path}")
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB)


def crop_box(bbox: Sequence[float], offset: Sequence[float], shape: Tuple[int, int]) -> Tuple[int, int, int, int]:
    """ensure_bbox_boundaries(extend_bbox(bbox, offset), shape) (data/utils.py:73-115): float64, truncation to int32, then
    x2 from the clipped x1.  offset = (left, right, top, bottom); shape = (H, W)."""
    x, y, w, h = (np.float64(v) for v in bbox)
    left, right, top, bottom = (np.float64(v) for v in offset)
    ex = np.array([x - w * left, y - h * top, w * ((1.0 + right) + left), h * ((1.0 + top) + bottom)]).astype(np.int32)
    H, W = int(shape[0]), int(shape[1])
    x1, y1 = min(max(0, int(ex[0])), W), min(max(0, int(ex[1])), H)
    x2, y2 = min(max(0, x1 + int(ex[2])), W), min(max(0, y1 + int(ex[3])), H)
    return x1, y1, x2 - x1, y2 - y1


def heatmap_window(radius) -> np.ndarray:
    """The uint8 window dad3d_heatmap_targets places: np.uint8(fp32(255 * fp32(g))) of draw_gaussian's kernel
    (data/utils.py:38-70): the 3x3 pointwise kernel, or exp(-(x^2 + y^2) / (2 sigma^2)) over [-r, r]^2 in float64 with
    sigma = (2r + 1) / 6 and entries below eps * max zeroed."""
    if radius == "pointwise":
        g = np.float32([[0.5, 0.75, 0.5], [0.75, 1.0, 0.75], [0.5, 0.75, 0.5]])
    else:
        sigma = (2 * radius + 1) / 6
        y, x = np.ogrid[-radius:radius + 1, -radius:radius + 1]
        g = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
        g[g < np.finfo(g.dtype).eps * g.max()] = 0
    return np.uint8(np.float32(255.0) * g.astype(np.float32))


class TargetConfig:
    """The reference's dataset configuration keys, checked once: img_size, stride (default 2), radius (default 5, or
    "pointwise"), num_classes, keypoints, coder, transform.normalize / resize_mode."""

    def __init__(self, config: Dict[str, Any]):
        self.img_size = int(config["img_size"])
        self.stride = config.get("stride", 2)
        self.radius = config.get("radius", 5)
        self.num_classes = config.get("num_classes")
        transform = config.get("transform") or {}
        mode = transform.get("resize_mode", "longest_max_size")
        if mode != "longest_max_size":
            raise ValueError(f"transform.resize_mode {mode!r}: only 'longest_max_size' is supported")
        norm = transform.get("normalize", "imagenet")
        if norm not in NORMALIZE:
            raise ValueError(f"transform.normalize {norm!r}: only 'imagenet' and 'mean' are supported")
        target = dict(config.get("coder") or {}).get("_target_")
        if not (isinstance(target, str) and target.rsplit(".", 1)[-1] == "HeatmapCoder"):
            raise ValueError(f"coder._target_ {target!r}: only model_training.data.coder.HeatmapCoder is supported")
        if not (isinstance(self.stride, int) and self.stride > 0 and self.img_size // self.stride > 0):
            raise ValueError(f"stride {self.stride!r}: a positive int no larger than img_size is supported")
        if not (self.radius == "pointwise" or (isinstance(self.radius, int) and 0 <= self.radius <= 1024)):
            raise ValueError(f"radius {self.radius!r}: an int in [0, 1024] or 'pointwise' is supported")
        self.keypoints_indices = load_2d_indices(config["keypoints"])
        if self.num_classes != 68 and (self.keypoints_indices is None or len(self.keypoints_indices) != self.num_classes):
            n = None if self.keypoints_indices is None else len(self.keypoints_indices)
            raise ValueError(f"num_classes {self.num_classes!r}: 68, or the {n} indices of keypoints, is supported")
        mean, std = NORMALIZE[norm]
        self.mean255 = np.array(mean, dtype=np.float32) * 255.0          # albumentations Normalize, in fp32
        self.inv_std255 = np.reciprocal(np.array(std, dtype=np.float32) * 255.0, dtype=np.float32)
        self.heatmap_size = self.img_size // self.stride


class FlameDataset(torch.utils.data.Dataset):
    """FlameDataset(data, config) of the reference: ``data`` the annotation list (img_path, bbox, annotation_path per
    item), ``config`` its dataset configuration.  ``__getitem__`` -> a host record; ``get_collate_fn()`` packs records for
    ``FlameBatchBuilder``."""

    def __init__(self, data: List[Dict[str, Any]], config: Dict[str, Any]):
        self.data = data
        self.config = config
        self.targets = TargetConfig(config)
        self.img_size = self.targets.img_size
        self.num_classes = self.targets.num_classes
        self.keypoints_indices = self.targets.keypoints_indices

    @classmethod
    def from_config(cls, config: Dict[str, Any]) -> "FlameDataset":
        with open(config["ann_path"]) as f:
            return cls(data=json.load(f), config=config)

    def __len__(self) -> int:
        return len(self.data)

    def __getitem__(self, idx: int) -> Dict[str, Any]:
        anno = self.data[idx]
        root = self.config["dataset_root"]
        img = read_as_rgb(os.path.join(root, anno["img_path"]))
        offset = tuple(0.1 * np.random.uniform(size=4) + 0.05)          # flame_dataset.py:97, once per item
        x, y, w, h = crop_box(anno["bbox"], offset, img.shape[:2])
        name = f"item {idx} ({anno['img_path']})"
        if w <= 0 or h <= 0:
            raise ValueError(f"{name}: the crop {(x, y, w, h)} is empty")
        scale = self.img_size / max(h, w)
        if round(h * scale) < 1 or round(w * scale) < 1:
            raise ValueError(f"{name}: the crop {(x, y, w, h)} letter-boxes to a side of 0 pixels")
        with open(os.path.join(root, anno["annotation_path"])) as f:
            mesh = json.load(f)
        return {"image": img[y:y + h, x:x + w], "crop": (x, y, w, h), "frame_height": int(img.shape[0]),
                "vertices": np.array(mesh["vertices"], dtype=np.float32),
                "model_view": np.array(mesh["model_view_matrix"], dtype=np.float32),
                "projection": np.array(mesh["projection_matrix"], dtype=np.float32),
                "index": idx, "filename": anno["img_path"]}

    def get_collate_fn(self):
        return collate_records


def collate_records(records: Sequence[Dict[str, Any]]) -> Dict[str, Any]:
    """Host records -> one packed CPU batch: "crops" [B,Hc,Wc,3] uint8 (each crop at the origin of its own zero frame),
    "ints" [12 B] int32 (the device's crop boxes [B,4] = (0, 0, w, h); origins [B,3] = (x, y, frame height); the crop
    boxes [4,B] = x, y, w, h rows; each item's frame index [B]),
    "vertices" [B,V,3], "model_view" and "projection" [B,4,4] fp32, "indices" [B] int64 and "filenames"."""
    B = len(records)
    if not 0 < B <= MAX_BATCH:
        raise ValueError(f"a batch holds 1 to {MAX_BATCH} items, got {B}")
    Hc = max(r["crop"][3] for r in records)
    Wc = max(r["crop"][2] for r in records)
    crops = np.zeros((B, Hc, Wc, 3), np.uint8)
    boxes, origins = np.zeros((B, 4), np.int32), np.zeros((B, 3), np.int32)
    for b, r in enumerate(records):
        x, y, w, h = r["crop"]
        crops[b, :h, :w] = r["image"]
        boxes[b, 2:] = (w, h)
        origins[b] = (x, y, r["frame_height"])
    bbox = np.array([r["crop"] for r in records], np.int32).T
    ints = np.concatenate([boxes.ravel(), origins.ravel(), bbox.ravel(), np.arange(B, dtype=np.int32)])
    return {"crops": torch.from_numpy(crops), "ints": torch.from_numpy(ints),
            "vertices": torch.from_numpy(np.stack([r["vertices"] for r in records])),
            "model_view": torch.from_numpy(np.stack([r["model_view"] for r in records])),
            "projection": torch.from_numpy(np.stack([r["projection"] for r in records])),
            "indices": torch.tensor([r["index"] for r in records], dtype=torch.int64),
            "filenames": [r["filename"] for r in records]}


def _to_device(t: Tensor, device: torch.device) -> Tensor:
    if t.device == device:                            # a packed batch already on the device is used in place
        return t
    return (t if t.is_pinned() else t.pin_memory()).to(device, non_blocking=True)


class FlameBatchBuilder:
    """FlameBatchBuilder(config, device)(packed) -> the reference's collated batch dict on ``device``:
    INPUT_IMAGE_KEY [B,3,S,S] fp32, TARGET_LANDMARKS_HEATMAP [B,C,S/stride,S/stride] uint8, TARGET_2D_LANDMARKS [B,C,2]
    (/ img_size), TARGET_2D_FULL_LANDMARKS [B,V,2] (network pixels), TARGET_2D_LANDMARKS_PRESENCE [B,C] bool,
    TARGET_3D_MODEL_VERTICES [B,V,3], INPUT_BBOX_KEY four [B] int32 (x, y, w, h), SAMPLE_INDEX_KEY [B] int64 and
    IMAGE_FILENAME_KEY.  Copies run from pinned memory on the current stream; nothing synchronises the host."""

    def __init__(self, config: Dict[str, Any], device):
        self.cfg = TargetConfig(config)
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        radius = self.cfg.radius
        self.radius = 1 if radius == "pointwise" else radius
        self.window = torch.from_numpy(heatmap_window(radius)).to(self.device)
        if self.cfg.num_classes == 68:
            from .submission import landmark68_tables
            tri, bary = landmark68_tables()
            self.lm_tri = tri.to(self.device, torch.int32).contiguous()
            self.lm_bary = bary.to(self.device, torch.float32).contiguous()
            self.lm_index = None
            self.max_vertex = int(tri.max())
        else:
            self.lm_index = torch.tensor(self.cfg.keypoints_indices, dtype=torch.int32, device=self.device)
            self.lm_tri = self.lm_bary = None
            self.max_vertex = max(self.cfg.keypoints_indices)
        self.num_classes = int(self.cfg.num_classes)

    def __call__(self, packed: Dict[str, Any]) -> Dict[str, Any]:
        dev, cfg = self.device, self.cfg
        S, C, Sh = cfg.img_size, self.num_classes, cfg.heatmap_size
        crops = _to_device(packed["crops"], dev)
        ints = _to_device(packed["ints"], dev)
        verts = _to_device(packed["vertices"], dev)
        mv = _to_device(packed["model_view"], dev)
        proj = _to_device(packed["projection"], dev)
        indices = _to_device(packed["indices"], dev)
        B, Hc, Wc = (int(d) for d in crops.shape[:3])
        V = int(verts.shape[1])
        if V <= self.max_vertex:
            raise ValueError(f"landmark vertex {self.max_vertex} outside the {V} vertices of the batch")
        boxes, origins, bbox, frame_index = ints.split([4 * B, 3 * B, 4 * B, B])
        rois = torch.empty(B, ROI_RECORD_BYTES, dtype=torch.uint8, device=dev)
        images = torch.empty(B, 3, S, S, dtype=torch.float32, device=dev)
        keypoints = torch.empty(B, V, 2, dtype=torch.float32, device=dev)
        landmarks = torch.empty(B, C, 2, dtype=torch.float32, device=dev)
        landmarks_norm = torch.empty(B, C, 2, dtype=torch.float32, device=dev)
        presence = torch.empty(B, C, dtype=torch.uint8, device=dev)
        heatmap = torch.empty(B, C, Sh, Sh, dtype=torch.uint8, device=dev)
        lib = _lib.load()
        zero_extend = np.zeros(4, np.float64)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(lib.dad3d_roi_setup(boxes.data_ptr(), frame_index.data_ptr(), B, B, Hc, Wc, S, zero_extend.ctypes.data,
                                           rois.data_ptr(), stream), "dad3d_roi_setup")
            _lib.check(lib.dad3d_preprocess_rois(crops.data_ptr(), Hc, Wc, rois.data_ptr(), B, S, cfg.mean255.ctypes.data,
                                                 cfg.inv_std255.ctypes.data, images.data_ptr(), stream),
                       "dad3d_preprocess_rois")
            _lib.check(lib.dad3d_training_targets(
                verts.data_ptr(), mv.data_ptr(), proj.data_ptr(), origins.data_ptr(), rois.data_ptr(), B, V,
                self.lm_index.data_ptr() if self.lm_index is not None else None,
                self.lm_tri.data_ptr() if self.lm_tri is not None else None,
                self.lm_bary.data_ptr() if self.lm_bary is not None else None, C, S, keypoints.data_ptr(),
                landmarks.data_ptr(), landmarks_norm.data_ptr(), presence.data_ptr(), stream), "dad3d_training_targets")
            _lib.check(lib.dad3d_heatmap_targets(landmarks.data_ptr(), presence.data_ptr(), B * C, Sh, cfg.stride,
                                                 self.window.data_ptr(), self.radius, heatmap.data_ptr(), stream),
                       "dad3d_heatmap_targets")
        return {INPUT_IMAGE_KEY: images, TARGET_LANDMARKS_HEATMAP: heatmap, TARGET_2D_LANDMARKS: landmarks_norm,
                TARGET_2D_FULL_LANDMARKS: keypoints, TARGET_2D_LANDMARKS_PRESENCE: presence.view(torch.bool),
                TARGET_3D_MODEL_VERTICES: verts, INPUT_BBOX_KEY: list(bbox.view(4, B).unbind(0)), SAMPLE_INDEX_KEY: indices,
                IMAGE_FILENAME_KEY: list(packed["filenames"])}
