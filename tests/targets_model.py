"""Exact numpy model of the training-target kernels (csrc/targets.cu) and of the batch FlameBatchBuilder assembles.

Every float operation is one numpy float32 (or, where numpy promotes, float64) operation in the kernels' order, so the GPU
tests compare the kernels with this model bit for bit; tests/test_targets_model_cpu.py pins the model against the live
reference FlameDataset, HeatmapCoder and draw_gaussian."""
from typing import Any, Dict, Optional, Tuple

import numpy as np

from dad_3dheads_b200.training_data import (IMAGE_FILENAME_KEY, INPUT_BBOX_KEY, INPUT_IMAGE_KEY, SAMPLE_INDEX_KEY,
                                             TARGET_2D_FULL_LANDMARKS, TARGET_2D_LANDMARKS, TARGET_2D_LANDMARKS_PRESENCE,
                                             TARGET_3D_MODEL_VERTICES, TARGET_LANDMARKS_HEATMAP, TargetConfig,
                                             heatmap_window)
from oracle.resize_oracle import resize_linear_u8
from tests.roi_model import geometry

f32 = np.float32


def fma32(a, b, c):
    """Correctly rounded float32 a * b + c: the product is exact in float64; where the float64 sum rounded, it is nudged one
    float64 ulp toward the exact value, so the rounding to float32 sees which side of a float32 midpoint the sum lies on."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                                # TwoSum: s + err == p + c exactly
    s = np.where(err == 0, s, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)))
    return s.astype(f32)


def _row(m, r, x, y, z, w):
    """One product, then an fma per term in k order (csrc/targets.cu mat_row)."""
    return fma32(m[r, 3], w, fma32(m[r, 2], z, fma32(m[r, 1], y, m[r, 0] * x)))


def to_world(mv: np.ndarray, v: np.ndarray) -> np.ndarray:
    """[N,3] model space -> [N,4] world_homo = model_view @ [v, 1], each row summed left to right in fp32."""
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    one = np.ones_like(x)
    return np.stack([_row(mv, r, x, y, z, one) for r in range(4)], -1)


def project(P: np.ndarray, X: np.ndarray, crop_x: int, crop_y: int, frame_h: int) -> np.ndarray:
    """[N,4] -> [N,2] crop pixels: fp32 P @ X, divide by w, fp32 height - y, float64 minus the crop origin, back to fp32."""
    cx = _row(P, 0, X[:, 0], X[:, 1], X[:, 2], X[:, 3])
    cy = _row(P, 1, X[:, 0], X[:, 1], X[:, 2], X[:, 3])
    cw = _row(P, 3, X[:, 0], X[:, 1], X[:, 2], X[:, 3])
    px = cx / cw
    py = f32(frame_h) - cy / cw
    return np.stack([(px.astype(np.float64) - crop_x).astype(f32), (py.astype(np.float64) - crop_y).astype(f32)], -1)


def to_network(p: np.ndarray, g: Dict[str, Any]) -> np.ndarray:
    s = f32(g["scale"])
    return np.stack([p[:, 0] * s + f32(g["pre_left"]), p[:, 1] * s + f32(g["pre_top"])], -1)


def head_targets(verts, mv, P, crop, frame_h: int, S: int, lm_index=None, lm_tri=None, lm_bary=None):
    """One head -> (keypoints [V,2], landmarks [C,2] network pixels, landmarks / S, presence [C] bool)."""
    with np.errstate(all="ignore"):
        x, y, w, h = crop
        g = geometry((0, 0, w, h), S)
        world = to_world(mv, verts)
        keypoints = to_network(project(P, world, x, y, frame_h), g)
        if lm_tri is not None:
            acc = None
            for k in range(3):
                t = world[lm_tri[:, k], :3] * lm_bary[:, k:k + 1]
                acc = t if acc is None else acc + t
            X = np.concatenate([acc, np.ones_like(acc[:, :1])], -1)
        else:
            X = world[lm_index]
        c = project(P, X, x, y, frame_h)
        presence = (c[:, 0] > 0) & (c[:, 0] < f32(w)) & (c[:, 1] > 0) & (c[:, 1] < f32(h))
        lm = to_network(c, g)
        return keypoints, lm, lm / f32(S), presence


def heat_cell(p, stride: int) -> Optional[int]:
    """numpy's float32 floor division (npy_divmodf) then int(); None where int() would raise; clamped to +-2^24."""
    p, b = f32(p), f32(stride)
    if not np.isfinite(p):
        return None
    with np.errstate(all="ignore"):
        mod = np.fmod(p, b)
        div = (p - mod) / b
        if mod != 0 and ((b < 0) != (mod < 0)):
            div = div - f32(1)
        fl = f32(0)
        if div != 0:
            fl = np.floor(div)
            if div - fl > f32(0.5):
                fl = fl + f32(1)
    return int(min(max(fl, f32(-16777216.0)), f32(16777216.0)))


def _bound(i: int, n: int) -> int:
    return max(i + n, 0) if i < 0 else min(i, n)


def window_span(c: int, r: int, S: int) -> Tuple[int, int, int]:
    """draw_gaussian's row or column ranges as Python slices normalise them -> (plane start, window start, length)."""
    D = 2 * r + 1
    lo, hi = min(c, r), min(S - c, r + 1)
    hs, he, gs, ge = _bound(c - lo, S), _bound(c + hi, S), _bound(r - lo, D), _bound(r + hi, D)
    n = max(he - hs, 0) if he - hs == ge - gs else 0
    return hs, gs, n


def heatmap_plane(lm, present: bool, S: int, stride: int, table: np.ndarray, radius: int) -> np.ndarray:
    out = np.zeros((S, S), np.uint8)
    if not present:
        return out
    cx, cy = heat_cell(lm[0], stride), heat_cell(lm[1], stride)
    if cx is None or cy is None:
        return out
    (hx, gx, nx), (hy, gy, ny) = window_span(cx, radius, S), window_span(cy, radius, S)
    if nx and ny:
        out[hy:hy + ny, hx:hx + nx] = table[gy:gy + ny, gx:gx + nx]
    return out


def heatmaps(landmarks: np.ndarray, presence: np.ndarray, S: int, stride: int, radius) -> np.ndarray:
    """[B,C,2] network pixels, [B,C] -> [B,C,S,S] uint8 (radius an int or "pointwise")."""
    table = heatmap_window(radius)
    r = 1 if radius == "pointwise" else radius
    B, C = presence.shape
    out = np.zeros((B, C, S, S), np.uint8)
    for b in range(B):
        for c in range(C):
            out[b, c] = heatmap_plane(landmarks[b, c], bool(presence[b, c]), S, stride, table, r)
    return out


def letterbox(crop: np.ndarray, S: int, mean255: np.ndarray, inv_std255: np.ndarray) -> np.ndarray:
    """[h,w,3] uint8 -> [3,S,S] fp32: LongestMaxSize (cv2 INTER_LINEAR restated), centred PadIfNeeded, Normalize."""
    h, w = crop.shape[:2]
    g = geometry((0, 0, w, h), S)
    img = np.zeros((S, S, 3), np.uint8)
    if (g["new_h"], g["new_w"]) != (h, w):
        crop = resize_linear_u8(crop, g["new_h"], g["new_w"])
    img[g["pre_top"]:g["pre_top"] + g["new_h"], g["pre_left"]:g["pre_left"] + g["new_w"]] = crop
    return ((img.astype(f32) - mean255) * inv_std255).transpose(2, 0, 1)


def build_batch(packed: Dict[str, Any], config: Dict[str, Any], lm_tri=None, lm_bary=None) -> Dict[str, Any]:
    """The dict FlameBatchBuilder returns, as numpy arrays (INPUT_BBOX_KEY a list of four arrays, filenames a list)."""
    cfg = TargetConfig(config)
    S, C = cfg.img_size, int(cfg.num_classes)
    crops = packed["crops"].numpy()
    B = crops.shape[0]
    ints = packed["ints"].numpy()
    origins = ints[4 * B:7 * B].reshape(B, 3)
    bbox = ints[7 * B:11 * B].reshape(4, B)
    verts, mv, P = (packed[k].numpy() for k in ("vertices", "model_view", "projection"))
    index = None if C == 68 else np.asarray(cfg.keypoints_indices)
    images, kps, lms, norms, pres = [], [], [], [], []
    for b in range(B):
        x, y, w, h = (int(v) for v in bbox[:, b])
        images.append(letterbox(crops[b, :h, :w], S, cfg.mean255, cfg.inv_std255))
        k, lm, n, p = head_targets(verts[b], mv[b], P[b], (x, y, w, h), int(origins[b, 2]), S, lm_index=index,
                                   lm_tri=lm_tri, lm_bary=lm_bary)
        kps.append(k)
        lms.append(lm)
        norms.append(n)
        pres.append(p)
    lms, pres = np.stack(lms), np.stack(pres)
    return {INPUT_IMAGE_KEY: np.stack(images),
            TARGET_LANDMARKS_HEATMAP: heatmaps(lms, pres, cfg.heatmap_size, cfg.stride, cfg.radius),
            TARGET_2D_LANDMARKS: np.stack(norms), TARGET_2D_FULL_LANDMARKS: np.stack(kps),
            TARGET_2D_LANDMARKS_PRESENCE: pres, TARGET_3D_MODEL_VERTICES: verts,
            INPUT_BBOX_KEY: [bbox[i] for i in range(4)], SAMPLE_INDEX_KEY: packed["indices"].numpy(),
            IMAGE_FILENAME_KEY: list(packed["filenames"]), "landmarks_px": lms}
