"""numpy model of heads-from-boxes (csrc/roi.cu): crop geometry, the letter-box of a crop, and the read-back of the encoder's
outputs into frame pixels, each restating the reference's dtype sequence.  Pinned against the reference's own functions in
tests/test_roi_model_cpu.py; the GPU tests compare the kernels with it bit for bit."""
from typing import Dict, Sequence

import numpy as np

from dad_3dheads_b200.predictor import _MEAN, _STD
from oracle.resize_oracle import resize_linear_u8

SCALE_IDX, TRANSLATION_IDX = 412, 409                 # the released 413-vector layout (dad_3dnet.yaml)


def crop_box(box: Sequence[int], extend: Sequence[float], H: int, W: int):
    """ensure_bbox_boundaries(extend_bbox(box, extend), (H, W)); extend = (left, right, top, bottom)."""
    x, y, w, h = (np.float64(v) for v in box)
    left, right, top, bottom = (np.float64(v) for v in extend)
    ex = np.array([x - w * left, y - h * top, w * ((1.0 + right) + left), h * ((1.0 + top) + bottom)]).astype(np.int32)
    x1 = min(max(0, int(ex[0])), W)
    y1 = min(max(0, int(ex[1])), H)
    x2 = min(max(0, x1 + int(ex[2])), W)
    y2 = min(max(0, y1 + int(ex[3])), H)
    return x1, y1, x2 - x1, y2 - y1


def geometry(crop, S: int = 256, frame_ok: bool = True) -> Dict[str, float]:
    """The dad3d_roi record of a crop: validity, scale, letter-boxed size, pre- and post-processing paddings."""
    x, y, w, h = crop
    g = dict(x=x, y=y, w=w, h=h, valid=False, scale=1.0, new_h=0, new_w=0, pre_top=0, pre_left=0, post_top=0, post_left=0)
    if not (frame_ok and w > 0 and h > 0):
        return g
    scale = S / float(max(h, w))
    nh, nw = int(np.rint(h * scale)), int(np.rint(w * scale))
    if nh < 1 or nw < 1:                               # cv2.resize refuses a zero-sized destination
        return g
    side = max(nh, nw)
    g.update(valid=True, scale=scale, new_h=nh, new_w=nw,
             pre_top=(S - nh) // 2 if nh < S else 0, pre_left=(S - nw) // 2 if nw < S else 0,
             post_top=(side - nh) // 2, post_left=(side - nw) // 2)
    return g


def letterbox(frame: np.ndarray, g, S: int = 256) -> np.ndarray:
    """[S,S,3] fp32 input image of one ROI: the crop read from the frame, resized with the cv2 restatement, padded and
    normalised; all padding when the ROI is invalid."""
    img = np.zeros((S, S, 3), np.uint8)
    if g["valid"]:
        crop = frame[g["y"]:g["y"] + g["h"], g["x"]:g["x"] + g["w"]]
        if (g["new_h"], g["new_w"]) != (g["h"], g["w"]):
            crop = resize_linear_u8(crop, g["new_h"], g["new_w"])
        img[g["pre_top"]:g["pre_top"] + g["new_h"], g["pre_left"]:g["pre_left"] + g["new_w"]] = crop
    mean = np.array(_MEAN, dtype=np.float32) * np.float32(255.0)
    inv = np.reciprocal(np.array(_STD, dtype=np.float32) * np.float32(255.0), dtype=np.float32)
    return (img.astype(np.float32) - mean) * inv


def readjust_params(params: np.ndarray, g, S: int = 256) -> np.ndarray:
    """[P] fp32 encoder params -> frame-space params: readjust_3dmm_to_the_input_image in fp32 with the scale rounded to
    fp32, translation z zeroed, then + [x, y, 0] * 2 / S."""
    f = np.float32
    p = np.array(params, dtype=np.float32, copy=True)
    sc = f(g["scale"])
    p[SCALE_IDX] = (p[SCALE_IDX] + f(1)) / sc - f(1)
    for k, pad, off in ((0, g["post_left"], g["x"]), (1, g["post_top"], g["y"])):
        t = p[TRANSLATION_IDX + k]
        t = ((t + f(1)) - f(pad) * f(2) / f(S)) / sc - f(1)
        p[TRANSLATION_IDX + k] = t + f(off) * f(2) / f(S)
    p[TRANSLATION_IDX + 2] = f(0)
    return p


def readjust_points(lms: np.ndarray, g) -> np.ndarray:
    """[L,2] encoder landmarks in [0,1] units -> int64 frame pixels: fp32 scale-up and clip, float64 subtract and divide,
    truncation, + [x, y]."""
    lm = np.clip(np.asarray(lms, dtype=np.float32) * np.float32(256.0), np.float32(0), np.float32(256))
    d = (lm.astype(np.float64) - np.array([g["post_left"], g["post_top"]], dtype=np.float64)) / g["scale"]
    return d.astype(np.int64) + np.array([g["x"], g["y"]], dtype=np.int64)
