#!/usr/bin/env python
"""Times the head and face wireframes (dad3d_overlay_mesh, csrc/overlay.cu) on one GPU: four 1920 x 1080 frames with R = 64
and 512 boxes.

1. Per kind, the kernel time (per-box pass plus tile pass, into a frame copy) for two kinds of heads: the predictions of
   one box step with the synthetic weights (boxes of 150-400 px; those weights do not give head-shaped wireframes), and
   FLAME template heads scaled to 60 px, 150-400 px and 1000 px -- the density of a real wireframe.
2. The captured box step ``predict_batch_graphed`` without and with ``overlay=("head_mesh", "face_mesh")``, alternating,
   three windows each: the time the wireframes add.
CUDA events around >= 1 s windows after a warm-up.  Prints the card's name, power limit and maximum SM clock first: the
numbers belong to that card.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from frame_render_bench import F, H, W, card, timed  # noqa: E402
from overlay_bench import _boxes  # noqa: E402

KINDS = ("head_mesh", "face_mesh")


def _template_heads(static, R, size, g):
    """[R, 5023, 2] fp32: the FLAME template seen from the front, its face-with-ears part ``size`` px (an int, or a
    (lo, hi) range drawn per head) wide, placed at random in the frame."""
    v = static["v_template"][:, :2].astype(np.float64) * [1, -1]
    sub = v[static["flame_indices_face_w_ears"]]
    v = (v - sub.min(0)) / (sub.max(0) - sub.min(0)).max()
    s = g.uniform(*size, R) if isinstance(size, tuple) else np.full(R, float(size))
    org = np.stack([g.uniform(-0.1, 1, R) * (W - 0.9 * s), g.uniform(-0.1, 1, R) * (H - 0.9 * s)], -1)
    return (v[None] * s[:, None, None] + org[:, None, :]).astype(np.float32)


def bench_kernels(pred, dev, R):
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200 import overlay as O
    from dad_3dheads_b200.predictor import ROI_RECORD_BYTES
    g = torch.Generator().manual_seed(R)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    boxes, fi = _boxes(R, dev, g)
    out = pred.predict_batch(frames, boxes=boxes, frame_index=fi)
    rois = torch.empty(R, ROI_RECORD_BYTES, dtype=torch.uint8, device=dev)
    _lib.check(_lib.load().dad3d_roi_setup(boxes.data_ptr(), fi.data_ptr(), R, F, H, W, 256, np.zeros(4).ctypes.data,
                                           rois.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "roi_setup")
    pred._mesh_edges("head_mesh")
    static = pred._static
    rng = np.random.default_rng(R)
    heads = {"synthetic": out["projected_vertices"].contiguous()}
    for name, size in (("template_60", 60), ("template_150_400", (150.0, 400.0)), ("template_1000", 1000)):
        heads[name] = torch.from_numpy(_template_heads(static, R, size, rng)).to(dev)
    img = frames.clone()
    res = {"what": "wireframe kernels", "frames": [F, H, W], "boxes": R}
    for name, v in heads.items():
        for k in KINDS:
            e = pred._mesh_edges(k)
            res[f"{k}_{name}_ms"] = round(timed(lambda: O.draw_mesh(img, v, rois, e)), 4)
    return res


def bench_step(pred, dev, R, rounds=3):
    g = torch.Generator().manual_seed(R + 1)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    boxes, fi = _boxes(R, dev, g)
    plain = lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi)              # noqa: E731
    drawn = lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, overlay=KINDS)  # noqa: E731
    res = {"plain": [], "wireframes": []}
    for _ in range(rounds):
        res["plain"].append(round(timed(plain), 4))
        res["wireframes"].append(round(timed(drawn), 4))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"what": "predict_batch_graphed boxes", "frames": [F, H, W], "boxes": R, "ms_per_step": res,
            "wireframes_ms": round(med["wireframes"] - med["plain"], 4),
            "wireframes_share": round((med["wireframes"] - med["plain"]) / med["wireframes"], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, nargs="+", default=[64, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wireframe_bench needs a GPU")
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG, FaceMeshPredictor
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card:", card())
    pred = FaceMeshPredictor(dict(DEFAULT_CONFIG), cuda_id=0, state_dict=synthetic_state_dict(0), precision="fp16x2")
    for R in args.boxes:
        print(json.dumps(bench_kernels(pred, dev, R)), flush=True)
    for R in args.boxes:
        print(json.dumps(bench_step(pred, dev, R)), flush=True)


if __name__ == "__main__":
    main()
