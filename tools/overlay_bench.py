#!/usr/bin/env python
"""Times the overlays (csrc/overlay.cu) on one GPU: four 1920 x 1080 frames with R = 64 and 512 boxes of 150-400 px.

1. Per kernel, on the predictions of one box step: "pose_geometry_ms" (dad3d_pose_geometry), "points_68_ms",
   "points_191_ms", "points_565_ms" (dad3d_overlay_points into a frame copy), "pose_raster_ms" (dad3d_overlay_pose: key
   memset, pass 1, pass 2) and "frame_copy_ms" (one device copy of the frames).
2. The captured box step ``predict_batch_graphed`` without and with ``overlay=`` all four kinds and ``rpy=True``,
   alternating, three windows each: the time the overlays add.
CUDA events around >= 1 s windows after a warm-up.  Prints the card's name, power limit and maximum SM clock first: the
numbers belong to that card.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from frame_render_bench import F, H, W, card, timed  # noqa: E402

KINDS = ("68_landmarks", "191_landmarks", "445_landmarks", "pose")


def _boxes(R, dev, g):
    side = torch.randint(150, 400, (R,), generator=g)
    boxes = torch.stack([torch.randint(0, W - 150, (R,), generator=g), torch.randint(0, H - 150, (R,), generator=g),
                         side, side], 1).to(dev, torch.int32)
    return boxes, torch.randint(0, F, (R,), generator=g, dtype=torch.int32).to(dev)


def bench_kernels(pred, dev, R):
    from dad_3dheads_b200 import overlay as O
    from dad_3dheads_b200.predictor import ROI_RECORD_BYTES
    from dad_3dheads_b200 import _lib
    import numpy as np
    g = torch.Generator().manual_seed(R)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    boxes, fi = _boxes(R, dev, g)
    out = pred.predict_batch(frames, boxes=boxes, frame_index=fi)
    rois = torch.empty(R, ROI_RECORD_BYTES, dtype=torch.uint8, device=dev)
    ext = np.zeros(4)
    _lib.check(_lib.load().dad3d_roi_setup(boxes.data_ptr(), fi.data_ptr(), R, F, H, W, 256, ext.ctypes.data,
                                           rois.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), "roi_setup")
    params, points, proj = out["3dmm_params"], out["points"], out["projected_vertices"].contiguous()
    ri = pred._rotation_index()
    _, pose = O.pose_geometry(params, ri, rois)
    img = frames.clone()
    res = {"what": "overlay kernels", "frames": [F, H, W], "boxes": R,
           "pose_geometry_ms": timed(lambda: O.pose_geometry(params, ri, rois)),
           "frame_copy_ms": timed(lambda: img.copy_(frames)),
           "points_68_ms": timed(lambda: O.draw_points(img, points, rois)),
           "points_191_ms": timed(lambda: O.draw_points(img, proj, rois, pred._landmark_index("191"))),
           "points_565_ms": timed(lambda: O.draw_points(img, proj, rois, pred._landmark_index("565"))),
           "pose_raster_ms": timed(lambda: O.draw_pose(img, pose))}
    return {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}


def bench_step(pred, dev, R, rounds=3):
    g = torch.Generator().manual_seed(R + 1)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    boxes, fi = _boxes(R, dev, g)
    plain = lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi)              # noqa: E731
    drawn = lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, overlay=KINDS, rpy=True)  # noqa: E731
    res = {"plain": [], "overlay": []}
    for _ in range(rounds):
        res["plain"].append(round(timed(plain), 4))
        res["overlay"].append(round(timed(drawn), 4))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"what": "predict_batch_graphed boxes", "frames": [F, H, W], "boxes": R, "ms_per_step": res,
            "overlay_ms": round(med["overlay"] - med["plain"], 4),
            "overlay_share": round((med["overlay"] - med["plain"]) / med["overlay"], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, nargs="+", default=[64, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("overlay_bench needs a GPU")
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG, FaceMeshPredictor
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card:", card())
    pred = FaceMeshPredictor(dict(DEFAULT_CONFIG), cuda_id=0, state_dict=synthetic_state_dict(0), precision="fp16x2")
    for R in args.boxes:
        print(json.dumps(bench_kernels(pred, dev, R)))
    for R in args.boxes:
        print(json.dumps(bench_step(pred, dev, R)))


if __name__ == "__main__":
    main()
