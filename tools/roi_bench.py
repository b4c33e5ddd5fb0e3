#!/usr/bin/env python
"""Times heads-from-boxes (csrc/roi.cu) on one GPU, from four 1920x1080 frames.

1. The three ROI kernels alone at R = 64 and 512 boxes: ``dad3d_roi_setup``, ``dad3d_preprocess_rois`` (writes the
   [R,3,256,256] fp32 encoder input) and ``dad3d_readjust_rois``, on preallocated buffers.  CUDA events around >= 1 s
   windows after a warm-up; the pre-processing also as bytes moved (fp32 output + uint8 crop pixels read) per second.
2. The captured step: ``predict_batch_graphed(frames, boxes=...)`` against ``predict_batch_graphed`` on the same heads
   pre-cropped to [R,256,256,3] uint8 (fp16x2 encoder), both from pinned host memory and both from device memory,
   alternating, three windows each; with the host-to-device bytes of each input.

Prints the card's name, power limit and maximum SM clock first: the numbers belong to that card.
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
from render_bench import card, timed  # noqa: E402

F, H, W, S = 4, 1080, 1920, 256


def boxes_for(R, seed):
    g = np.random.default_rng(seed)
    side = g.integers(120, 600, R)
    b = np.stack([g.integers(0, W - 600, R), g.integers(0, H - 600, R), side, (side * g.uniform(1.0, 1.4, R)).astype(int)], 1)
    return torch.from_numpy(b.astype(np.int32)), torch.from_numpy(g.integers(0, F, R).astype(np.int32))


def kernel_times(pred, frames_d, R):
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.predictor import _MEAN, _STD, ROI_RECORD_BYTES
    lib = _lib.load()
    dev = pred.device
    boxes, fi = (t.to(dev) for t in boxes_for(R, R))
    rois = torch.empty(R, ROI_RECORD_BYTES, dtype=torch.uint8, device=dev)
    x = torch.empty(R, 3, S, S, device=dev)
    params = torch.randn(R, 413, device=dev)
    lms = torch.rand(R, 68, 2, device=dev)
    p_out = torch.empty_like(params)
    pts = torch.empty(R, 68, 2, dtype=torch.int64, device=dev)
    ext = np.array([0.1] * 4)
    mean = (np.array(_MEAN, dtype=np.float32) * 255.0).astype(np.float32)
    inv = np.reciprocal(np.array(_STD, dtype=np.float32) * 255.0, dtype=np.float32)
    st = torch.cuda.current_stream(dev).cuda_stream

    def setup():
        _lib.check(lib.dad3d_roi_setup(boxes.data_ptr(), fi.data_ptr(), R, F, H, W, S, ext.ctypes.data, rois.data_ptr(), st),
                   "setup")

    def pre():
        _lib.check(lib.dad3d_preprocess_rois(frames_d.data_ptr(), H, W, rois.data_ptr(), R, S, mean.ctypes.data,
                                             inv.ctypes.data, x.data_ptr(), st), "preprocess")

    def readjust():
        _lib.check(lib.dad3d_readjust_rois(params.data_ptr(), lms.data_ptr(), rois.data_ptr(), R, 413, 68, 412, 409, S,
                                           p_out.data_ptr(), pts.data_ptr(), st), "readjust")

    setup()
    torch.cuda.synchronize()
    rec = rois.view(torch.int32).cpu()
    read = int((rec[:, 6] * rec[:, 7]).sum()) * 3 * 4          # <= 4 bilinear taps of 3 bytes per resized pixel (upper bound)
    out = {"R": R, "setup_ms": timed(setup), "preprocess_ms": timed(pre), "readjust_ms": timed(readjust)}
    out["preprocess_GBps_fp32_out"] = R * 3 * S * S * 4 / out["preprocess_ms"] / 1e6
    out["preprocess_bytes_out"] = R * 3 * S * S * 4
    out["preprocess_bytes_read_upper_bound"] = read
    return out


def step_times(pred, frames_h, R, reps=3):
    dev = pred.device
    boxes, fi = boxes_for(R, R + 1)
    crops = torch.from_numpy(np.random.default_rng(R).integers(0, 256, (R, S, S, 3), dtype=np.uint8)).pin_memory()
    frames_d, crops_d = frames_h.to(dev), crops.to(dev)
    boxes_d, fi_d = boxes.to(dev), fi.to(dev)
    legs = {
        "boxes_host": lambda: pred.predict_batch_graphed(frames_h, boxes=boxes, frame_index=fi, extend=0.1),
        "crops_host": lambda: pred.predict_batch_graphed(crops),
        "boxes_device": lambda: pred.predict_batch_graphed(frames_d, boxes=boxes_d, frame_index=fi_d, extend=0.1),
        "crops_device": lambda: pred.predict_batch_graphed(crops_d),
    }
    res = {k: [] for k in legs}
    for _ in range(reps):
        for k, fn in legs.items():
            res[k].append(round(timed(fn), 4))
    return {"R": R, "step_ms": res,
            "h2d_bytes": {"boxes": frames_h.numel() + boxes.numel() * 4 + fi.numel() * 4, "crops": crops.numel()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "roi_bench needs a GPU"
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    print("card:", card(), flush=True)
    pred = FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0), precision="fp16x2")
    frames_h = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (F, H, W, 3), dtype=np.uint8)).pin_memory()
    frames_d = frames_h.to(pred.device)
    res = {"card": card(), "kernels": [], "steps": []}
    for R in (64, 512):
        k = kernel_times(pred, frames_d, R)
        print(json.dumps(k), flush=True)
        res["kernels"].append(k)
    for R in (64, 512):
        s = step_times(pred, frames_h, R)
        print(json.dumps(s), flush=True)
        res["steps"].append(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
