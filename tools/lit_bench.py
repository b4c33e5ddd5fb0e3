#!/usr/bin/env python
"""Times the lit render (LitRenderer: dad3d_light_batch + the two raster passes in dad3d_render_lit) on one GPU.

1. B = 64 and 512 decoded heads at 256 x 256, one image each: "light_ms" (dad3d_light_batch alone) and "call_ms"
   (LitRenderer.__call__: output allocation and fill, light, key memset and both passes).
2. Four 1920 x 1080 frames with B = 64 and 512 heads of 150-400 px (tools/frame_render_bench.py's placement): the same
   two numbers for LitRenderer.render_frames over black.
3. The captured steps: ``predict_batch_graphed`` at batch 64 (256 x 256 inputs) without and with ``render=("lit",)``, and
   with 64 boxes on four 1920 x 1080 frames without and with ``frame_render=("lit",)``, alternating, three windows each.
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

from frame_render_bench import F, H, W, card, frame_heads, timed  # noqa: E402


def _light_fn(r, v):
    from dad_3dheads_b200.rasterizer import light_batch
    return lambda: light_batch(v, r.faces, negate_z=True)


def bench_network_size(dev, B, S=256):
    from dad_3dheads_b200.rasterizer import LitRenderer
    r = LitRenderer(dev)
    v, _ = frame_heads(B, dev)
    v[..., :2] = v[..., :2] * (S / 1920.0)               # same heads, shrunk into an S x S image
    v = v.contiguous()
    light_ms, call_ms = timed(_light_fn(r, v)), timed(lambda: r(v, S))
    covered = int(r(v, S)["lit"].any(-1).sum())
    return {"what": "LitRenderer", "size": S, "heads": B, "covered_px": covered, "light_ms": round(light_ms, 4),
            "call_ms": round(call_ms, 4)}


def bench_frames(dev, B):
    from dad_3dheads_b200.rasterizer import LitRenderer
    r = LitRenderer(dev)
    v, frame = frame_heads(B, dev)
    light_ms = timed(_light_fn(r, v))
    call_ms = timed(lambda: r.render_frames(v, frame, F, (H, W)))
    return {"what": "LitRenderer.render_frames", "frames": [F, H, W], "heads": B, "light_ms": round(light_ms, 4),
            "call_ms": round(call_ms, 4)}


def _step_pair(fn_plain, fn_lit, rounds):
    res = {"plain": [], "lit": []}
    for _ in range(rounds):
        res["plain"].append(round(timed(fn_plain), 4))
        res["lit"].append(round(timed(fn_lit), 4))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return res, round(med["lit"] - med["plain"], 4), round((med["lit"] - med["plain"]) / med["lit"], 4)


def bench_steps(dev, rounds=3):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG, FaceMeshPredictor
    pred = FaceMeshPredictor(dict(DEFAULT_CONFIG), cuda_id=dev.index, state_dict=synthetic_state_dict(0), precision="fp16x2")
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(64, 3, 256, 256, generator=g).to(dev)
    res, add, share = _step_pair(lambda: pred.predict_batch_graphed(x, to_2d=False),
                                 lambda: pred.predict_batch_graphed(x, to_2d=False, render=("lit",)), rounds)
    out = [{"what": "predict_batch_graphed batch 64", "ms_per_step": res, "lit_ms": add, "lit_share": share}]
    R = 64
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    side = torch.randint(150, 400, (R,), generator=g)
    boxes = torch.stack([torch.randint(0, W - 150, (R,), generator=g), torch.randint(0, H - 150, (R,), generator=g),
                         side, side], 1).to(dev, torch.int32)
    fi = torch.randint(0, F, (R,), generator=g, dtype=torch.int32).to(dev)
    res, add, share = _step_pair(
        lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, to_2d=False),
        lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, to_2d=False, frame_render=("lit",)), rounds)
    out.append({"what": "predict_batch_graphed 64 boxes", "frames": [F, H, W], "ms_per_step": res, "frame_lit_ms": add,
                "frame_lit_share": share})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", type=int, nargs="+", default=[64, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lit_bench needs a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card:", card())
    for B in args.heads:
        print(json.dumps(bench_network_size(dev, B)))
    for B in args.heads:
        print(json.dumps(bench_frames(dev, B)))
    for r in bench_steps(dev):
        print(json.dumps(r))


if __name__ == "__main__":
    main()
