#!/usr/bin/env python
"""Times the whole-frame render (PnccRenderer.render_frames / dad3d_rasterize_frames) and its share of the captured box step,
on one GPU.

1. Four 1920x1080 frames with B = 64 and 512 decoded heads of realistic size (150-400 px wide) at random places, each on a
   random frame, drawing PNCC + depth + tri_index + head_index:
   - "call_ms": render_frames as a caller uses it (output allocation, the fills, key memset and the two launches);
   - "fills_kernels_ms": on preallocated buffers, the fills (pncc = 0, depth = -1e8), the key memset and the two launches.
   CUDA events around >= 1 s windows after a warm-up.  Bytes the work must move at least, from the shapes:
       min_bytes = 38 * F*H*W + 12 * covered
   per frame pixel: pncc fill 3 + depth fill 4 + key memset 8 + key read 8 + pncc 3, depth 4, tri_index 4 and head_index 4
   stores = 38 B; per covered pixel (head_index >= 0): at least one 8-byte key atomic and one 4-byte depth-buffer read in
   pass 1 = 12 B.
2. ``predict_batch_graphed`` with 64 boxes on four 1920x1080 frames (fp16x2 encoder, to_2d=False), without and with
   ``frame_render`` of all four maps, alternating, three windows each.

Prints the card's name, power limit and maximum SM clock first: the numbers belong to that card.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAPS = ("pncc", "depth", "tri_index", "head_index")
F, H, W = 4, 1080, 1920


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, min_s=1.0, warmup=3):
    """Mean ms per call over a window of at least ``min_s`` seconds (CUDA events)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    n = 1
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= 1e3 * min_s:
            return ms / n
        n = max(2 * n, int(n * 1.2e3 * min_s / max(ms, 1e-3)))


def frame_heads(B, dev, seed=7):
    """B decoded heads [B,5023,3] (HeadMesh.decode(to_2d=False) layout), each scaled to 150-400 px wide and placed at a
    random point of a 1920x1080 frame (some cut by the border), and a random frame for each."""
    from dad_3dheads_b200.head_mesh import HeadMesh
    from oracle.flame_oracle import sample_params
    g = torch.Generator().manual_seed(seed)
    p = sample_params(B, seed=seed)
    p[:, 409:411] = 0.0
    p[:, 412] = 1.0
    v = HeadMesh(cuda_id=dev.index).decode(p.to(dev), to_2d=False)[1]
    xy = v[..., :2]
    centre = (xy.amax(1) + xy.amin(1)) / 2
    width = (xy[..., 0].amax(1) - xy[..., 0].amin(1))
    scale = (torch.rand(B, generator=g) * 250 + 150).to(dev) / width
    at = torch.stack([torch.rand(B, generator=g) * W, torch.rand(B, generator=g) * H], 1).to(dev)
    out = v.clone()
    out[..., :2] = (xy - centre[:, None]) * scale[:, None, None] + at[:, None]
    out[..., 2] = v[..., 2] * scale[:, None]
    frame = torch.randint(0, F, (B,), generator=g, dtype=torch.int32).to(dev)
    return out.contiguous(), frame


def bench_render(dev, B):
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.rasterizer import PnccRenderer
    r = PnccRenderer(dev)
    v, frame = frame_heads(B, dev)
    lib = _lib.load()
    img = torch.empty(F, H, W, 3, dtype=torch.uint8, device=dev)
    depth = torch.empty(F, H, W, device=dev)
    tri = torch.empty(F, H, W, dtype=torch.int32, device=dev)
    head = torch.empty(F, H, W, dtype=torch.int32, device=dev)
    key = torch.empty(F * H * W, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    nv, ntri = int(v.shape[1]), int(r.faces.shape[0])

    def kernels():
        img.zero_()
        depth.fill_(-1e8)
        _lib.check(lib.dad3d_rasterize_frames(v.data_ptr(), nv, B, r.faces.data_ptr(), ntri, r.colors.data_ptr(), 3,
                                              frame.data_ptr(), F, H, W, 1, img.data_ptr(), depth.data_ptr(),
                                              tri.data_ptr(), head.data_ptr(), key.data_ptr(), stream),
                   "dad3d_rasterize_frames")

    def call():
        r.render_frames(v, frame, F, (H, W))

    ms_k, ms_c = timed(kernels), timed(call)
    maps = r.render_frames(v, frame, F, (H, W))
    assert torch.equal(maps["head_index"], head) and torch.equal(maps["pncc"], img)
    covered = int((maps["head_index"] >= 0).sum())
    nbytes = 38 * F * H * W + 12 * covered
    return {"what": "render_frames", "frames": [F, H, W], "heads": B, "covered_px": covered,
            "covered_share": round(covered / (F * H * W), 3), "call_ms": round(ms_c, 4),
            "fills_kernels_ms": round(ms_k, 4), "min_bytes": nbytes, "gb_per_s_fills_kernels": round(nbytes / ms_k / 1e6, 1),
            "gb_per_s_call": round(nbytes / ms_c / 1e6, 1)}


def bench_step(dev, R=64, rounds=3):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG, FaceMeshPredictor
    pred = FaceMeshPredictor(dict(DEFAULT_CONFIG), cuda_id=dev.index, state_dict=synthetic_state_dict(0), precision="fp16x2")
    g = torch.Generator().manual_seed(1234)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    side = torch.randint(150, 400, (R,), generator=g)
    boxes = torch.stack([torch.randint(0, W - 150, (R,), generator=g), torch.randint(0, H - 150, (R,), generator=g),
                         side, side], 1).to(dev, torch.int32)
    fi = torch.randint(0, F, (R,), generator=g, dtype=torch.int32).to(dev)
    arms = {"plain": dict(to_2d=False), "frame_render": dict(to_2d=False, frame_render=MAPS)}
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, kw in arms.items():
            res[k].append(round(timed(lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, **kw)), 4))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"what": "predict_batch_graphed boxes", "frames": [F, H, W], "boxes": R, "ms_per_step": res,
            "frame_render_ms": round(med["frame_render"] - med["plain"], 4),
            "frame_render_share": round((med["frame_render"] - med["plain"]) / med["frame_render"], 4),
            "heads_per_s": {k: round(R / m * 1e3) for k, m in med.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", type=int, nargs="+", default=[64, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_render_bench needs a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card:", card())
    for B in args.heads:
        print(json.dumps(bench_render(dev, B)))
    print(json.dumps(bench_step(dev)))


if __name__ == "__main__":
    main()
