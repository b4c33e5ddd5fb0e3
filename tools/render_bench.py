#!/usr/bin/env python
"""Times the batched rasteriser and its share of the captured predict step, on one GPU.

1. ``rasterize_batch`` rendering PNCC + depth + tri_index at 256x256 for B = 64 and 512 decoded heads: the whole call
   (output allocation and fills included) and the library call alone (key memset + the two kernels) on preallocated
   buffers.  CUDA events around >= 1 s windows after a warm-up.  Reports heads/s and the bytes the kernels must move
   (key memset + image, depth and tri_index stores, from the shapes) over that time.
2. ``predict_batch_graphed`` at batch 64 (raw 256x256 uint8 frames, fp16x2 encoder) without and with
   ``render=("pncc", "depth", "tri_index")``, alternating, three windows each.
3. ``--profile``: one eager rendered step under torch.profiler, the top CUDA kernels by device time.

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

RENDER = ("pncc", "depth", "tri_index")


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


def heads(B, dev):
    """B decoded heads in the 256x256 network frame, [B,5023,3] as HeadMesh.decode(to_2d=False) returns them, with scales
    that make a head cover roughly 10-40 % of the image."""
    from dad_3dheads_b200.head_mesh import HeadMesh
    from oracle.flame_oracle import sample_params
    p = sample_params(B, seed=7)
    p[:, 409:411] *= 0.3
    p[:, 412] = torch.linspace(2.0, 4.0, B)
    return HeadMesh(cuda_id=dev.index).decode(p.to(dev), to_2d=False)[1].contiguous()


def bench_raster(dev, B, S=256):
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.rasterizer import PnccRenderer, rasterize_batch
    r = PnccRenderer(dev)
    v = heads(B, dev)
    lib = _lib.load()
    img = torch.zeros(B, S, S, 3, dtype=torch.uint8, device=dev)
    depth = torch.full((B, S, S), -1e8, device=dev)
    tri = torch.empty(B, S, S, dtype=torch.int32, device=dev)
    key = torch.empty(B * S * S, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    nv, ntri = int(v.shape[1]), int(r.faces.shape[0])

    def kernels():
        _lib.check(lib.dad3d_rasterize_batch(v.data_ptr(), nv, B, r.faces.data_ptr(), ntri, r.colors.data_ptr(), 3, S, S, 0,
                                             1, img.data_ptr(), depth.data_ptr(), tri.data_ptr(), key.data_ptr(), stream),
                   "dad3d_rasterize_batch")

    def call():
        rasterize_batch(v, r.faces, r.colors, height=S, width=S, negate_z=True)

    ms_k, ms_c = timed(kernels), timed(call)
    px = B * S * S
    nbytes = px * (8 + 3 + 4 + 4)                   # key memset + pncc + depth + tri_index stores
    cover = (r(v, S)["tri_index"] >= 0).float().mean().item()
    return {"what": "rasterize_batch", "B": B, "size": S, "covered": round(cover, 3), "kernels_ms": round(ms_k, 4),
            "call_ms": round(ms_c, 4), "heads_per_s_kernels": round(B / ms_k * 1e3), "heads_per_s_call": round(B / ms_c * 1e3),
            "min_bytes": nbytes, "gb_per_s_kernels": round(nbytes / ms_k / 1e6, 1)}


def bench_step(dev, B=64, rounds=3):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG, FaceMeshPredictor
    pred = FaceMeshPredictor(dict(DEFAULT_CONFIG), cuda_id=dev.index, state_dict=synthetic_state_dict(0), precision="fp16x2")
    g = torch.Generator().manual_seed(1234)
    x = torch.randint(0, 256, (B, 256, 256, 3), generator=g, dtype=torch.uint8).to(dev)
    arms = {"plain": dict(to_2d=False), "render": dict(to_2d=False, render=RENDER)}
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, kw in arms.items():
            res[k].append(round(timed(lambda: pred.predict_batch_graphed(x, **kw)), 4))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return pred, x, {"what": "predict_batch_graphed", "B": B, "ms_per_step": res,
                     "render_share": round((med["render"] - med["plain"]) / med["render"], 4),
                     "heads_per_s": {k: round(B / m * 1e3) for k, m in med.items()}}


def profile(pred, x):
    from torch.profiler import ProfilerActivity, profile as prof
    for _ in range(3):
        pred.predict_batch(x, to_2d=False, render=RENDER)
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        pred.predict_batch(x, to_2d=False, render=RENDER)
        torch.cuda.synchronize()
    print(p.key_averages().table(sort_by="cuda_time_total", row_limit=15))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 512])
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_bench needs a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card:", card())
    for B in args.batches:
        print(json.dumps(bench_raster(dev, B)))
    pred, x, step = bench_step(dev)
    print(json.dumps(step))
    if args.profile:
        profile(pred, x)


if __name__ == "__main__":
    main()
