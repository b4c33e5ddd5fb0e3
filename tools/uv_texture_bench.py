#!/usr/bin/env python
"""Times the UV textures (csrc/uv_texture.cu) on one GPU, on tools/overlay_bench.py's workload: four 1920 x 1080 frames
with 64 boxes of 150-400 px.

1. The captured box step ``predict_batch_graphed(to_2d=False)`` without and with ``uv_texture=``, alternating, three
   windows each (CUDA events around >= 1 s windows after a warm-up): the time the textures add.
2. In a separate run under ``torch.profiler``: each kernel's mean time and its share of the HBM bound, the least time the
   bytes it must move take at 3.35 TB/s (the texture it writes, the vertices it reads, the table once per call).
3. The reference's ``_compute_texture_map`` loop per head on the host (on tests/psbody_mesh.py's ``Mesh``), for scale.
Prints the card's name, power limit and maximum SM clock first: the numbers belong to that card.  The JSON goes to
``uv_texture_bench_out/`` (``--out``).
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from frame_render_bench import F, H, W, card, timed  # noqa: E402
from overlay_bench import _boxes  # noqa: E402

HBM_BYTES_PER_S = 3.35e12                       # H100 SXM data sheet


def bench_step(pred, dev, R, table, rounds=3):
    g = torch.Generator().manual_seed(R + 1)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    boxes, fi = _boxes(R, dev, g)
    plain = lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, to_2d=False)   # noqa: E731
    uv = lambda: pred.predict_batch_graphed(frames, boxes=boxes, frame_index=fi, to_2d=False, uv_texture=table)  # noqa: E731
    res = {"plain": [], "uv_texture": []}
    for _ in range(rounds):
        res["plain"].append(round(timed(plain), 4))
        res["uv_texture"].append(round(timed(uv), 4))
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"what": "predict_batch_graphed boxes, to_2d=False", "frames": [F, H, W], "boxes": R, "ms_per_step": res,
            "uv_texture_ms": round(med["uv_texture"] - med["plain"], 4),
            "uv_texture_share": round((med["uv_texture"] - med["plain"]) / med["uv_texture"], 4)}


def bench_kernels(pred, dev, R, table, calls=50):
    from torch.profiler import ProfilerActivity, profile
    from dad_3dheads_b200.uv_texture import uv_textures
    g = torch.Generator().manual_seed(R)
    frames = torch.randint(0, 256, (F, H, W, 3), generator=g, dtype=torch.uint8).to(dev)
    boxes, fi = _boxes(R, dev, g)
    out = pred.predict_batch(frames, boxes=boxes, frame_index=fi, to_2d=False)
    v, valid = out["projected_vertices"].contiguous(), out["valid"]
    run = lambda: uv_textures(table, frames, v, fi, valid)        # noqa: E731
    for _ in range(5):
        run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            run()
        torch.cuda.synchronize()
    S, V, T = table.img_size, table.n_vertices, int(table.texel.shape[0])
    need = {"uv_normals_kernel": R * V * 12 + R * V * 8,                         # vertices in, normal z out
            "uv_texels_kernel": R * S * S * 3 + S * S * 36 + R * V * 20 + R * T * 3}   # texture, table, v + nz, pixels
    res = {"what": "uv_textures kernels (torch.profiler)", "frames": [F, H, W], "boxes": R, "calls": calls}
    for e in prof.key_averages():
        for name, nbytes in need.items():
            if name in e.key:
                ms = e.device_time_total / 1e3 / e.count if e.count else float("nan")
                res[name] = {"ms": round(ms, 4), "count": e.count, "hbm_bound_ms": round(nbytes / HBM_BYTES_PER_S * 1e3, 4),
                             "share_of_hbm_bound": round(nbytes / HBM_BYTES_PER_S * 1e3 / ms, 3)}
    return res


def bench_reference(path, heads=3):
    """The reference's per-texel Python loop on the host, seconds per head."""
    sys.path.insert(0, ROOT)
    from dad_3dheads_b200.flame import load_flame_static
    from dad_3dheads_b200.uv_texture import read_table
    from tests import uv_model as M
    faces = load_flame_static()["faces"]
    table = read_table(path)
    v = M.flame_heads(heads, 0)
    frame = np.random.default_rng(0).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    M.reference_texture_map(frame, v[0], faces, table)
    t = time.perf_counter()
    for r in range(heads):
        M.reference_texture_map(frame, v[r], faces, table)
    return {"what": "reference _compute_texture_map (host, psbody restated)", "heads": heads,
            "s_per_head": round((time.perf_counter() - t) / heads, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=64)
    ap.add_argument("--table", default=None, help="texture_data.npy (default: the reference's, via oracle/ref_harness)")
    ap.add_argument("--out", default=os.path.join(ROOT, "uv_texture_bench_out"))
    ap.add_argument("--part", choices=("step", "kernels", "reference", "all"), default="all")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("uv_texture_bench needs a GPU")
    from tests import uv_model as M
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import DEFAULT_CONFIG, FaceMeshPredictor
    from dad_3dheads_b200.uv_texture import UvTextureTable
    path = args.table or M.reference_table_path()
    if path is None:
        raise SystemExit("no texture_data.npy: pass --table")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    results = {"card": card()}
    print("card:", results["card"])
    pred = FaceMeshPredictor(dict(DEFAULT_CONFIG), cuda_id=0, state_dict=synthetic_state_dict(0), precision="fp16x2")
    table = UvTextureTable.load(path, dev)
    if args.part in ("step", "all"):
        results["step"] = bench_step(pred, dev, args.boxes, table)
        print(json.dumps(results["step"]))
    if args.part in ("kernels", "all"):
        results["kernels"] = bench_kernels(pred, dev, args.boxes, table)
        print(json.dumps(results["kernels"]))
    if args.part in ("reference", "all"):
        results["reference"] = bench_reference(path)
        print(json.dumps(results["reference"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, f"uv_texture_bench_{args.part}.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
