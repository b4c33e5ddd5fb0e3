#!/usr/bin/env python
"""Per-layer roofline table of the encoder's tile-engine launches, timed live with CUDA events (no profiler attached).

usage: tools/layer_table.py [--batch 64] [--precision fp32] [--reps 7] [--out profiles/r01_layers.md]
Every row: GEMM shape, device time (median over reps), useful TFLOP/s, executed TFLOP/s (x products per MAC), algorithmic
GB/s, and the fraction of the larger of its two roofline times (HBM and 16-bit dense tensor peaks as bench.py uses them:
MEASURED_PEAKS.json when present, else the H100 SXM data sheet).  The header records the card, its power limit and SM clock."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dad_3dheads_b200.encoder import Dad3dEncoder  # noqa: E402
from dad_3dheads_b200.encoder_weights import synthetic_state_dict  # noqa: E402
from bench import _peaks  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--precision", default="fp32")
ap.add_argument("--out", default="")
a = ap.parse_args()

pk = _peaks()
hbm, tens = float(pk["hbm_gbs"]), float(pk["bf16_tflops_sustained"])   # GB/s, TFLOP/s


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unknown (nvidia-smi unavailable)"


dev = torch.device("cuda", 0)
enc = Dad3dEncoder(synthetic_state_dict(0), dev, precision=a.precision, want_heatmap=False)
x = torch.randn(a.batch, 3, 256, 256, device=dev)
for _ in range(3):
    enc.forward_raw(x)
torch.cuda.synchronize()
gpu_before = card()
runs = []
for _ in range(a.reps):
    enc.set_profile(True)
    enc.forward_raw(x)
    torch.cuda.synchronize()
    runs.append(enc.profile_layers())
    enc.profile_read()
enc.set_profile(False)
gpu_after = card()
# ping-pong consumers per layer (tile_gemm.cuh); builds without them do not report the field
pingpong = {s["layer"]: s.get("pingpong", 0) for s in enc.describe_plan()["steps"] if s["kind"] == "conv"}
rows = []
for i, r in enumerate(runs[0]):
    r = dict(r)
    r["ms"] = statistics.median(run[i]["ms"] for run in runs)
    rows.append(r)
tot = sum(r["ms"] for r in rows)
lines = [f"# encoder tile-engine launches, batch {a.batch}, precision {a.precision}: {len(rows)} launches, {tot * 1e3:.0f} us "
         f"(median of {a.reps} forwards, CUDA events around each launch, so launch gaps are excluded)", "",
         f"GPU (name, power limit, SM clock, max SM clock) before / after the timed forwards: {gpu_before} / {gpu_after}", "",
         f"roofline denominators ({pk['source']}): HBM {hbm:.0f} GB/s, 16-bit dense {tens:.0f} TFLOP/s; "
         "`frac` = max(bytes/HBM, executed flops/tensor) / time; `pp` = 1 for ping-pong launches", "",
         "| layer | M | K | N | bn | kblk | tiles | stg | us | useful TF/s | exec TF/s | GB/s | t_hbm us | t_mma us | frac | pp |",
         "|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
for r in rows:
    us = r["ms"] * 1e3
    ex = r["flops"] * r["products"]
    t_h = r["bytes"] / (hbm * 1e9) * 1e6
    t_m = ex / (tens * 1e12) * 1e6
    lines.append(f"| {r['name']} | {r['M']} | {r['K']} | {r['N']} | {r['block_n']} | {r['k_blocks']} | {r['tiles']} | {r['stages']} | {us:.1f} | "
                 f"{r['flops'] / us / 1e6:.0f} | {ex / us / 1e6:.0f} | {r['bytes'] / us / 1e3:.0f} | {t_h:.1f} | {t_m:.1f} | "
                 f"{max(t_h, t_m) / us:.2f} | {pingpong.get(r['name'], 0)} |")
ideal = sum(max(r["bytes"] / (hbm * 1e9), r["flops"] * r["products"] / (tens * 1e12)) for r in rows) * 1e6
lines += ["", f"sum of per-layer roofline times: {ideal:.0f} us = {ideal / (tot * 1e3):.2f} of the measured {tot * 1e3:.0f} us"]
txt = "\n".join(lines) + "\n"
print(txt)
if a.out:
    os.makedirs(os.path.dirname(os.path.join(ROOT, a.out)) or ".", exist_ok=True)
    open(os.path.join(ROOT, a.out), "w").write(txt)
