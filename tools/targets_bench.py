#!/usr/bin/env python
"""Times FlameBatchBuilder (dad_3dheads_b200.training_data) on one GPU at B = 64 (train_stage/flame_landmarks.yaml's batch
size) and B = 256, with crops of 150 to 600 px a side, 68 landmarks, stride 4, radius 5 (config/dataset/dad_3d_heads.yaml):

  build    the four kernels of one build (letter-box setup and pre-processing, targets, heat-maps) on inputs already on the
           device, with the bytes they must move over their time against the H100 SXM data sheet's 3.35 TB/s of HBM3
           bandwidth (a lower bound on the time, not a claim that the kernels reach it)
  copy     the non-blocking host-to-device copy of the packed batch from pinned memory
  total    one call on the pinned packed batch: copy plus build
  reference_ms_per_item  on this host's CPU, the reference's FlameDataset._transform + _form_anno_dict per item
           (oracle/_ref, with the keypoint path of tests/albumentations_keypoints.py), file reading excluded

Each GPU number is the mean over a window of at least one second after a warm-up, from CUDA events.  The card's name, power
limit and maximum SM clock are read in the same run.  Writes <out>/targets_bench.json and prints it.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


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


def records(B, seed):
    from tests.test_targets_gpu import synthetic_records
    rng = np.random.default_rng(seed)
    sides = [(int(rng.integers(150, 601)), int(rng.integers(150, 601))) for _ in range(B)]
    return synthetic_records(B, seed, sides)


def moved_bytes(packed, S, C, Sh):
    """Bytes a build must read and write: the crop pixels and the per-head inputs; the images, keypoints, landmarks,
    presence and heat-maps."""
    ints = packed["ints"].numpy()
    B = int(packed["crops"].shape[0])
    w, h = ints[9 * B:10 * B].astype(np.int64), ints[10 * B:11 * B].astype(np.int64)
    V = int(packed["vertices"].shape[1])
    read = int((w * h * 3).sum()) + B * V * 3 * 4 + B * 32 * 4
    written = B * 3 * S * S * 4 + B * V * 2 * 4 + B * C * (2 * 2 * 4 + 1) + B * C * Sh * Sh
    return read, written


def reference_per_item(n=16):
    from oracle import ref_harness as R
    from tests.test_targets_model_cpu import dataset_config, make_dataset
    R.activate()
    from model_training.data.flame_dataset import FlameDataset as RefDataset
    root = tempfile.mkdtemp(prefix="targets_bench_")
    config = dataset_config(root, "68")
    data = make_dataset(root, n, seed=1)
    from tests.albumentations_keypoints import keypoint_albumentations
    with keypoint_albumentations():
        ds = RefDataset(data, config)
        np.random.seed(0)
        parsed = [ds._parse_anno(a) for a in data]              # file reading, outside the timed loop
        t0 = time.perf_counter()
        reps = 0
        while time.perf_counter() - t0 < 2.0:
            for item in parsed:
                ds._form_anno_dict(ds._transform(dict(item)))
            reps += 1
    return 1e3 * (time.perf_counter() - t0) / (reps * len(parsed))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="targets_bench_out")
    ap.add_argument("--batches", default="64,256")
    args = ap.parse_args()
    from dad_3dheads_b200.training_data import FlameBatchBuilder, collate_records
    from tests.test_targets_model_cpu import dataset_config
    dev = torch.device("cuda", 0)
    config = dataset_config(tempfile.mkdtemp(prefix="targets_bench_"), "68")
    builder = FlameBatchBuilder(config, dev)
    S, C, Sh = 256, 68, 64
    result = {"card": card(), "config": "68 landmarks, stride 4, radius 5, imagenet, crops 150-600 px", "batches": {}}
    for B in (int(b) for b in args.batches.split(",")):
        packed = collate_records(records(B, B))
        pinned = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in packed.items()}
        on_dev = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in packed.items()}
        copy_bytes = sum(v.numel() * v.element_size() for v in pinned.values() if isinstance(v, torch.Tensor))
        build_ms = timed(lambda: builder(on_dev))
        copy_ms = timed(lambda: [v.to(dev, non_blocking=True) for v in pinned.values() if isinstance(v, torch.Tensor)])
        total_ms = timed(lambda: builder(pinned))
        rd, wr = moved_bytes(packed, S, C, Sh)
        result["batches"][str(B)] = {
            "build_ms": round(build_ms, 4), "build_bytes_read": rd, "build_bytes_written": wr,
            "build_TBps": round((rd + wr) / (build_ms * 1e-3) / 1e12, 3),
            "build_bound_ms_at_3.35TBps": round((rd + wr) / HBM_BYTES_PER_S * 1e3, 4),
            "copy_ms": round(copy_ms, 4), "copy_bytes": copy_bytes,
            "copy_GBps": round(copy_bytes / (copy_ms * 1e-3) / 1e9, 2), "total_ms": round(total_ms, 4),
            "crop_buffer": list(packed["crops"].shape)}
    result["reference_ms_per_item"] = round(reference_per_item(), 3)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "targets_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
