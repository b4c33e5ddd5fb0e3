#!/usr/bin/env python
"""Times the training step's metric block on one GPU at B = 64 (train_stage/flame_landmarks.yaml's batch size) and B = 256,
68 landmarks and 64 x 64 heat-maps:

  new      FlameStepMetrics.step (csrc/metrics.cu, two hi/lo decodes included)
  torch    the same block written as torch ops on the GPU over the package's same two decodes
  kernels  the three metric kernels alone (IoU statistics, per-head errors, reduction), with the bytes they must read over
           their time, against the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth

Each number is the mean over a window of at least one second after a warm-up, from CUDA events; the variants alternate over
three rounds and the median is reported.  The card's name, power limit and maximum SM clock are read in the same run.
Writes <out>/metrics_bench.json and prints it.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
C, HM, V = 68, 64, 5023
THR = (0.05, 0.1)


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


def inputs(B, dev, seed=0):
    from dad_3dheads_b200 import metrics as PM
    from oracle.flame_oracle import sample_params
    g = torch.Generator().manual_seed(seed)
    p = sample_params(B, seed=seed)
    lm_t = torch.rand(B, C, 2, generator=g)
    box = torch.randint(60, 600, (4, B), generator=g, dtype=torch.int32)
    batch = {PM.TARGET_LANDMARKS_HEATMAP: (torch.rand(B, C, HM, HM, generator=g) * 255).to(torch.uint8),
             PM.TARGET_2D_LANDMARKS: lm_t, PM.TARGET_2D_LANDMARKS_PRESENCE: torch.rand(B, C, generator=g) < 0.9,
             PM.TARGET_2D_FULL_LANDMARKS: torch.rand(B, V, 2, generator=g) * 256,
             PM.TARGET_3D_MODEL_VERTICES: 0.1 * torch.randn(B, V, 3, generator=g)}
    batch = {k: v.to(dev) for k, v in batch.items()}
    batch[PM.INPUT_BBOX_KEY] = list(box.to(dev).unbind(0))
    outputs = {PM.OUTPUT_3DMM_PARAMS: p.to(dev), PM.OUTPUT_2D_LANDMARKS: (lm_t + 0.02 * torch.randn(B, C, 2, generator=g)).to(dev),
               PM.OUTPUT_LANDMARKS_HEATMAP: (3 * torch.randn(B, C, HM, HM, generator=g) - 2).to(dev)}
    return outputs, batch


def torch_block(m, outputs, batch):
    """The step's metric block as torch ops (train/flame_lightning_model.py:304-357, metrics/iou.py, metrics/keypoints.py)."""
    from dad_3dheads_b200 import metrics as PM
    params = outputs[PM.OUTPUT_3DMM_PARAMS]
    B = params.shape[0]
    dec = m.head_mesh.flame.decoder(params.device)
    v3, _ = dec.decode(params, want_vertices=True, want_projected=False, zero_rot=True, hilo=True)
    _, pj = dec.decode(params, want_vertices=False, want_projected=True, to_2d=True, image_size=256.0, hilo=True)
    o = outputs[PM.OUTPUT_LANDMARKS_HEATMAP].sigmoid()
    t = batch[PM.TARGET_LANDMARKS_HEATMAP].div(255.0)
    it = (t * o).sum((2, 3))
    out = [((it + 1e-6) / ((t ** 2).sum((2, 3)) + (o ** 2).sum((2, 3)) - it + 1e-6)).mean()]
    bbox = torch.stack(batch[PM.INPUT_BBOX_KEY]).T
    pres = batch[PM.TARGET_2D_LANDMARKS_PRESENCE][..., None]
    face = m._face(params.device).long()

    def cube(v):
        v = v - v.min(1, True)[0]
        v = v - 0.5 * v.max(1, True)[0]
        return v / v.max(-1, True)[0].max(-2, True)[0]

    groups = [(outputs[PM.OUTPUT_2D_LANDMARKS] * 256 * pres, batch[PM.TARGET_2D_LANDMARKS] * pres * 256, bbox),
              (pj[:, face], batch[PM.TARGET_2D_FULL_LANDMARKS][:, face], bbox),
              (cube(v3[:, face]), cube(batch[PM.TARGET_3D_MODEL_VERTICES][:, face]), None)]
    for p, q, bb in groups:
        err = (p - q).norm(2, -1).mean(-1)
        norm = torch.sqrt(bb[:, 2] * bb[:, 3]) if bb is not None else 2.0
        out.append(100 * (err / norm).mean())
        out += [(err < thr * norm).sum() / B for thr in THR]
    return torch.stack(out)


def kernel_bytes(B):
    """Bytes the three metric kernels must read: logits (fp32) and uint8 targets of the heat-maps, then per head both
    operands of 68 + 2 x 2094 keypoints, presence and box, then the records."""
    heat = B * C * HM * HM * (4 + 1)
    kp = B * (2 * C * 2 * 4 + C + 2 * 2094 * 2 * 4 + 2 * 2094 * 3 * 4 + 2 * 2094 * 4 + 8)
    return heat + kp + B * C * 16 + B * 3 * 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="metrics_bench_out")
    ap.add_argument("--min-s", type=float, default=1.0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "metrics_bench needs a GPU"
    from dad_3dheads_b200 import metrics as PM
    dev = torch.device("cuda", 0)
    m = PM.FlameStepMetrics()
    res = {"card": card(), "B": {}}
    for B in (64, 256):
        outputs, batch = inputs(B, dev, seed=B)
        got = m.step(outputs, batch)
        new = torch.stack([got[f"valid/metrics/{n}"] for n in m.names])
        ref = torch_block(m, outputs, batch)
        cont = [i for i, n in enumerate(m.names) if "fr_" not in n]
        agree = {"max_rel_continuous": max(abs((new[i] - ref[i]) / ref[i]).item() for i in cont),
                 "counts_equal": all(new[i].item() == ref[i].item() for i in range(len(m.names)) if i not in cont)}
        # the three metric kernels alone, on prepared decodes
        dec = m.head_mesh.flame.decoder(dev)
        params = outputs[PM.OUTPUT_3DMM_PARAMS]
        v3, _ = dec.decode(params, want_vertices=True, want_projected=False, zero_rot=True, hilo=True)
        _, pj = dec.decode(params, want_vertices=False, want_projected=True, to_2d=True, image_size=256.0, hilo=True)
        hm, hm_t = outputs[PM.OUTPUT_LANDMARKS_HEATMAP], batch[PM.TARGET_LANDMARKS_HEATMAP]
        box = (batch[PM.INPUT_BBOX_KEY][2], batch[PM.INPUT_BBOX_KEY][3])
        face = m._face(dev)
        pres = batch[PM.TARGET_2D_LANDMARKS_PRESENCE].view(torch.uint8)
        groups = [PM._Group(outputs[PM.OUTPUT_2D_LANDMARKS], batch[PM.TARGET_2D_LANDMARKS], presence=pres, box=box,
                            pred_scale=256.0, target_scale=256.0),
                  PM._Group(pj, batch[PM.TARGET_2D_FULL_LANDMARKS], index=face, box=box),
                  PM._Group(v3, batch[PM.TARGET_3D_MODEL_VERTICES], index=face, normalize=True)]

        def kernels():
            stats = PM._iou_stats(hm, hm_t, logits=True)
            rec = PM._keypoint_errors(groups, B, dev)
            PM._reduce(dev, 10, stats=stats, records=rec, nme_scale=100.0, thresholds=THR)

        times = {"new": [], "torch": [], "kernels": []}
        for _ in range(3):
            times["new"].append(timed(lambda: m.step(outputs, batch), a.min_s))
            times["torch"].append(timed(lambda: torch_block(m, outputs, batch), a.min_s))
            times["kernels"].append(timed(kernels, a.min_s))
        med = {k: sorted(v)[1] for k, v in times.items()}
        nbytes = kernel_bytes(B)
        res["B"][str(B)] = {"agreement": agree, "ms": med, "ms_all_rounds": times, "kernel_bytes": nbytes,
                            "kernel_TBps": nbytes / (med["kernels"] * 1e-3) / 1e12,
                            "kernel_bound_ms": nbytes / HBM_BYTES_PER_S * 1e3}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "metrics_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
