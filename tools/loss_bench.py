#!/usr/bin/env python
"""Times the train_loss.yaml objective (heat-map IoU + 50 x vertices l2 + 0.05 x reprojection smooth-L1 + 100 x landmarks
smooth-L1) forward plus backward on one GPU, at B = 64 (train_stage/flame_landmarks.yaml's batch size) and B = 256:

  new     the package's loss classes (csrc/loss.cu) through the reference's sum
  torch   the same formulas written as torch ops on the GPU over HeadMesh.decode_with_grad
  heatmap dad3d_iou_forward and dad3d_iou_backward alone, with the bytes they must move over their time, against the
          H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth

Each number is the mean over a window of at least one second after a warm-up, from CUDA events.  The card's name, power limit
and maximum SM clock are read in the same run.  Writes <out>/loss_bench.json and prints it.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
FILES = {"head": "head.npy", "face_w_ears": "face_w_ears.npy", "face": "face.npy"}
V_WEIGHTS = {"head": .5, "face_w_ears": .75, "face": 1.}
P_WEIGHTS = {"face": .5, "face_w_ears": .5}
C, HM = 68, 64                                 # heat-map channels and side (stride 4 of 256 x 256 inputs)


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
    from oracle.flame_oracle import sample_params
    g = torch.Generator().manual_seed(seed)
    p = sample_params(B, seed=seed)
    x = torch.randn(B, C, HM, HM, generator=g) * 3
    th = torch.rand(B, C, HM, HM, generator=g)
    tv = torch.randn(B, 5023, 3, generator=g) * 0.1
    tp = torch.rand(B, 5023, 2, generator=g) * 256
    lm, lt = torch.rand(B, C, 2, generator=g) * 64, torch.rand(B, C, 2, generator=g) * 64
    pres = (torch.rand(B, C, generator=g) < 0.8).float()
    leaves = [a.to(dev).requires_grad_(True) for a in (x, p, lm)]
    return leaves + [a.to(dev) for a in (th, tv, tp, lt, pres)]


def normalize_to_cube(v):
    v = v - v.min(1, True)[0]
    v = v - 0.5 * v.max(1, True)[0]
    return v / v.max(-1, True)[0].max(-2, True)[0]


class Objective:
    def __init__(self, folder):
        from dad_3dheads_b200.flame import FLAME_CONSTS
        from dad_3dheads_b200.losses import IoULoss, LandmarksLossWVisibility, ReprojectionLoss, Vertices3DLoss
        wi = lambda w: {"flame_indices": {"folder": folder, "files": dict(FILES)}, "weights": dict(w)}
        self.iou = IoULoss()
        self.v = Vertices3DLoss("l2", 64, FLAME_CONSTS, wi(V_WEIGHTS))
        self.p = ReprojectionLoss("smooth_l1", 64, FLAME_CONSTS, 256, wi(P_WEIGHTS))
        self.lmk = LandmarksLossWVisibility("smooth_l1")
        self.v_idx = [torch.as_tensor(i).cuda() for i in self.v.indices]
        self.p_idx = [torch.as_tensor(i).cuda() for i in self.p.indices]

    def new(self, params, x, th, tv, tp, lm, lt, pres):
        return (self.iou(x, th) + 50. * self.v(params, tv) + 0.05 * self.p(params, [tp])
                + 100. * self.lmk([lm, pres], [lt, pres]))

    def torch_ops(self, params, x, th, tv, tp, lm, lt, pres):
        s = torch.sigmoid(x)
        op = lambda a: a.flatten(2).sum(2)
        lh = 1 - ((op(th * s) + 1e-6) / (op(th ** 2) + op(s ** 2) - op(th * s) + 1e-6)).mean()
        v3, _ = self.v.head_mesh.decode_with_grad(params, zero_rotation=True)
        lv = torch.stack([F.mse_loss(normalize_to_cube(v3[:, i]), normalize_to_cube(tv[:, i])) * w
                          for w, i in zip(self.v.weights, self.v_idx)]).sum()
        _, pj = self.p.head_mesh.decode_with_grad(params, to_2d=True)
        self.p.head_mesh.flame_params(params).translation[..., 2] = 0.0
        lp = torch.stack([F.smooth_l1_loss(pj[:, i], tp[:, i]) * w for w, i in zip(self.p.weights, self.p_idx)]).sum()
        ll = F.smooth_l1_loss(lm * pres[..., None], lt * pres[..., None])
        return lh + 50. * lv + 0.05 * lp + 100. * ll


def step(fn, data):
    """fn's total and its gradients w.r.t. the three network outputs; data[:3] are the leaves (logits, params, landmarks)."""
    x, p, lm, th, tv, tp, lt, pres = data
    total = fn(p * 1.0, x, th, tv, tp, lm, lt, pres)
    return (total,) + torch.autograd.grad(total, [x, p, lm])


def heatmap_kernels(B, dev):
    from dad_3dheads_b200 import _lib
    lib = _lib.load()
    x, t = torch.randn(B, C, HM, HM, device=dev), torch.rand(B, C, HM, HM, device=dev)
    P, hw = B * C, HM * HM
    stats = torch.empty(P, 4, device=dev)
    loss, g = torch.empty((), device=dev), torch.ones((), device=dev)
    gx = torch.empty_like(x)
    stream = torch.cuda.current_stream(dev).cuda_stream
    fwd = lambda: lib.dad3d_iou_forward(x.data_ptr(), t.data_ptr(), P, hw, stats.data_ptr(), loss.data_ptr(), stream)
    bwd = lambda: lib.dad3d_iou_backward(x.data_ptr(), t.data_ptr(), P, hw, stats.data_ptr(), g.data_ptr(), gx.data_ptr(),
                                         stream)
    assert fwd() == 0 and bwd() == 0
    plane_bytes = 4 * x.numel()
    out = {}
    for name, fn, nbytes in (("forward", fwd, 2 * plane_bytes), ("backward", bwd, 3 * plane_bytes)):
        ms = timed(fn)
        out[name] = {"ms": round(ms, 4), "bytes": nbytes, "TB_per_s": round(nbytes / ms / 1e9, 3),
                     "share_of_3.35TB_per_s": round(nbytes / ms / 1e9 / 3.35, 3)}
    total = 5 * plane_bytes
    out["bound_us_at_3.35TB_per_s"] = round(total / HBM_BYTES_PER_S * 1e6, 1)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--flame-indices", default=os.path.join(ROOT, "oracle", "_ref", "model_training", "model", "static",
                                                              "flame_indices"),
                    help="folder with head.npy, face_w_ears.npy and face.npy (the reference's flame_indices)")
    ap.add_argument("--out", default="loss_bench_out")
    ap.add_argument("--batches", default="64,256")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_bench needs a GPU")
    for f in FILES.values():
        if not os.path.isfile(os.path.join(args.flame_indices, f)):
            raise SystemExit(f"{args.flame_indices}/{f} is missing (pass --flame-indices)")
    dev = torch.device("cuda", 0)
    result = {"card": card(), "runs": []}
    obj = Objective(args.flame_indices)
    for B in [int(b) for b in args.batches.split(",")]:
        data = inputs(B, dev)
        a, b = step(obj.new, data), step(obj.torch_ops, data)
        agree = {"total_rel": abs((a[0] - b[0]).item()) / abs(b[0].item())}
        for name, ga, gb in zip(("heatmap", "params", "landmarks"), a[1:], b[1:]):
            agree[f"grad_{name}_relL2"] = ((ga - gb).norm() / gb.norm()).item()
        run = {"B": B, "agreement_new_vs_torch": {k: float(f"{v:.3e}") for k, v in agree.items()}}
        times = {"new": [], "torch": []}
        for _ in range(3):                                   # alternate, three windows each
            times["new"].append(round(timed(lambda: step(obj.new, data)), 4))
            times["torch"].append(round(timed(lambda: step(obj.torch_ops, data)), 4))
        med = {k: sorted(v)[1] for k, v in times.items()}
        run["fwd_bwd_ms"] = times
        run["median_ms"] = med
        run["speedup"] = round(med["torch"] / med["new"], 3)
        run["heatmap_kernels"] = heatmap_kernels(B, dev)
        result["runs"].append(run)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "loss_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
