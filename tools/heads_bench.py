#!/usr/bin/env python
"""Times DAD-3DNet's regression heads (csrc/heads.cu) on one GPU at B = 64 and 256 over frozen-backbone features:

  heads    FlameHeads forward + backward (8 launches), training mode
  torch    the same heads as torch ops (F.linear on cuBLAS, relu, dropout, tanh) forward + backward over the same features
  step     a whole captured fine-tuning step: Dad3dEncoder.features + heads + the reference's LossModule over the package
           losses + backward + Adam(capturable=True), replayed from a CUDA graph
  kernels  every heads_* kernel's time (torch.profiler, a run of its own) with its FLOP and byte bounds against the H100
           SXM data sheet's 67 TFLOP/s fp32 and 3.35 TB/s HBM3
  agree    relL2 of the outputs and the four gradients against the torch variant run with the kernels' own keep mask

Each timing is the mean over a window of at least one second after a warm-up, from CUDA events; the two head variants
alternate over three rounds and the median is reported.  The card's name, power limit and maximum SM clock are read in the
same run.  Writes <out>/heads_bench.json and prints it.
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_FLOPS, HBM_BYTES_PER_S = 67e12, 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, min_s=1.0, warmup=3):
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


def torch_heads(f, w1, b1, w2, b2, keep=None, p=0.3, limit=3.0):
    """The reference's three ClassificationHeads + epilogue as torch ops over packed weights; ``keep`` replaces dropout."""
    h = torch.relu(F.linear(f, w1, b1))
    d = F.dropout(h, p, True) if keep is None else h * keep * (1.0 / (1.0 - p))
    outs, r = [], 0
    for i, n in enumerate((403, 10, 136)):
        outs.append(F.linear(d[:, i * 512:(i + 1) * 512], w2[r:r + n], b2[r:r + n]))
        r += n
    params = torch.cat([outs[0].tanh() * limit, outs[1]], 1)
    return params, torch.relu(outs[2].reshape(-1, 68, 2))


def kernel_bounds(B):
    """(FLOPs, bytes) each heads kernel must do / move, from shapes (fp32 words).  Bytes count the weights and features
    read, the tensors the forward saves (read back by the backward) and every result the step keeps; the split partials
    and the backward's do / dd / dh scratch are left out: the previous launch writes them and they stay in the 50 MB L2
    (at most 13 MB at B = 256), so counting them would not give a lower bound."""
    w = 4
    fc1 = (2 * B * 1536 * 2048, w * (B * 2048 + 1536 * 2048))
    fc2 = (2 * B * 549 * 512, w * (549 * 512))
    bwd = (2 * 2 * B * 549 * 512, w * (B * 1536 + 2 * 549 * 512))
    dw1 = (2 * B * 1536 * 2048, w * (B * 2048 + 1536 * 2048))
    return {"gemm0": fc1, "gemm1": fc2, "gemm2": bwd, "gemm3": dw1,
            "heads_hidden_kernel": (2 * B * 1536, w * (1536 + 2 * B * 1536 + B * 48)),
            "heads_output_kernel": (2 * B * 549, w * (549 + B * (413 + 136 + 403) + B * 18)),
            "heads_dout_kernel": (3 * B * 549, w * (549 + B * 403 + B * 18)),
            "heads_dhidden_kernel": (2 * B * 1536, w * (1536 + B * 1536 + B * 48))}


def kernel_times(heads, f, iters=50):
    from torch.profiler import ProfilerActivity, profile
    params, lms = heads(f)
    g1, g2 = torch.ones_like(params), torch.ones_like(lms)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            params, lms = heads(f)
            torch.autograd.backward([params, lms], [g1, g2])
        torch.cuda.synchronize()
    events = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "heads_" in e.name),
                    key=lambda e: e.time_range.start)
    names = [re.search(r"heads_\w+_kernel", e.name).group(0) for e in events]
    # the four GEMM launches share one kernel: each is named by its neighbour in the fixed launch sequence
    # gemm0 -> hidden -> gemm1 -> output | dout -> gemm2 -> dhidden -> gemm3
    per = {}
    for i, (e, name) in enumerate(zip(events, names)):
        if name == "heads_gemm_kernel":
            prev, nxt = (names[i - 1] if i else None), (names[i + 1] if i + 1 < len(names) else None)
            name = {"heads_hidden_kernel": "gemm1", "heads_dout_kernel": "gemm2",
                    "heads_dhidden_kernel": "gemm3"}.get(prev, "gemm0" if nxt == "heads_hidden_kernel" else None)
            if name is None:
                continue
        per.setdefault(name, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    return {k: v[-iters:] for k, v in per.items()}         # the profiled iterations' launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "heads_bench_out"))
    ap.add_argument("--sizes", default="64,256")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "heads_bench needs a GPU"
    from dad_3dheads_b200.encoder import Dad3dEncoder
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.heads import FlameHeads, FrozenBackboneRegression
    dev = torch.device("cuda", 0)
    sd = synthetic_state_dict(0)
    res = {"card": card(), "sizes": {}}
    for B in (int(s) for s in a.sizes.split(",")):
        g = torch.Generator().manual_seed(B)
        f = torch.rand(B, 2048, generator=g).to(dev)
        heads = FlameHeads.from_state_dict(sd, seed=1).to(dev).train()
        tw = [p.detach().clone().requires_grad_(True) for p in heads.parameters()]
        g1, g2 = torch.ones(B, 413, device=dev), torch.ones(B, 68, 2, device=dev)

        def mine():
            params, lms = heads(f)
            torch.autograd.backward([params, lms], [g1, g2])

        def ref():
            params, lms = torch_heads(f, *tw)
            torch.autograd.backward([params, lms], [g1, g2])

        rounds = [(timed(mine), timed(ref)) for _ in range(3)]
        t_mine = sorted(r[0] for r in rounds)[1]
        t_ref = sorted(r[1] for r in rounds)[1]

        # agreement with the kernels' own mask
        for p in list(heads.parameters()) + tw:
            p.grad = None
        params, lms = heads(f)
        from dad_3dheads_b200 import _lib
        c = heads.counter.clone() - 1
        outs = [torch.empty(B, n, device=dev) for n in (413, 136, 1536, 1536, 48, 403, 18)]
        ws = torch.empty(int(_lib.load().dad3d_heads_workspace_bytes(B)), dtype=torch.uint8, device=dev)
        _lib.check(_lib.load().dad3d_heads_forward(f.data_ptr(), B, *(p.data_ptr() for p in heads.parameters()), 3.0, 1,
                                                   0.3, heads.seed, c.data_ptr(), *(o.data_ptr() for o in outs),
                                                   ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream),
                   "forward")
        keep = (outs[4].view(torch.int32).unsqueeze(-1) >> torch.arange(32, device=dev, dtype=torch.int32)) & 1
        keep = keep.reshape(B, 1536).float()
        torch.autograd.backward([params, lms], [g1, g2])
        rp, rl = torch_heads(f, *tw, keep=keep)
        torch.autograd.backward([rp, rl], [g1, g2])
        rel = lambda x, y: ((x - y).norm() / y.norm()).item()      # noqa: E731
        agree = {"params": rel(params, rp), "landmarks": rel(lms, rl)}
        for n, p, q in zip(("dw1", "db1", "dw2", "db2"), heads.parameters(), tw):
            agree[n] = rel(p.grad, q.grad)

        ktimes = kernel_times(heads, f)
        bounds = kernel_bounds(B)
        kern = {}
        for name, us in ktimes.items():
            fl, by = bounds[name]
            t = sum(us) / len(us) * 1e-6
            lb = max(fl / FP32_FLOPS, by / HBM_BYTES_PER_S)
            kern[name] = {"us": t * 1e6, "launches": len(us), "gflop": fl / 1e9, "mb": by / 1e6, "of_bound": lb / t,
                          "bound": "flop" if fl / FP32_FLOPS > by / HBM_BYTES_PER_S else "bytes"}

        step_ms = captured_step(B, sd, dev, FrozenBackboneRegression, Dad3dEncoder, FlameHeads)
        res["sizes"][str(B)] = {"heads_ms": t_mine, "torch_ms": t_ref, "speedup": t_ref / t_mine, "step_ms": step_ms,
                                "agree_relL2": agree, "kernels": kern}
    os.makedirs(a.out, exist_ok=True)
    line = json.dumps(res)
    with open(os.path.join(a.out, "heads_bench.json"), "w") as fh:
        fh.write(line + "\n")
    print(line)


def captured_step(B, sd, dev, FBR, Enc, Heads):
    """ms per replay of the whole fine-tuning step on a builder batch (fp16x2 backbone, the bench's default mode)."""
    import tempfile
    from dad_3dheads_b200.training_data import FlameBatchBuilder, collate_records
    from tests.test_losses_gpu import _mine
    from tests.test_metrics_gpu import _config, _mixin_form
    from tests.test_targets_gpu import synthetic_records

    with tempfile.TemporaryDirectory() as tmp:
        batch = FlameBatchBuilder(_config(tmp), dev)(collate_records(synthetic_records(B, 41)))
    images, targets = batch["INPUT_IMAGE_KEY"], _mixin_form(batch)
    model = FBR(Enc(sd, dev, precision="fp16x2"), Heads.from_state_dict(sd, seed=5).to(dev).train())
    _, module = _mine()
    opt = torch.optim.Adam(model.parameters(), capturable=True)

    def step():
        total, _ = module(model(images), targets, epoch=0)
        opt.zero_grad(set_to_none=False)
        total.backward()
        opt.step()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return timed(g.replay)


if __name__ == "__main__":
    main()
