"""Exact numpy model of csrc/metrics.cu: the per-plane soft-IoU statistics on probabilities with fp32 or uint8 targets
(iou_forward_kernel<false, T>), the per-head keypoint errors (keypoint_errors_kernel) and the batch reduction
(metrics_reduce_kernel).  Every fp32 operation is one IEEE rounding in the kernels' order, fmaf included (emulated in
fp64 with round-to-odd), and the block reductions follow the kernels' thread, butterfly and warp order, so given the same
inputs the model reproduces every output bit for bit."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

THREADS = 256
WARPS = THREADS // 32
f32, f64 = np.float32, np.float64


def fma32(a, b, c):
    """fmaf: fp32(a * b + c) rounded once.  The product is exact in fp64; the sum is rounded to odd in fp64, which then
    rounds to fp32 correctly (53 >= 2 * 24 + 2)."""
    a, b, c = (np.asarray(x, f32).astype(f64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    with np.errstate(invalid="ignore"):
        inexact = (e != 0) & np.isfinite(s)
        bits = s.view(np.int64).copy()
        even = (bits & 1) == 0
        up = np.sign(e) == np.sign(s)
    adj = inexact & even
    bits = np.where(adj, np.where(up, bits + 1, bits - 1), bits)
    return bits.view(f64).astype(f32)


def butterfly(x):
    """__shfl_xor_sync sums over lanes 16, 8, 4, 2, 1 of x [..., 32]: every lane ends with the same value."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = x + x[..., lanes ^ o]
    return x[..., 0]


def block_sum(partials):
    """block_sum / block_dsum of per-thread partials [..., 256] (fp32 or fp64): warps' butterflies, then the warps in order
    from zero."""
    w = butterfly(partials.reshape(partials.shape[:-1] + (WARPS, 32)))
    s = np.zeros(partials.shape[:-1], partials.dtype)
    for i in range(WARPS):
        s = s + w[..., i]
    return s


def strided(values, fill):
    """values [..., n] -> [..., rounds, 256]: thread t's elements t, t + 256, ... in order (``fill`` past the end)."""
    n = values.shape[-1]
    rounds = max(1, -(-n // THREADS))
    out = np.full(values.shape[:-1] + (rounds * THREADS,), fill, values.dtype)
    out[..., :n] = values
    return out.reshape(values.shape[:-1] + (rounds, THREADS)), n


# ---------------------------------------------------------------------------------------------------------- soft IoU
def target_value(t):
    t = np.asarray(t)
    return t.astype(f32) / f32(255) if t.dtype == np.uint8 else t.astype(f32)


def iou_stats(x, t):
    """iou_forward_kernel<false, T>: x [P, hw] probabilities, t [P, hw] fp32 or uint8 -> stats [P, 4] fp32."""
    x = np.asarray(x, f32)
    tv = target_value(t)
    P, hw = x.shape
    a = np.zeros((3, P, THREADS), f32)
    if hw % 4 == 0:        # the float4 path: thread i takes elements 4i .. 4i + 3, then i + 256
        xs, _ = strided(x.reshape(P, hw // 4, 4).transpose(0, 2, 1), 0)   # [P, 4, rounds, 256]
        ts, _ = strided(tv.reshape(P, hw // 4, 4).transpose(0, 2, 1), 0)
        valid, _ = strided(np.ones((1, 4, hw // 4), bool), False)
        for r in range(xs.shape[2]):
            for e in range(4):
                s, tt, m = xs[:, e, r], ts[:, e, r], valid[:, e, r]
                a[0] = np.where(m, fma32(s, tt, a[0]), a[0])
                a[1] = np.where(m, fma32(tt, tt, a[1]), a[1])
                a[2] = np.where(m, fma32(s, s, a[2]), a[2])
    else:
        xs, _ = strided(x, 0)
        ts, _ = strided(tv, 0)
        valid, _ = strided(np.ones((1, hw), bool), False)
        for r in range(xs.shape[1]):
            s, tt, m = xs[:, r], ts[:, r], valid[:, r]
            a[0] = np.where(m, fma32(s, tt, a[0]), a[0])
            a[1] = np.where(m, fma32(tt, tt, a[1]), a[1])
            a[2] = np.where(m, fma32(s, s, a[2]), a[2])
    I, T, S = (block_sum(a[k]) for k in range(3))
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = (I + f32(1e-6)) / iou_den(I, T, S, f32(1e-6))
    return np.stack([I, T, S, iou], 1).astype(f32)


def iou_den(I, T, S, eps):
    return ((T + S) - I) + f32(eps)


# ---------------------------------------------------------------------------------------------------- keypoint errors
def group(pred, target, index=None, presence=None, box=None, pred_scale=1.0, target_scale=1.0, normalize=False):
    """A keypoint group as the kernel reads it: pred / target [B, rows, K] fp32, index [n] or None, presence [B, n] or
    None, box (w [B], h [B]) int32 or None."""
    return dict(pred=np.asarray(pred, f32), target=np.asarray(target, f32), index=index, presence=presence, box=box,
                pred_scale=f32(pred_scale), target_scale=f32(target_scale), normalize=normalize)


def _operands(g):
    p, t = g["pred"], g["target"]
    if g["index"] is not None:
        p, t = p[:, np.asarray(g["index"])], t[:, np.asarray(g["index"])]
    m = (np.asarray(g["presence"]).astype(f32) if g["presence"] is not None else np.ones(p.shape[:2], f32))[..., None]
    with np.errstate(invalid="ignore", over="ignore"):
        return (p * g["pred_scale"]) * m, (t * m) * g["target_scale"]


def _ext(v, fn, init):
    """min / max over axis 1 ignoring NaN (a NaN never wins); ``init`` when every value is NaN."""
    with np.errstate(invalid="ignore"):
        allnan = np.isnan(v).all(1)
        r = fn.reduce(v, axis=1)
    return np.where(allnan, f32(init), r).astype(f32)


def _normalize(v):
    """normalize_to_cube over axis 1 of v [B, n, K], with the kernel's reductions."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        mn = _ext(v, np.fmin, np.inf)[:, None]
        half = f32(0.5) * _ext(v - mn, np.fmax, -np.inf)[:, None]
        c = (v - mn) - half
        M = _ext(c.reshape(c.shape[0], -1), np.fmax, -np.inf)[:, None, None]
        return c / M


def _dist(d):
    s = d[..., 0] * d[..., 0]
    s = fma32(d[..., 1], d[..., 1], s)
    if d.shape[-1] == 3:
        s = fma32(d[..., 2], d[..., 2], s)
    with np.errstate(invalid="ignore"):
        return np.sqrt(s)


def keypoint_errors(groups: Sequence[Dict]):
    """keypoint_errors_kernel: records [B, G, 2] = (err, norm)."""
    B = groups[0]["pred"].shape[0]
    rec = np.zeros((B, len(groups), 2), f32)
    for gi, g in enumerate(groups):
        p, t = _operands(g)
        if g["normalize"]:
            p, t = _normalize(p), _normalize(t)
        with np.errstate(invalid="ignore", over="ignore"):
            d = _dist(p - t)                                            # [B, n]
        ds, n = strided(d, 0)
        part = np.zeros((B, THREADS), f32)
        for r in range(ds.shape[1]):
            with np.errstate(invalid="ignore", over="ignore"):
                part = part + ds[:, r]
        with np.errstate(invalid="ignore", over="ignore"):
            rec[:, gi, 0] = block_sum(part) / f32(n)
        if g["box"] is not None:
            w, h = (np.asarray(c).astype(np.int64) for c in g["box"])
            prod = ((w * h + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(np.int32)         # the int32 product wraps
            with np.errstate(invalid="ignore"):
                rec[:, gi, 1] = np.sqrt(prod.astype(f32))
        else:
            rec[:, gi, 1] = f32(2.0)
    return rec


# ------------------------------------------------------------------------------------------------------- reduction
def dsum(x):
    """block_dsum over x [n] fp64 summed per thread (t, t + 256, ...) from zero."""
    xs, _ = strided(np.asarray(x, f64)[None], 0.0)
    part = np.zeros((1, THREADS), f64)
    for r in range(xs.shape[1]):
        part = part + xs[:, r]
    return block_sum(part)[0]


def reduce(stats=None, eps=1e-6, records=None, nme_scale=1.0, below=True, thresholds=(), epoch=None, weight=0.0):
    """metrics_reduce_kernel: (values, per_head [B, G] or None, epoch after the update or None)."""
    values: List[np.float32] = []
    per_head = None
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if stats is not None:
            st = np.asarray(stats, f32)
            iou = (st[:, 0] + f32(eps)) / iou_den(st[:, 0], st[:, 1], st[:, 2], f32(eps))
            values.append(f32(dsum(iou.astype(f64)) / st.shape[0]))
        if records is not None:
            rec = np.asarray(records, f32)
            B, G = rec.shape[:2]
            per_head = rec[..., 0] / rec[..., 1]
            for g in range(G):
                err, norm = rec[:, g, 0], rec[:, g, 1]
                values.append(f32(f32(dsum(per_head[:, g].astype(f64)) / B) * f32(nme_scale)))
                for thr in thresholds:
                    bound = f32(thr) * norm
                    cnt = int(((err < bound) if below else (err > bound)).sum())
                    values.append(f32(cnt) / f32(B))
    values = np.array(values, f32)
    if epoch is not None:
        epoch = np.array(epoch, f64)
        n = len(values)
        epoch[:n] += values.astype(f64) * weight
        epoch[n] += weight
    return values, per_head, epoch


def epoch_values(epoch):
    epoch = np.asarray(epoch, f64)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (epoch[:-1] / epoch[-1]).astype(f32)
