"""Exact numpy model of csrc/loss.cu: the heat-map IoU statistics on logits (iou_forward_kernel<true, float>, float4 and
scalar paths) and their backward, the landmark forward (fp64 per-head sum of fp32 criterion values) and backward, the
vertex-subset forward for K in {2, 3} with and without normalize_to_cube (the whole per-(head, set) record) and its
backward, and finalize_kernel's fp64 sum.  Every fp32 / fp64 operation is one IEEE rounding in the kernels' order, with
the fused sites fused as the kernel writes them, and the block sums follow the kernels' thread, butterfly and warp order,
so given the same inputs the model reproduces every output bit for bit.

The extreme-value reductions (``Ext`` in reductions.cuh) keep the first index on ties and never select a NaN: a candidate
(v, i) beats (v', i') iff v < v' (or v > v' for a maximum) or v == v' and i < i'.  Over the non-NaN candidates, with +0 and
-0 equal as values, that is a strict total order (indices are distinct), so whatever tree the threads reduce in, the
winner is the order's least element: the first position whose value equals the extreme.  The model takes that position
and its own value, so the winning element's sign of zero is kept.

expf is not modelled: the kernel's expf ends in MUFU.EX2, whose rounding is not specified.  The sigmoid is taken only at
logits where q = expf(-|x|) is exact: q = 1 at x = +-0 and q = 0 at |x| >= 110 (exp(-110) is below half the least
subnormal).  There s is 1/2, 1 or 0 and s (1 - s) is 1/4 or 0; any other finite logit raises.
"""
from __future__ import annotations

from fractions import Fraction
from typing import Sequence

import numpy as np

from tests.metrics_model import THREADS, block_sum, butterfly, fma32, strided  # noqa: F401  (butterfly: block_sum's)

f32, f64 = np.float32, np.float64
EPS = f32(1e-6)
INT_MAX = 2 ** 31 - 1
L1, L2, SMOOTH_L1 = 0, 1, 2
CRITERIA = {"l1": L1, "l2": L2, "smooth_l1": SMOOTH_L1}
RECORD_FLOATS = 32
# word offsets of a normalised record (VsubRec); a record without normalisation writes only LOSS
LOSS, MN, HALF, M_, TMN, THALF, TM, AMIN, AMAX, NSTAR, CSTAR, SCO, SG = 0, 1, 4, 7, 8, 11, 14, 15, 18, 21, 22, 23, 24
RECORD_WRITTEN = 27                       # words 0 .. 26; 27 .. 31 are never written
EXACT_LOGIT = 110.0


def _err():
    return np.errstate(invalid="ignore", divide="ignore", over="ignore", under="ignore")


# ---------------------------------------------------------------------------------------------------------- criteria
def crit_value(crit, d):
    d = np.asarray(d, f32)
    with _err():
        a = np.abs(d)
        if crit == L1:
            return a
        if crit == L2:
            return d * d
        return np.where(a < f32(1), (f32(0.5) * d) * d, a - f32(0.5)).astype(f32)


def crit_accum(crit, d, acc):
    """acc + crit_value(d), l2's square fused into the sum."""
    if crit == L2:
        return fma32(d, d, acc)
    with _err():
        return (np.asarray(acc, f32) + crit_value(crit, d)).astype(f32)


def crit_grad(crit, d):
    d = np.asarray(d, f32)
    sg = np.where(d > 0, f32(1), np.where(d < 0, f32(-1), f32(0))).astype(f32)
    if crit == L1:
        return sg
    if crit == L2:
        with _err():
            return d + d
    with _err():
        return np.where(np.abs(d) < f32(1), d, sg).astype(f32)


# ---------------------------------------------------------------------------------------------------------- sigmoid
def sigmoid2(x):
    """sigmoid2 (reductions.cuh) where expf is exact: (s, ds) fp32.  NaN gives NaN."""
    x = np.asarray(x, f32)
    with _err():
        ax = np.abs(x)
        ok = (ax == 0) | (ax >= f32(EXACT_LOGIT)) | np.isnan(x)
        if not ok.all():
            raise ValueError("sigmoid2 is modelled only at x = +-0, |x| >= 110 and NaN")
        q = np.where(ax == 0, f32(1), np.where(np.isnan(x), f32(np.nan), f32(0))).astype(f32)
        r = f32(1) / (f32(1) + q)
        s = np.where(x >= 0, r, q * r).astype(f32)
        ds = (q * r) * r
    return s, ds.astype(f32)


# ---------------------------------------------------------------------------------------------------------- finalize
def _fma64(a, b, c):
    a, b, c = float(a), float(b), float(c)
    if not all(np.isfinite(v) for v in (a, b, c)):
        return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))          # int / int division rounds correctly


def finalize(x, scale, bias, weights=None, sizes=None):
    """finalize_kernel: x [B, S] fp32 -> fp32(bias + sum_s coef_s * sum_b x[b, s]), coef_s = scale * w_s / |s| (weights,
    sizes given) else scale."""
    x = np.asarray(x, f32)
    if x.ndim == 1:
        x = x[:, None]
    total = f64(bias)
    with _err():
        for s in range(x.shape[1]):
            xs, _ = strided(x[:, s].astype(f64)[None], 0.0)
            part = np.zeros((1, THREADS), f64)
            for r in range(xs.shape[1]):
                part = part + xs[:, r]
            total_s = block_sum(part)[0]
            coef = f64(scale) if weights is None else (f64(scale) * f64(f32(weights[s]))) / f64(sizes[s])
            total = f64(_fma64(coef, total_s, total))
        return f32(total)


# ---------------------------------------------------------------------------------------------------------- IoU
def iou_forward(x, t, vector=True):
    """iou_forward_kernel<true, float> and the loss: x, t [P, hw] fp32 -> (stats [P, 4], loss).  ``vector`` is the float4
    path, which the kernel takes when hw % 4 == 0 and x, t are 16-byte aligned."""
    x, t = np.asarray(x, f32), np.asarray(t, f32)
    P, hw = x.shape
    s, _ = sigmoid2(x)
    vector = vector and hw % 4 == 0
    a = np.zeros((3, P, THREADS), f32)
    with _err():
        if vector:                 # thread i: elements 4i .. 4i + 3, then 4 (i + 256) ...
            ss, _ = strided(s.reshape(P, hw // 4, 4).transpose(0, 2, 1), 0)
            ts, _ = strided(t.reshape(P, hw // 4, 4).transpose(0, 2, 1), 0)
            valid, _ = strided(np.ones((1, 4, hw // 4), bool), False)
            steps = [(ss[:, e, r], ts[:, e, r], valid[:, e, r]) for r in range(ss.shape[2]) for e in range(4)]
        else:
            ss, _ = strided(s, 0)
            ts, _ = strided(t, 0)
            valid, _ = strided(np.ones((1, hw), bool), False)
            steps = [(ss[:, r], ts[:, r], valid[:, r]) for r in range(ss.shape[1])]
        for sv, tv, m in steps:
            a[0] = np.where(m, fma32(sv, tv, a[0]), a[0])
            a[1] = np.where(m, fma32(tv, tv, a[1]), a[1])
            a[2] = np.where(m, fma32(sv, sv, a[2]), a[2])
        I, T, S = (block_sum(a[k]) for k in range(3))
        iou = (I + EPS) / iou_den(I, T, S)
    stats = np.stack([I, T, S, iou], 1).astype(f32)
    return stats, finalize(stats[:, 3], -1.0 / P, 1.0)


def iou_den(I, T, S):
    with _err():
        return ((T + S) - I) + EPS


def iou_backward(x, t, stats, g):
    """iou_backward_kernel: d loss / d x [P, hw]; elementwise, so the same on both paths."""
    x, t, st = np.asarray(x, f32), np.asarray(t, f32), np.asarray(stats, f32)
    P = x.shape[0]
    s, ds = sigmoid2(x)
    with _err():
        N = (st[:, 0] + EPS)[:, None]
        D = iou_den(st[:, 0], st[:, 1], st[:, 2])[:, None]
        coef = -f32(g) / ((f32(P) * D) * D)
        inner = fma32(t, np.broadcast_to(D, t.shape), -(N * ((s + s) - t)))
        return ((coef * inner) * ds).astype(f32)


# ---------------------------------------------------------------------------------------------------------- landmarks
def _lmk_diff(p, pm, t, tm):
    p, t = np.asarray(p, f32), np.asarray(t, f32)
    pm, tm = np.asarray(pm, f32)[..., None], np.asarray(tm, f32)[..., None]
    with _err():
        return fma32(p, np.broadcast_to(pm, p.shape), -(t * tm))


def landmarks_forward(p, pm, t, tm, crit):
    """lmk_forward_kernel + finalize: p, t [B, N, 2], pm, tm [B, N] -> (partial [B], loss)."""
    B, N, _ = np.shape(p)
    cv = crit_value(crit, _lmk_diff(p, pm, t, tm)).reshape(B, 2 * N)
    acc = np.zeros(B, f64)
    for k in range(2 * N):
        acc = acc + cv[:, k].astype(f64)
    partial = acc.astype(f32)
    return partial, finalize(partial, 1.0 / (2.0 * B * N), 0.0)


def landmarks_backward(p, pm, t, tm, crit, g):
    B, N, _ = np.shape(p)
    with _err():
        scale = f32(g) / ((f32(2) * f32(B)) * f32(N))
        cg = crit_grad(crit, _lmk_diff(p, pm, t, tm))
        return ((scale * cg) * np.asarray(pm, f32)[..., None]).astype(f32)


# ---------------------------------------------------------------------------------------------------------- vertex subsets
class Subsets:
    """The tables dad3d_vsub_create builds: sets as given (indices in [0, V)), weights fp32."""

    def __init__(self, sets: Sequence, weights: Sequence[float], V: int):
        self.sets = [np.asarray(s, np.int64).reshape(-1) for s in sets]
        self.w = np.asarray(weights, f32)
        self.V = V
        self.sizes = [len(s) for s in self.sets]
        self.off = np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int64)
        idx = np.concatenate(self.sets)
        self.ent_set = np.repeat(np.arange(len(self.sets)), self.sizes)
        self.ent_pos = np.arange(len(idx)) - self.off[self.ent_set]
        order = np.argsort(idx, kind="stable")                       # ascending entries per vertex
        self.idx = idx
        self._order = order
        counts = np.bincount(idx, minlength=V)
        self.inv_off = np.concatenate([[0], np.cumsum(counts)])


def _ext(vals, is_max, init):
    """Ext reduction over axis 1 of vals [B, n]: (value [B], index [B]) -- the first position equal to the extreme among
    the non-NaN values, its own value (sign of zero kept); (init, INT_MAX) when every value is NaN."""
    with _err():
        ext = (np.fmax if is_max else np.fmin).reduce(np.where(np.isnan(vals), f32(np.nan), vals), axis=1)
        hit = vals == ext[:, None]
        anyhit = hit.any(1)
        i = np.where(anyhit, hit.argmax(1), INT_MAX)
        v = np.where(anyhit, vals[np.arange(len(vals)), np.minimum(i, vals.shape[1] - 1)], f32(init))
    return v.astype(f32), i.astype(np.int64)


def vsub_forward(v, t, subsets: Subsets, crit, normalize):
    """vsub_forward_kernel<K, NORM> + finalize: v, t [B, V, K] -> (records [B, S, 32] fp32 with unwritten words NaN,
    loss)."""
    v, t = np.asarray(v, f32), np.asarray(t, f32)
    B, V, K = v.shape
    S = len(subsets.sets)
    rec = np.full((B, S, RECORD_FLOATS), np.nan, f32)
    ri = rec.view(np.int32)
    for s, I in enumerate(subsets.sets):
        n = len(I)
        vs, ts = v[:, I], t[:, I]                                   # [B, n, K]
        with _err():
            if not normalize:
                dv = vs - ts
                a = np.zeros((B, THREADS), f32)
                for r in range(-(-n // THREADS)):
                    j = np.arange(r * THREADS, min(n, (r + 1) * THREADS))
                    for c in range(K):
                        a[:, j % THREADS] = crit_accum(crit, dv[:, j, c], a[:, j % THREADS])
                rec[:, s, LOSS] = block_sum(a)
                continue
            lo = [_ext(x[:, :, c], False, np.inf) for x in (vs, ts) for c in range(K)]
            hi = [_ext(x[:, :, c] - lo[k * K + c][0][:, None], True, -np.inf) for k, x in enumerate((vs, ts))
                  for c in range(K)]
            half = [f32(0.5) * h[0] for h in hi]
            cen = [np.stack([(x[:, :, c] - lo[k * K + c][0][:, None]) - half[k * K + c][:, None] for c in range(K)], 2)
                   for k, x in enumerate((vs, ts))]                  # [B, n, K]
            top = [_ext(cc.reshape(B, n * K), True, -np.inf) for cc in cen]
            M, tM = top[0][0], top[1][0]
            u = cen[0] / M[:, None, None]
            w = cen[1] / tM[:, None, None]
            d = u - w
            cd = crit_grad(crit, d)
            a = np.zeros((2 + K, B, THREADS), f32)
            for r in range(-(-n // THREADS)):
                j = np.arange(r * THREADS, min(n, (r + 1) * THREADS))
                lane = j % THREADS
                for c in range(K):
                    a[0][:, lane] = crit_accum(crit, d[:, j, c], a[0][:, lane])
                    a[1][:, lane] = fma32(cd[:, j, c], u[:, j, c], a[1][:, lane])
                    a[2 + c][:, lane] = a[2 + c][:, lane] + cd[:, j, c]
            sums = [block_sum(a[k]) for k in range(2 + K)]
        rec[:, s, LOSS] = sums[0]
        rec[:, s, M_], rec[:, s, TM], rec[:, s, SCO] = M, tM, sums[1]
        ni = top[0][1]
        ri[:, s, NSTAR] = np.where(ni == INT_MAX, -1, ni // K)
        ri[:, s, CSTAR] = np.where(ni == INT_MAX, -1, ni % K)
        for c in range(3):
            if c < K:
                rec[:, s, MN + c], rec[:, s, TMN + c] = lo[c][0], lo[K + c][0]
                rec[:, s, HALF + c], rec[:, s, THALF + c] = half[c], half[K + c]
                ri[:, s, AMIN + c], ri[:, s, AMAX + c] = lo[c][1], hi[c][1]
                rec[:, s, SG + c] = sums[2 + c]
            else:
                rec[:, s, [MN + c, TMN + c, HALF + c, THALF + c, SG + c]] = 0
                ri[:, s, AMIN + c] = ri[:, s, AMAX + c] = -1
    loss = finalize(rec[:, :, LOSS], 1.0 / (float(B) * K), 0.0, subsets.w, subsets.sizes)
    return rec, loss


def vsub_backward(v, t, subsets: Subsets, crit, normalize, rec, g):
    """vsub_backward_kernel<K, NORM>: d loss / d v [B, V, K], each vertex's entries summed in ascending entry order."""
    v, t, rec = np.asarray(v, f32), np.asarray(t, f32), np.asarray(rec, f32)
    B, V, K = v.shape
    ri = rec.view(np.int32)
    acc = np.zeros((B, V, K), f32)
    counts = np.diff(subsets.inv_off)
    order = subsets._order
    with _err():
        for k in range(int(counts.max(initial=0))):
            vt = np.nonzero(counts > k)[0]                          # vertices with a k-th entry
            ent = order[subsets.inv_off[vt] + k]
            s = subsets.ent_set[ent]
            pos = subsets.ent_pos[ent]
            n = np.asarray(subsets.sizes)[s]
            coef = f32(g) * (subsets.w[s] / ((f32(B) * n.astype(f32)) * f32(K)))    # [m]
            x, y = v[:, vt], t[:, vt]                                # [B, m, K]
            R, Ri = rec[:, s], ri[:, s]                              # [B, m, 32]
            if not normalize:
                for c in range(K):
                    acc[:, vt, c] = fma32(np.broadcast_to(coef, (B, len(vt))), crit_grad(crit, x[..., c] - y[..., c]),
                                          acc[:, vt, c])
                continue
            M = R[..., M_]
            dM = ((-coef) * R[..., SCO]) / M
            for c in range(K):
                u = ((x[..., c] - R[..., MN + c]) - R[..., HALF + c]) / M
                w = ((y[..., c] - R[..., TMN + c]) - R[..., THALF + c]) / R[..., TM]
                d = (coef * crit_grad(crit, u - w)) / M
                A = f32(-0.5) * (((coef * R[..., SG + c]) / M) + np.where(Ri[..., CSTAR] == c, dM, f32(0)))
                d = np.where((pos == Ri[..., NSTAR]) & (Ri[..., CSTAR] == c), d + dM, d)
                d = np.where(pos == Ri[..., AMAX + c], d + A, d)
                d = np.where(pos == Ri[..., AMIN + c], d + A, d)
                acc[:, vt, c] = acc[:, vt, c] + d
    return acc
