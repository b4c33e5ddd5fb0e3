"""-m gpu: every kernel of csrc/loss.cu against the exact model (tests/loss_model.py), bit for bit, through the C ABI.

Every output -- statistics, partial sums, records, the loss scalar and the gradients -- sits at a base offset of 0-7 floats
between guard bands filled with a NaN whose payload the device never produces (0x7fbadbad; the GPU's canonical NaN is
0x7fffffff).  The bands must come back unchanged, and no word the kernel writes may keep the sentinel.  Model NaNs are
compared by NaN-ness, every other value by its bits.  The incoming loss gradient is read from device memory and takes the
values 1, 0.37, -2, +0 and -0.

The sigmoid's expf cannot be modelled (MUFU.EX2), so designed logits are +-0 and |x| >= 110, where expf is exact; the
targets carry the rounding variety.  test_device_sigmoid_on_designed_logits confirms the device's s on those logits first.
"""
import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from tests import loss_model as L

pytestmark = pytest.mark.gpu

SENT = 0x7FBADBAD
BAND = 64
GRADS = (1.0, 0.37, -2.0, 0.0, -0.0)
CRITS = (L.L1, L.L2, L.SMOOTH_L1)


def _lib_stream():
    return _lib.load(), torch.cuda.current_stream().cuda_stream


class Guarded:
    """n fp32 words at base offset ``off`` inside a sentinel-filled device buffer."""

    def __init__(self, n, off, dev):
        self.n, self.off = n, off
        self.buf = torch.full((n + 2 * BAND + 8,), SENT, dtype=torch.int32, device=dev)
        self.t = self.buf[BAND + off:BAND + off + n].view(torch.float32)

    def ptr(self):
        return self.t.data_ptr()

    def check(self, written=None):
        """The bands are unchanged; no written word keeps the sentinel.  Returns the words as numpy fp32."""
        b = self.buf.cpu().numpy()
        lo, hi = BAND + self.off, BAND + self.off + self.n
        assert (b[:lo] == SENT).all() and (b[hi:] == SENT).all(), "a guard band was written"
        body = b[lo:hi]
        w = np.ones(self.n, bool) if written is None else np.asarray(written, bool).reshape(-1)
        assert not (body[w] == SENT).any(), "an output word was not written"
        return body.view(np.float32).copy()


def _dev_input(a, off, dev):
    """a (fp32 numpy) as a contiguous device view at float offset ``off``."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1)
    buf = torch.zeros(a.size + 8, dtype=torch.float32, device=dev)
    v = buf[off:off + a.size]
    v.copy_(torch.from_numpy(a))
    return v


def _grad_out(g, dev, off=3):
    go = Guarded(1, off, dev)
    go.t.copy_(torch.tensor([g], dtype=torch.float32))
    return go


def same(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    bad = (gn != wn) | (~gn & (got.view(np.int32) != want.view(np.int32)))
    if bad.any():
        i = np.argwhere(bad)[:5]
        raise AssertionError(f"{int(bad.sum())} of {bad.size} differ, first at {i.tolist()}: "
                             f"got {got[tuple(i.T)]}, want {want[tuple(i.T)]}")


# ---------------------------------------------------------------------------------------------------------- sigmoid
def test_device_sigmoid_on_designed_logits(cuda_device):
    """Planes of one element with t = 1: I = fmaf(s, 1, 0) = s and S = s * s, so the stats show the device's s."""
    lib, st = _lib_stream()
    x = np.array([0.0, -0.0, 110.0, -110.0, 111.5, -300.0, 1e30, -1e30, np.inf, -np.inf], np.float32)
    P = x.size
    xd, td = _dev_input(x, 0, cuda_device), _dev_input(np.ones(P), 0, cuda_device)
    stats, loss = Guarded(4 * P, 0, cuda_device), Guarded(1, 0, cuda_device)
    _lib.check(lib.dad3d_iou_forward(xd.data_ptr(), td.data_ptr(), P, 1, stats.ptr(), loss.ptr(), st), "iou_forward")
    got = stats.check().reshape(P, 4)
    s, ds = L.sigmoid2(x)
    same(got[:, 0], s)
    same(got[:, 2], s * s)
    assert np.array_equal(s, np.array([.5, .5, 1, 0, 1, 0, 1, 0, 1, 0], np.float32))
    same(got, L.iou_forward(x[:, None], np.ones((P, 1), np.float32))[0])


# ---------------------------------------------------------------------------------------------------------- IoU
def _iou_inputs(P, hw, seed):
    rng = np.random.default_rng(seed)
    x = rng.choice(np.array([0.0, -0.0, 110.0, -110.0, 300.0, -300.0], np.float32), (P, hw))
    t = rng.random((P, hw)).astype(np.float32) ** 2
    t[rng.random((P, hw)) < 0.2] = 0
    t[rng.random(P) < 0.15] = 0                                     # empty-target planes
    return x, t


IOU_SHAPES = [(p, hw) for hw in (1, 3, 4, 5) for p in (1, 255, 256, 257, 68 * 64)] + \
    [(p, hw) for hw in (63 * 65, 4096) for p in (1, 255, 257)] + [(68 * 64, 4096)]
# (x offset, t offset, output offset): the float4 path both ways, and the scalar path from each misaligned operand
IOU_OFFSETS = [(0, 0, 0), (1, 1, 5), (0, 1, 4), (1, 0, 0), (0, 0, 3)]


@pytest.mark.parametrize("offsets", IOU_OFFSETS, ids=lambda o: "x%d_t%d_out%d" % o)
@pytest.mark.parametrize("P,hw", IOU_SHAPES)
def test_iou_forward_backward_bit_exact(cuda_device, P, hw, offsets):
    xo, to, oo = offsets
    lib, st = _lib_stream()
    x, t = _iou_inputs(P, hw, P * 7 + hw)
    xd, td = _dev_input(x, xo, cuda_device), _dev_input(t, to, cuda_device)
    stats, loss = Guarded(4 * P, oo, cuda_device), Guarded(1, 7 - oo, cuda_device)
    _lib.check(lib.dad3d_iou_forward(xd.data_ptr(), td.data_ptr(), P, hw, stats.ptr(), loss.ptr(), st), "iou_forward")
    vector = hw % 4 == 0 and xo == 0 and to == 0
    want_stats, want_loss = L.iou_forward(x, t, vector=vector)
    same(stats.check().reshape(P, 4), want_stats)
    same(loss.check(), [want_loss])
    grads = GRADS if P * hw <= 300_000 else GRADS[1:3]
    for g in grads:
        go = _grad_out(g, cuda_device)
        gx = Guarded(P * hw, oo, cuda_device)
        _lib.check(lib.dad3d_iou_backward(xd.data_ptr(), td.data_ptr(), P, hw, stats.t.data_ptr(), go.ptr(), gx.ptr(), st),
                   "iou_backward")
        same(gx.check().reshape(P, hw), L.iou_backward(x, t, want_stats, np.float32(g)))
        go.check()


def test_iou_target_statistic_exact_and_bounds_on_generic_logits(cuda_device):
    """T = sum t^2 does not read x, so it is exact for any logits.  I and S, with s from expf: the kernel's s differs
    from the correctly rounded sigmoid by at most 4 ulp (expf's documented 2 ulp in q, then 1 / (1 + q) and q * r, one
    rounding each), i.e. relatively by 4 * 2^-23; each fmaf adds one rounding (2^-24 relative) per step of the longest
    chain -- the per-thread terms, 5 butterfly steps and 8 warp partials -- to a sum of non-negative terms.  So
    |I - I_64| <= (8 * 2^-23 + (k + 13) * 2^-24) * I_64 (s^2 doubles the s error for S), with k the terms per thread."""
    lib, st = _lib_stream()
    rng = np.random.default_rng(5)
    for P, hw, xo in ((64, 4096, 0), (3, 4095, 1)):
        x = (rng.standard_normal((P, hw)) * 4).astype(np.float32)
        t = (rng.random((P, hw)) ** 3).astype(np.float32)
        xd, td = _dev_input(x, xo, cuda_device), _dev_input(t, 0, cuda_device)
        stats, loss = Guarded(4 * P, 2, cuda_device), Guarded(1, 1, cuda_device)
        _lib.check(lib.dad3d_iou_forward(xd.data_ptr(), td.data_ptr(), P, hw, stats.ptr(), loss.ptr(), st), "iou_forward")
        got = stats.check().reshape(P, 4)
        zero_x = np.zeros_like(x)                                    # T from the exact model with any logits
        same(got[:, 1], L.iou_forward(zero_x, t, vector=(hw % 4 == 0 and xo == 0))[0][:, 1])
        s64 = 1 / (1 + np.exp(-x.astype(np.float64)))
        I64, S64 = (s64 * t).sum(1), (s64 * s64).sum(1)
        k = -(-hw // 256)
        tol = 8 * 2.0 ** -23 + (k + 13) * 2.0 ** -24
        assert (np.abs(got[:, 0] - I64) <= tol * I64).all()
        assert (np.abs(got[:, 2] - S64) <= (tol + 8 * 2.0 ** -23) * S64).all()


# ---------------------------------------------------------------------------------------------------------- landmarks
def _lmk_inputs(B, N, seed):
    rng = np.random.default_rng(seed)
    p = (rng.random((B, N, 2)) * 64).astype(np.float32)
    t = (p + rng.standard_normal((B, N, 2)) * 1.5).astype(np.float32)
    pm = (rng.random((B, N)) < 0.8).astype(np.float32)
    tm = np.where(rng.random((B, N)) < 0.9, pm, 1 - pm).astype(np.float32)
    frac = rng.random((B, N)) < 0.2                                  # fractional presences
    pm[frac] = rng.random(int(frac.sum())).astype(np.float32)
    # exact differences +-0 and +-1: the smooth-l1 branch point and sign's zero
    k = rng.random((B, N)) < 0.25
    q = np.round(p[k] * 4) / 4
    p[k] = q
    pm[k] = tm[k] = 1
    t[k] = q + rng.choice(np.array([0.0, 1.0, -1.0], np.float32), q.shape)
    z = rng.random((B, N)) < 0.05
    p[z], t[z], pm[z], tm[z] = -0.0, 0.0, 1, 1                      # d = fmaf(-0, 1, -(0 * 1)) = -0
    return p, pm, t, tm


@pytest.mark.parametrize("crit", CRITS)
@pytest.mark.parametrize("N", [1, 68, 69])
@pytest.mark.parametrize("B", [1, 127, 128, 129, 300, 4133])
def test_landmarks_bit_exact(cuda_device, B, N, crit):
    lib, st = _lib_stream()
    p, pm, t, tm = _lmk_inputs(B, N, B * 100 + N * 3 + crit)
    off = (B + N) % 8
    d = [_dev_input(a, i % 2, cuda_device) for i, a in enumerate((p, pm, t, tm))]
    partial, loss = Guarded(B, off, cuda_device), Guarded(1, 7 - off, cuda_device)
    _lib.check(lib.dad3d_landmarks_forward(*(a.data_ptr() for a in d), B, N, crit, partial.ptr(), loss.ptr(), st),
               "landmarks_forward")
    want_partial, want_loss = L.landmarks_forward(p, pm, t, tm, crit)
    same(partial.check(), want_partial)
    same(loss.check(), [want_loss])
    for g in GRADS:
        go = _grad_out(g, cuda_device)
        gp = Guarded(B * N * 2, off, cuda_device)
        _lib.check(lib.dad3d_landmarks_backward(*(a.data_ptr() for a in d), B, N, crit, go.ptr(), gp.ptr(), st),
                   "landmarks_backward")
        same(gp.check().reshape(B, N, 2), L.landmarks_backward(p, pm, t, tm, crit, np.float32(g)))


# ---------------------------------------------------------------------------------------------------------- vertex subsets
def _sets(V, rng, singletons):
    """Synthetic index sets: sizes 2 .. ~3000 (1 too when ``singletons``), a nested set, an overlapping one, repeats."""
    sizes = [2, 31, 32, 255, 256, 257]
    sets = [rng.choice(V, n, replace=False) for n in sizes]
    big = np.concatenate([rng.permutation(V)[:2990], rng.choice(V, 10)])  # ~3000, with repeated indices
    sets.append(big)
    sets.append(sets[4][:40])                                        # nested in the 256-set
    sets.append(np.concatenate([sets[3][100:], sets[5][:50], sets[3][100:110]]))   # overlapping, repeats
    if singletons:
        sets = [np.array([7])] + sets + [np.array([V - 1])]
    weights = rng.uniform(0.25, 1.5, len(sets)).astype(np.float32)
    return sets, weights


def _vertices(B, V, K, rng):
    """A dyadic grid (exact ties at every reduction, +-0 included) for half the heads, random values for the rest."""
    v = (rng.integers(-4, 5, (B, V, K)) / 4).astype(np.float32)
    v[v == 0] = rng.choice(np.array([0.0, -0.0], np.float32), int((v == 0).sum()))
    gen = rng.random(B) < 0.5
    v[gen] = rng.standard_normal((int(gen.sum()), V, K)).astype(np.float32)
    t = (v + rng.standard_normal(v.shape).astype(np.float32) * np.float32(0.3)).astype(np.float32)
    tie = rng.random(B) < 0.3                                        # grid targets too: ties in the target's reductions
    t[tie] = (rng.integers(-4, 5, (int(tie.sum()), V, K)) / 4).astype(np.float32)
    return v, t


def _record_mask(S, B, norm):
    m = np.zeros((B, S, L.RECORD_FLOATS), bool)
    m[..., :L.RECORD_WRITTEN if norm else 1] = True
    return m


def _vsub_run(lib, st, dev, v, t, sub_model, sets, weights, crit, norm, grads, off):
    B, V, K = v.shape
    S = len(sets)
    idx = np.ascontiguousarray(np.concatenate(sets).astype(np.int32))
    offs = np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.int32))
    w = np.ascontiguousarray(weights, np.float32)
    import ctypes as C
    h = C.c_void_p()
    _lib.check(lib.dad3d_vsub_create(C.byref(h), idx.ctypes.data, offs.ctypes.data, w.ctypes.data, S, V,
                                     torch.cuda.current_device()), "vsub_create")
    try:
        vd, td = _dev_input(v, off % 2, dev), _dev_input(t, 1 - off % 2, dev)
        rec, loss = Guarded(B * S * L.RECORD_FLOATS, off, dev), Guarded(1, 7 - off, dev)
        _lib.check(lib.dad3d_vsub_forward(h, vd.data_ptr(), td.data_ptr(), B, K, int(norm), crit, rec.ptr(), loss.ptr(),
                                          st), "vsub_forward")
        got_rec = rec.check(_record_mask(S, B, norm)).reshape(B, S, L.RECORD_FLOATS)
        got_loss = loss.check()[0]
        out = []
        for g in grads:
            go = _grad_out(g, dev)
            gv = Guarded(B * V * K, off, dev)
            _lib.check(lib.dad3d_vsub_backward(h, vd.data_ptr(), td.data_ptr(), B, K, int(norm), crit, rec.t.data_ptr(),
                                               go.ptr(), gv.ptr(), st), "vsub_backward")
            out.append(gv.check().reshape(B, V, K))
        return got_rec, got_loss, out
    finally:
        lib.dad3d_vsub_destroy(h)


def _compare_records(got, want, norm):
    n = L.RECORD_WRITTEN if norm else 1
    ints = np.zeros(L.RECORD_FLOATS, bool)
    ints[[L.AMIN, L.AMIN + 1, L.AMIN + 2, L.AMAX, L.AMAX + 1, L.AMAX + 2, L.NSTAR, L.CSTAR]] = True
    for word in range(n):
        if ints[word]:
            assert np.array_equal(got[..., word].view(np.int32), want[..., word].view(np.int32)), word
        else:
            same(got[..., word], want[..., word])


@pytest.mark.parametrize("crit", CRITS)
@pytest.mark.parametrize("K,norm", [(2, False), (2, True), (3, False), (3, True)])
@pytest.mark.parametrize("B", [1, 3, 300])
def test_vertex_subsets_bit_exact(cuda_device, B, K, norm, crit):
    lib, st = _lib_stream()
    rng = np.random.default_rng(B * 10 + K * 2 + int(norm) + 100 * crit)
    V = 3100
    sets, weights = _sets(V, rng, singletons=not norm)
    v, t = _vertices(B, V, K, rng)
    for s in sets:                       # the size-2 set's two vertices differ, so its M and tM are not 0
        if len(s) == 2:
            v[:, s[1], 0], t[:, s[1], 0] = v[:, s[0], 0] + 1, t[:, s[0], 0] + 1
    sub = L.Subsets(sets, weights, V)
    grads = GRADS if B <= 3 else (0.37, -2.0)
    got_rec, got_loss, got_g = _vsub_run(lib, st, cuda_device, v, t, sub, sets, weights, crit, norm, grads, (B + K) % 8)
    want_rec, want_loss = L.vsub_forward(v, t, sub, crit, norm)
    _compare_records(got_rec, want_rec, norm)
    same([got_loss], [want_loss])
    assert np.isfinite(want_loss)
    in_sets = np.zeros(V, bool)
    in_sets[np.concatenate(sets)] = True
    assert not in_sets.all()
    for g, gv in zip(grads, got_g):
        want = L.vsub_backward(v, t, sub, crit, norm, want_rec, np.float32(g))
        same(gv, want)
        assert (gv[:, ~in_sets].view(np.int32) == 0).all()          # a vertex in no set: a written +0


@pytest.mark.parametrize("K", [2, 3])
def test_vertex_subsets_singletons_and_nan_head(cuda_device, K):
    """A size-1 normalised set gives M = 0 and 0 / 0; a NaN in one head's vertices (and one in another head's target)
    stays in that head: every other head's records and gradients are bit-identical to the clean run."""
    lib, st = _lib_stream()
    rng = np.random.default_rng(40 + K)
    V, B = 600, 6
    sets = [rng.choice(V, 300, replace=False), np.array([5]), rng.choice(V, 257, replace=False)]
    weights = np.array([0.5, 0.75, 1.0], np.float32)
    sub = L.Subsets(sets, weights, V)
    v, t = _vertices(B, V, K, rng)
    for crit in CRITS:
        clean = _vsub_run(lib, st, cuda_device, v, t, sub, sets, weights, crit, True, (0.37,), 2)
        vn, tn = v.copy(), t.copy()
        vn[2, sets[0][7], 0] = np.nan
        tn[4, sets[2][3], K - 1] = np.nan
        dirty = _vsub_run(lib, st, cuda_device, vn, tn, sub, sets, weights, crit, True, (0.37,), 5)
        for (rec, loss, gs), (vv, tt) in ((clean, (v, t)), (dirty, (vn, tn))):
            want_rec, want_loss = L.vsub_forward(vv, tt, sub, crit, True)
            _compare_records(rec, want_rec, True)
            same([loss], [want_loss])
            same(gs[0], L.vsub_backward(vv, tt, sub, crit, True, want_rec, np.float32(0.37)))
            assert np.isnan(rec[:, 1, L.LOSS]).all() and np.isnan(loss)          # the singleton's 0 / 0
        keep = [b for b in range(B) if b not in (2, 4)]
        assert np.array_equal(clean[0][keep].view(np.int32), dirty[0][keep].view(np.int32))
        assert np.array_equal(clean[2][0][keep].view(np.int32), dirty[2][0][keep].view(np.int32))


# ---------------------------------------------------------------------------------------------------------- wrappers
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_wrappers_give_the_c_abi_bits(cuda_device, dtype):
    """losses.IoULoss, LandmarksLossWVisibility and vertex_subset_loss: inputs cast to fp32, gradients cast back."""
    from dad_3dheads_b200 import losses
    rng = np.random.default_rng(9)
    g = 0.37
    cast = lambda a: torch.from_numpy(np.asarray(a, np.float32)).to(cuda_device, dtype)
    as32 = lambda a: cast(a).float().cpu().numpy()
    # IoU: [B, C, H, W] = [2, 5, 6, 8]
    x, t = _iou_inputs(10, 48, 1)
    xd = cast(x.reshape(2, 5, 6, 8)).requires_grad_(True)
    loss = losses.IoULoss()(xd, cast(t.reshape(2, 5, 6, 8)))
    (loss * g).backward()
    st, want = L.iou_forward(as32(x), as32(t))
    same([loss.item()], [want])
    want_g = torch.from_numpy(L.iou_backward(as32(x), as32(t), st, np.float32(g))).to(dtype)
    assert torch.equal(xd.grad.cpu().view(-1), want_g.view(-1))
    # landmarks
    p, pm, tt, tm = _lmk_inputs(5, 68, 2)
    for crit, name in zip(CRITS, ("l1", "l2", "smooth_l1")):
        pd = cast(p).requires_grad_(True)
        loss = losses.LandmarksLossWVisibility(name)([pd, cast(pm)], [cast(tt), cast(tm)])
        (loss * g).backward()
        args = [as32(a) for a in (p, pm, tt, tm)]
        same([loss.item()], [L.landmarks_forward(*args, crit)[1]])
        want_g = torch.from_numpy(L.landmarks_backward(*args, crit, np.float32(g))).to(dtype)
        assert torch.equal(pd.grad.cpu(), want_g)
    # vertex subsets, negative indices through VertexSubsets
    V = 300
    sets = [rng.choice(V, 100, replace=False) - V, rng.choice(V, 40, replace=False), np.array([3, -1, 3, 17])]
    weights = [0.5, 0.75, 1.0]
    sub = losses.VertexSubsets(sets, weights, V)
    msub = L.Subsets([np.where(s < 0, s + V, s) for s in sets], weights, V)
    for K, norm in ((3, True), (2, False)):
        v, tv = _vertices(3, V, K, rng)
        for crit, name in zip(CRITS, ("l1", "l2", "smooth_l1")):
            vd = cast(v).requires_grad_(True)
            loss = losses.vertex_subset_loss(vd, cast(tv), sub, name, norm)
            (loss * g).backward()
            rec, want = L.vsub_forward(as32(v), as32(tv), msub, crit, norm)
            same([loss.item()], [want])
            want_g = torch.from_numpy(L.vsub_backward(as32(v), as32(tv), msub, crit, norm, rec, np.float32(g))).to(dtype)
            assert torch.equal(vd.grad.cpu(), want_g)
