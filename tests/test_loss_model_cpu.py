"""-m "not gpu": the exact model of csrc/loss.cu (tests/loss_model.py) pinned to meaning: within rounding of fp64 torch
autograd of the reference's expressions for all three criteria, torch's tie winners at normalize_to_cube's reductions,
the torch arithmetic its explicit-rounding forms restate, and which outputs a NaN reaches."""
import numpy as np
import pytest
import torch

from tests import loss_model as L

TORCH = {L.L1: torch.nn.L1Loss(), L.L2: torch.nn.MSELoss(), L.SMOOTH_L1: torch.nn.SmoothL1Loss()}


def _cube(x):
    """normalize_to_cube (model/utils.py:55-68), restated."""
    x = x - x.min(1, keepdim=True)[0]
    x = x - 0.5 * x.max(1, keepdim=True)[0]
    return x / x.reshape(x.shape[0], -1).max(1)[0][:, None, None]


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


# ---------------------------------------------------------------------------------------------- model vs fp64 autograd
@pytest.mark.parametrize("crit", [L.L1, L.L2, L.SMOOTH_L1])
@pytest.mark.parametrize("K,norm", [(2, False), (2, True), (3, False), (3, True)])
def test_vertex_subset_model_matches_fp64_autograd(K, norm, crit):
    """Loss within 1e-6 relative and gradient within 1e-6 relL2 (a few fp32 roundings per term) on heads without
    near-ties at the reductions or near-kinks of the criterion (random normal vertices)."""
    rng = np.random.default_rng(K * 10 + crit)
    B, V = 4, 400
    v = rng.standard_normal((B, V, K)).astype(np.float32)
    t = (v + 0.3 * rng.standard_normal(v.shape)).astype(np.float32)
    sets = [rng.choice(V, 300, replace=False), rng.choice(V, 40, replace=False), np.array([1, 2, 3, 1, 9])]
    w = [0.5, 0.75, 1.0]
    rec, loss = L.vsub_forward(v, t, L.Subsets(sets, w, V), crit, norm)
    grad = L.vsub_backward(v, t, L.Subsets(sets, w, V), crit, norm, rec, np.float32(1))
    q = torch.from_numpy(v).double().requires_grad_(True)
    f = _cube if norm else (lambda x: x)
    want = sum(TORCH[crit](f(q[:, i]), f(torch.from_numpy(t).double()[:, i])) * wi for wi, i in zip(w, sets))
    want.backward()
    assert abs(loss - want.item()) <= 1e-6 * abs(want.item())
    assert _rel(grad, q.grad.numpy()) <= 1e-6


@pytest.mark.parametrize("crit", [L.L1, L.L2, L.SMOOTH_L1])
def test_landmark_and_iou_models_match_fp64_autograd(crit):
    rng = np.random.default_rng(crit)
    B, N = 9, 68
    p = (rng.random((B, N, 2)) * 64).astype(np.float32)
    t = (p + rng.standard_normal((B, N, 2)) * 1.5).astype(np.float32)
    pm = (rng.random((B, N)) < 0.8).astype(np.float32)
    tm = np.where(rng.random((B, N)) < 0.9, pm, 1 - pm).astype(np.float32)
    _, loss = L.landmarks_forward(p, pm, t, tm, crit)
    grad = L.landmarks_backward(p, pm, t, tm, crit, np.float32(1))
    q = torch.from_numpy(p).double().requires_grad_(True)
    P, T = torch.from_numpy(pm).double()[..., None], torch.from_numpy(tm).double()[..., None]
    want = TORCH[crit](q * P, torch.from_numpy(t).double() * T)
    want.backward()
    assert abs(loss - want.item()) <= 1e-6 * abs(want.item())
    assert _rel(grad, q.grad.numpy()) <= 1e-6
    # IoU on the exact logits
    x = rng.choice(np.array([0.0, -0.0, 110.0, -120.0], np.float32), (12, 64))
    tt = (rng.random((12, 64)) ** 2).astype(np.float32)
    st, loss = L.iou_forward(x, tt)
    gx = L.iou_backward(x, tt, st, np.float32(1))
    q = torch.from_numpy(x).double().requires_grad_(True)
    s, T = q.sigmoid(), torch.from_numpy(tt).double()
    I = (s * T).sum(1)
    want = 1 - ((I + 1e-6) / ((T * T).sum(1) + (s * s).sum(1) - I + 1e-6)).mean()     # keypoint_losses.py:5-31
    want.backward()
    assert abs(loss - want.item()) <= 1e-6 * abs(want.item())
    assert _rel(gx, q.grad.numpy()) <= 1e-6


# ---------------------------------------------------------------------------------------------- tie winners
def test_tie_winners_match_torch_min_max():
    """Exact ties, +-0 among them, at all three reductions: the model's winner is torch's CPU min / max index and keeps
    the winning element's sign of zero."""
    rng = np.random.default_rng(3)
    B, n, K = 64, 33, 3
    v = (rng.integers(-2, 3, (B, n, K)) / 2).astype(np.float32)
    v[v == 0] = rng.choice(np.array([0.0, -0.0], np.float32), int((v == 0).sum()))
    sub = L.Subsets([np.arange(n)], [1.0], n)
    rec, _ = L.vsub_forward(v, v, sub, L.L2, True)
    ri = rec.view(np.int32)
    T = torch.from_numpy(v)
    mn, amin = T.min(1)
    v1 = T - mn[:, None]
    mx, amax = v1.max(1)
    v2 = v1 - 0.5 * mx[:, None]
    top, atop = v2.reshape(B, -1).max(1)
    assert np.array_equal(ri[:, 0, L.AMIN:L.AMIN + 3], amin.numpy())
    assert np.array_equal(ri[:, 0, L.AMAX:L.AMAX + 3], amax.numpy())
    assert np.array_equal(rec[:, 0, L.MN:L.MN + 3].view(np.int32), mn.numpy().view(np.int32))   # sign of zero too
    assert np.array_equal(rec[:, 0, L.HALF:L.HALF + 3], (0.5 * mx).numpy())
    assert np.array_equal(rec[:, 0, L.M_].view(np.int32), top.numpy().view(np.int32))
    assert np.array_equal(ri[:, 0, L.NSTAR] * K + ri[:, 0, L.CSTAR], atop.numpy())


# ---------------------------------------------------------------------------------------------- the pinned arithmetic
def test_torch_arithmetic_the_kernels_restate():
    rng = np.random.default_rng(0)
    a, b, c, d = (rng.standard_normal(100000).astype(np.float32) * 8 for _ in range(4))
    A, Bt, Ct, D = map(torch.from_numpy, (a, b, c, d))
    # fp32 products and differences: one rounding each, as numpy's fp32 operations
    assert np.array_equal((A * Bt).numpy(), a * b) and np.array_equal((A - Bt).numpy(), a - b)
    # 0.5 * d * d is (0.5 d) d; 2 d == d + d exactly
    assert np.array_equal((0.5 * A * A).numpy(), (np.float32(0.5) * a) * a)
    assert np.array_equal((2 * A).numpy(), a + a)
    # the fused forms differ from the unfused ones somewhere: fmaf(p, mp, -(t mt)) vs p mp - t mt
    fused = L.fma32(a, b, -(c * d))
    assert not np.array_equal(fused, a * b - c * d)
    want = (torch.from_numpy(a).double() * torch.from_numpy(b).double() - (Ct * D).double()).float().numpy()
    assert np.array_equal(fused, want)                       # fp64 of exact products is exact here, rounded once
    # fmaf(d, d, acc): the exact square plus acc, rounded once
    acc = rng.standard_normal(100000).astype(np.float32)
    assert np.array_equal(L.crit_accum(L.L2, a, acc), (A.double() * A.double() + torch.from_numpy(acc).double()).float().numpy())
    # smooth l1 matches torch's value and gradient on both sides of |d| = 1, and at +-1, +-0
    e = np.concatenate([a, np.float32([1, -1, 0, -0.0, np.nextafter(1, 0, dtype=np.float32)])])
    E = torch.from_numpy(e).requires_grad_(True)
    torch.nn.functional.smooth_l1_loss(E, torch.zeros_like(E), reduction="sum").backward()
    assert np.array_equal(L.crit_value(L.SMOOTH_L1, e), torch.nn.functional.smooth_l1_loss(
        E.detach(), torch.zeros_like(E), reduction="none").numpy())
    assert np.array_equal(L.crit_grad(L.SMOOTH_L1, e), E.grad.numpy())
    assert np.array_equal(L.crit_grad(L.L1, e), torch.sign(torch.from_numpy(e)).numpy())
    # finalize: fp64 fma of the coefficient and the sum, then fp32
    x = rng.standard_normal((1000, 3)).astype(np.float32)
    got = L.finalize(x, 1.0 / 3000, 0.0, np.float32([0.5, 0.75, 1.0]), [7, 9, 11])
    want = sum((1 / 3000 * w / n) * x[:, s].astype(np.float64).sum() for s, (w, n) in enumerate(((0.5, 7), (0.75, 9), (1, 11))))
    assert abs(got - want) <= 2 ** -23 * abs(want)


# ---------------------------------------------------------------------------------------------- NaN patterns
def test_nan_patterns():
    """A NaN difference: l2 passes it to the value and gradient; l1 and smooth l1 pass it to the value, while their
    gradient is sign(d) = 0 for NaN (d > 0 and d < 0 are both false), unlike torch's sign(NaN) = NaN."""
    nan = np.float32([np.nan])
    for crit in (L.L1, L.L2, L.SMOOTH_L1):
        assert np.isnan(L.crit_value(crit, nan)).all()
    assert np.isnan(L.crit_grad(L.L2, nan)).all()
    assert (L.crit_grad(L.L1, nan) == 0).all() and (L.crit_grad(L.SMOOTH_L1, nan) == 0).all()
    # landmarks: a NaN prediction (present) makes that head's partial NaN; a NaN target likewise; a NaN prediction under a
    # zero presence is still NaN (NaN * 0), as in torch
    B, N = 3, 4
    p, t = np.ones((B, N, 2), np.float32), np.zeros((B, N, 2), np.float32)
    pm = np.ones((B, N), np.float32)
    p[0, 1, 0], t[1, 2, 1] = np.nan, np.nan
    pm[2, 3] = 0
    p[2, 3, 1] = np.nan
    for crit in (L.L1, L.L2, L.SMOOTH_L1):
        part, loss = L.landmarks_forward(p, pm, t, pm, crit)
        assert np.isnan(part).all() and np.isnan(loss)
        g = L.landmarks_backward(p, pm, t, pm, crit, np.float32(1))
        bad = np.isnan(g)
        if crit == L.L2:
            assert bad[0, 1, 0] and bad[1, 2, 1] and bad[2, 3, 1] and bad.sum() == 3
        else:
            assert not bad.any()
    # vertex subsets, normalised: a NaN in a head's prediction never wins a reduction; it makes that head's set loss NaN,
    # and the gradient NaN at that vertex (through u) -- a NaN target likewise reaches the loss and, through w, the
    # gradient of the vertex that shares its index
    rng = np.random.default_rng(1)
    v = rng.standard_normal((2, 20, 3)).astype(np.float32)
    t = (v + 0.1).astype(np.float32)
    v[0, 4, 1] = np.nan
    t[1, 6, 0] = np.nan
    sub = L.Subsets([np.arange(20)], [1.0], 20)
    rec, loss = L.vsub_forward(v, t, sub, L.L2, True)
    assert np.isnan(rec[:, 0, L.LOSS]).all() and np.isnan(loss)
    assert np.isfinite(rec[0, 0, L.MN:L.M_ + 1]).all()                    # the NaN never won a reduction
    g = L.vsub_backward(v, t, sub, L.L2, True, rec, np.float32(1))
    assert np.isnan(g[0, 4, 1]) and np.isnan(g[1, 6, 0])
