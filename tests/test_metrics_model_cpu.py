"""-m "not gpu": the exact model of csrc/metrics.cu (tests/metrics_model.py) against the reference's own metric functions and
classes (model_training/metrics/iou.py, keypoints.py, loaded through the reference harness with the torchmetrics stand-in
of tests/torchmetrics_stub), the torch arithmetic the kernels restate, exact threshold ties, and the package's input
errors (checked before any device work, so they hold without a GPU)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ref_harness as R
from tests import metrics_model as M

STUB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "torchmetrics_stub")


def _ref():
    if not R.available():
        pytest.skip("reference harness not available")
    R.activate()
    if STUB not in sys.path:
        sys.path.insert(0, STUB)
    from model_training.metrics import iou, keypoints
    return iou, keypoints


# ---------------------------------------------------------------------------------------------- the pinned arithmetic
def test_torch_arithmetic_the_kernels_restate():
    rng = np.random.default_rng(0)
    norm = rng.uniform(1, 1000, 100000).astype(np.float32)
    # threshold * norm: fp32(threshold) times the fp32 tensor, one rounding (not the product in double)
    assert np.array_equal((0.05 * torch.from_numpy(norm)).numpy(), np.float32(0.05) * norm)
    assert not np.array_equal((0.05 * torch.from_numpy(norm)).numpy(), (0.05 * norm.astype(np.float64)).astype(np.float32))
    # err < 0.05 * 2.0: the double bound is rounded to fp32 before the comparison; fp32(0.1) > 0.1 in double
    e = torch.tensor([np.float32(0.1)])
    assert float(np.float32(0.1)) > 0.1 and not bool(e > 0.05 * 2.0) and not bool(e < 0.05 * 2.0)
    assert np.float32(0.05) * np.float32(2.0) == np.float32(0.05 * 2.0)           # so fp32(thr) * 2.0 is that bound
    # count / bs: fp32(count) / fp32(bs)
    for B in (3, 7, 999, 4133):
        for k in range(0, B + 1, max(1, B // 50)):
            assert ((torch.arange(B) < k).sum() / B).numpy() == np.float32(k) / np.float32(B)
    # the box norm: an int32 product (wrapping), then fp32 sqrt
    box = torch.tensor([[0, 0, 70000, 70000], [0, 0, 3, 5]], dtype=torch.int32)
    got = torch.sqrt(box[:, 2] * box[:, 3])
    assert got.dtype == torch.float32
    w = [(70000, 70000), (3, 5)]
    want = M.keypoint_errors([M.group(np.zeros((2, 1, 2)), np.zeros((2, 1, 2)),
                                      box=(np.array([a for a, _ in w]), np.array([b for _, b in w])))])[:, 0, 1]
    assert np.array_equal(got.numpy(), want)
    # uint8_to_float32 (model/flame.py:232-236): fp32(u) / 255 rounded once
    u = torch.arange(256, dtype=torch.uint8)
    assert np.array_equal(u.div(255.0).to(torch.float32).numpy(), M.target_value(u.numpy()))


def test_fma_emulation_is_correctly_rounded():
    from fractions import Fraction
    rng = np.random.default_rng(1)
    a, b, c = (rng.standard_normal(3000).astype(np.float32) * 10 ** rng.uniform(-3, 3, 3000).astype(np.float32)
               for _ in range(3))
    got = M.fma32(a, b, c)
    for i in range(0, 3000, 7):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda x: (abs(Fraction(float(x)) - exact), int(np.float32(x).view(np.int32)) & 1))
        assert got[i] == best, i


# ---------------------------------------------------------------------------------------------- model vs reference
def _heatmaps(B, C, H, seed, u8=False):
    g = torch.Generator().manual_seed(seed)
    o = torch.rand(B, C, H, H, generator=g)
    t = (torch.rand(B, C, H, H, generator=g) * 255).to(torch.uint8)
    return o, (t if u8 else t.float() / 255)


@pytest.mark.parametrize("shape", [(2, 3, 8, 8), (3, 68, 64, 64), (1, 2, 5, 7)])
def test_iou_model_matches_reference(shape):
    iou, _ = _ref()
    B, C, H, W = shape
    g = torch.Generator().manual_seed(B * H)
    o = torch.rand(B, C, H, W, generator=g)
    t = torch.rand(B, C, H, W, generator=g) ** 3
    want = iou.soft_iou(o.double(), t.double()).item()
    stats = M.iou_stats(o.numpy().reshape(B * C, -1), t.numpy().reshape(B * C, -1))
    got = M.reduce(stats=stats)[0][0]
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)
    tu = (t * 255).to(torch.uint8)
    want = iou.soft_iou(o.double(), tu.double() / 255).item()
    got = M.reduce(stats=M.iou_stats(o.numpy().reshape(B * C, -1), tu.numpy().reshape(B * C, -1)))[0][0]
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)


def _keypoints(B, N, K, seed, box=True):
    rng = np.random.default_rng(seed)
    t = rng.uniform(0, 256, (B, N, K)).astype(np.float32)
    p = (t + rng.normal(0, 1, (B, N, K)) * rng.uniform(0.5, 15, (B, 1, 1))).astype(np.float32)
    bb = np.stack([rng.integers(0, 300, B), rng.integers(0, 300, B), rng.integers(40, 400, B), rng.integers(40, 400, B)],
                  1).astype(np.int32) if box else None
    return p, t, bb


def _clear(err, norm, thresholds, gap=1e-4):
    """True where no err / (thr * norm) is within ``gap`` of 1."""
    ok = np.ones(err.shape, bool)
    for thr in thresholds:
        ok &= np.abs(err.astype(np.float64) / (thr * norm.astype(np.float64)) - 1) > gap
    return ok


@pytest.mark.parametrize("K,box", [(2, True), (3, False), (2, False)])
@pytest.mark.parametrize("B", [1, 5, 300])
def test_keypoint_model_matches_reference(B, K, box):
    _, kp = _ref()
    p, t, bb = _keypoints(B, 68, K, B * K, box)
    if K == 3:
        p, t = p / 256, t / 256
    rec = M.keypoint_errors([M.group(p, t, box=(bb[:, 2], bb[:, 3]) if box else None)])
    vals, per_head, _ = M.reduce(records=rec, thresholds=(0.05, 0.1))
    P, T = torch.from_numpy(p).double(), torch.from_numpy(t).double()
    BB = torch.from_numpy(bb) if box else None
    want_nme = kp.keypoints_nme(P, T, BB).item()
    assert abs(vals[0] - want_nme) <= 1e-6 * abs(want_nme)
    want_heads = kp.keypoints_nme(P, T, BB, reduce="none").numpy()
    assert np.allclose(per_head[:, 0], want_heads, rtol=1e-6, atol=0)
    ok = _clear(rec[:, 0, 0], rec[:, 0, 1], (0.05, 0.1))
    for i, thr in enumerate((0.05, 0.1)):
        for below in (True, False):
            want = kp.percentage_of_errors_below_IOD(P[ok], T[ok], BB[ok] if box else None, threshold=thr, below=below)
            got = M.reduce(records=rec[ok], thresholds=(thr,), below=below)[0][1]
            assert got == np.float32(want.item()), (thr, below)


def test_normalized_group_matches_reference_normalize_to_cube():
    _, kp = _ref()
    from model_training.model.utils import normalize_to_cube
    rng = np.random.default_rng(4)
    p = rng.normal(0, 0.1, (9, 5023, 3)).astype(np.float32)
    t = (p + rng.normal(0, 0.003, p.shape)).astype(np.float32)
    idx = np.sort(rng.choice(5023, 191, replace=False)).astype(np.int32)
    rec = M.keypoint_errors([M.group(p, t, index=idx, normalize=True)])
    P, T = torch.from_numpy(p).double()[:, idx], torch.from_numpy(t).double()[:, idx]
    want = kp.keypoints_nme(normalize_to_cube(P), normalize_to_cube(T), reduce="none").numpy()
    assert np.allclose(rec[:, 0, 0] / rec[:, 0, 1], want, rtol=1e-5, atol=0)


def test_presence_products_follow_the_step():
    """(lm * img_size) * presence and (t * presence) * img_size (flame_lightning_model.py:316-319), one rounding each."""
    rng = np.random.default_rng(2)
    lm = rng.uniform(-0.2, 1.2, (4, 68, 2)).astype(np.float32)
    t = rng.uniform(0, 1, (4, 68, 2)).astype(np.float32)
    pres = rng.random((4, 68)) < 0.7
    pres[1] = False
    lm[2, 3, 0] = np.nan                               # masked out: NaN * 0 is still NaN, as in torch
    pres[2, 3] = False
    g = M.group(lm, t, presence=pres, pred_scale=256, target_scale=256)
    p_m, t_m = M._operands(g)
    P, T, PR = torch.from_numpy(lm), torch.from_numpy(t), torch.from_numpy(pres)
    assert np.array_equal((P * 256 * PR[..., None]).numpy(), p_m, equal_nan=True)
    assert np.array_equal((T * PR[..., None] * 256).numpy(), t_m)
    rec = M.keypoint_errors([g])
    assert rec[1, 0, 0] == 0 and np.isnan(rec[2, 0, 0])


@pytest.mark.parametrize("below", [True, False])
def test_exact_ties_are_not_counted(below):
    """err == fp32(thr) * norm exactly: neither err < bound nor err > bound, in the reference and in the model."""
    _, kp = _ref()
    B = 6
    side = np.array([10, 20, 7, 30, 11, 40], np.int32)
    box = np.stack([np.zeros(B), np.zeros(B), side, side], 1).astype(np.int32)
    bound = np.float32(0.05) * np.sqrt(side.astype(np.int64) ** 2).astype(np.float32)
    p = np.zeros((B, 1, 2), np.float32)
    t = np.zeros((B, 1, 2), np.float32)
    p[:, 0, 0] = bound
    p[3, 0, 0] = np.nextafter(bound[3], np.float32(0))              # one just below, one just above
    p[4, 0, 0] = np.nextafter(bound[4], np.float32(1))
    rec = M.keypoint_errors([M.group(p, t, box=(box[:, 2], box[:, 3]))])
    assert np.array_equal(rec[:, 0, 0], p[:, 0, 0])
    got = M.reduce(records=rec, thresholds=(0.05,), below=below)[0][1]
    want = kp.percentage_of_errors_below_IOD(torch.from_numpy(p), torch.from_numpy(t), torch.from_numpy(box),
                                             threshold=0.05, below=below)
    assert got == np.float32(want.item()) == np.float32(1) / np.float32(B)
    # the 3D bound 0.05 * 2.0 with err exactly fp32(0.1)
    e = np.full((2, 1, 3), 0, np.float32)
    e[0, 0, 0] = np.float32(0.1)
    z = np.zeros_like(e)
    rec = M.keypoint_errors([M.group(e, z)])
    got = M.reduce(records=rec, thresholds=(0.05,), below=below)[0][1]
    want = kp.percentage_of_errors_below_IOD(torch.from_numpy(e), torch.from_numpy(z), threshold=0.05, below=below)
    assert got == np.float32(want.item())


def test_non_finite_values_propagate():
    _, kp = _ref()
    p, t, bb = _keypoints(5, 68, 2, 3)
    p[1, 7, 0] = np.nan
    bb[3, 2] = 0                                                       # zero-area box: err / 0
    rec = M.keypoint_errors([M.group(p, t, box=(bb[:, 2], bb[:, 3]))])
    vals = M.reduce(records=rec, thresholds=(0.05, 0.1))[0]
    P, T, BB = torch.from_numpy(p), torch.from_numpy(t), torch.from_numpy(bb)
    assert np.isnan(vals[0]) and np.isnan(kp.keypoints_nme(P, T, BB).item())
    for i, thr in enumerate((0.05, 0.1)):
        assert vals[1 + i] == np.float32(kp.percentage_of_errors_below_IOD(P, T, BB, threshold=thr).item())
    # a degenerate normalize_to_cube (every vertex equal) divides 0 / 0
    v = np.ones((1, 4, 3), np.float32)
    rec = M.keypoint_errors([M.group(v, v, normalize=True)])
    assert np.isnan(rec[0, 0, 0])


def test_reference_classes_forward_and_multi_batch_compute():
    """The reference's classes over the stand-in: forward returns the batch's value (compute_on_step), compute() the mean
    of the batch values -- what the model gives per batch."""
    iou, kp = _ref()
    from torchmetrics import MetricCollection
    m_iou = iou.SoftIoUMetric(compute_on_step=True)
    coll = MetricCollection({"fr_2d_005": kp.FailureRate(compute_on_step=True, threshold=0.05, below=True),
                             "fr_2d_01": kp.FailureRate(compute_on_step=True, threshold=0.1, below=True),
                             "nme_2d": kp.KeypointsNME(compute_on_step=True)})
    batch_vals = []
    for i, B in enumerate((7, 3, 11)):
        o, t = _heatmaps(B, 4, 8, i)
        got = m_iou(o, t)
        want = M.reduce(stats=M.iou_stats(o.numpy().reshape(B * 4, -1), t.numpy().reshape(B * 4, -1)))[0][0]
        assert abs(got.item() - want) <= 1e-6 * abs(want)
        p, tk, bb = _keypoints(B, 68, 2, 10 + i)
        rec = M.keypoint_errors([M.group(p, tk, box=(bb[:, 2], bb[:, 3]))])
        assert _clear(rec[:, 0, 0], rec[:, 0, 1], (0.05, 0.1)).all()
        vals = M.reduce(records=rec, nme_scale=100.0, thresholds=(0.05, 0.1))[0]
        out = coll(torch.from_numpy(p), {"keypoints": torch.from_numpy(tk), "bboxes": torch.from_numpy(bb)})
        assert list(out) == ["fr_2d_005", "fr_2d_01", "nme_2d"]
        assert out["fr_2d_005"].item() == vals[1] and out["fr_2d_01"].item() == vals[2]
        assert abs(out["nme_2d"].item() - vals[0]) <= 1e-5 * abs(vals[0])
        batch_vals.append((got.item(), [out[k].item() for k in out]))
    assert abs(m_iou.compute().item() - np.mean([v[0] for v in batch_vals])) <= 1e-6
    final = coll.compute()
    for j, k in enumerate(final):
        assert abs(final[k].item() - np.mean([v[1][j] for v in batch_vals])) <= 1e-5 * max(1, abs(final[k].item()))
    m_iou.reset()
    assert m_iou.total.item() == 0


def test_epoch_accumulation_is_batch_size_weighted():
    epoch = np.zeros(3)
    sizes, vals = (64, 64, 17), []
    for i, B in enumerate(sizes):
        p, t, bb = _keypoints(B, 68, 2, 20 + i)
        rec = M.keypoint_errors([M.group(p, t, box=(bb[:, 2], bb[:, 3]))])
        v, _, epoch = M.reduce(records=rec, thresholds=(0.05,), epoch=epoch, weight=float(B))
        vals.append(v)
    want = (np.array(vals, np.float64) * np.array(sizes)[:, None]).sum(0) / sum(sizes)
    assert np.array_equal(M.epoch_values(epoch), want.astype(np.float32))


# ---------------------------------------------------------------------------------------------- the package's errors
def test_input_errors():
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.metrics import FlameStepMetrics, keypoints_nme, percentage_of_errors_below_IOD, soft_iou
    z = torch.zeros
    with pytest.raises(TypeError):
        soft_iou(z(2, 3, 4, 4), z(2, 3, 4, 4, dtype=torch.uint8))        # the reference's target ** 2 wraps on uint8
    with pytest.raises(TypeError):
        soft_iou(z(2, 3, 4, 4, dtype=torch.int32), z(2, 3, 4, 4))
    with pytest.raises(ValueError):
        soft_iou(z(2, 3, 4, 4), z(2, 3, 4, 5))
    with pytest.raises(ValueError):
        soft_iou(z(2, 3, 16), z(2, 3, 16))
    with pytest.raises(ValueError):
        keypoints_nme(z(2, 5, 4), z(2, 5, 4))
    with pytest.raises(ValueError):
        keypoints_nme(z(2, 5, 2), z(2, 6, 2))
    with pytest.raises(ValueError):
        percentage_of_errors_below_IOD(z(2, 5), z(2, 5))
    with pytest.raises(TypeError):
        percentage_of_errors_below_IOD(z(2, 5, 2, dtype=torch.int64), z(2, 5, 2))
    with pytest.raises(_lib.Dad3dError):                                 # there is no CPU path
        keypoints_nme(z(2, 5, 2), z(2, 5, 2))
    with pytest.raises(ValueError):
        FlameStepMetrics(face_indices=[0, 5023])
    with pytest.raises(ValueError):
        FlameStepMetrics(thresholds=())
    m = FlameStepMetrics()
    assert m.names == ["heatmap_iou", "nme_2d", "fr_2d_005", "fr_2d_01", "reproject_nme_2d", "reproject_fr_2d_005",
                       "reproject_fr_2d_01", "nme_3d", "fr_3d_005", "fr_3d_01"]
    with pytest.raises(ValueError):
        m.step({"OUTPUT_3DMM_PARAMS": z(2, 413), "OUTPUT_LANDMARKS_HEATMAP": z(2, 68, 64, 64)}, {})
