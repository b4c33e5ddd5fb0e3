"""-m gpu: the training metrics (dad_3dheads_b200.metrics, csrc/metrics.cu) against the exact model (tests/metrics_model.py)
bit for bit, and against the reference's metric functions and the metric block of FlameLightningModel._step_fn, restated
here from the reference's own pieces and run in fp64 on the CPU.

Bounds: continuous values within 1e-5 relative; counts exactly.  Counts compare exactly only where no head's
err / (thr * norm) lies within 1e-4 of 1 (an fp32 / fp64 difference could flip it there), so the reference comparison runs
on the heads that are clear of every threshold; exact ties are checked in tests/test_metrics_model_cpu.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from dad_3dheads_b200 import metrics as PM
from dad_3dheads_b200.encoder import OUTPUT_2D_LANDMARKS, OUTPUT_3DMM_PARAMS, OUTPUT_LANDMARKS_HEATMAP
from dad_3dheads_b200.training_data import (INPUT_BBOX_KEY, TARGET_2D_FULL_LANDMARKS, TARGET_2D_LANDMARKS,
                                             TARGET_2D_LANDMARKS_PRESENCE, TARGET_3D_MODEL_VERTICES,
                                             TARGET_LANDMARKS_HEATMAP, FlameBatchBuilder, collate_records)
from oracle import ref_harness as R
from tests import metrics_model as M

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB = os.path.join(ROOT, "tests", "torchmetrics_stub")
THR = (0.05, 0.1)
GAP = 1e-4


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.int32 if a.dtype == np.float32 else np.int64)


def _same(a, b):
    return np.array_equal(_bits(np.asarray(a.cpu().numpy() if isinstance(a, torch.Tensor) else a)),
                          _bits(np.asarray(b.cpu().numpy() if isinstance(b, torch.Tensor) else b)))


# ---------------------------------------------------------------------------------------------- kernels vs the model
def _kernel_inputs(B, dev, seed):
    rng = np.random.default_rng(seed)
    V = 500
    lm_t = rng.uniform(0, 1, (B, 68, 2)).astype(np.float32)
    lm = (lm_t + rng.normal(0, 0.02, lm_t.shape)).astype(np.float32)
    pres = rng.random((B, 68)) < 0.6
    pres[: B // 3] = True                                   # all-true, mixed and all-false heads
    pres[2 * B // 3:] = False if B >= 3 else pres[2 * B // 3:]
    full_t = rng.uniform(0, 256, (B, V, 2)).astype(np.float32)
    full = (full_t + rng.normal(0, 3, full_t.shape)).astype(np.float32)
    v3_t = rng.normal(0, 0.1, (B, V, 3)).astype(np.float32)
    v3 = (v3_t + rng.normal(0, 0.005, v3_t.shape)).astype(np.float32)
    idx = np.sort(rng.choice(V, 191, replace=False)).astype(np.int32)
    box = np.stack([rng.integers(0, 300, B), rng.integers(0, 300, B), rng.integers(20, 500, B),
                    rng.integers(20, 500, B)], 1).astype(np.int32)
    d = {k: torch.from_numpy(v).to(dev) for k, v in dict(lm=lm, lm_t=lm_t, full=full, full_t=full_t, v3=v3, v3_t=v3_t,
                                                         idx=idx, box=box).items()}
    d["pres"] = torch.from_numpy(pres.astype(np.uint8)).to(dev)
    host = dict(lm=lm, lm_t=lm_t, pres=pres, full=full, full_t=full_t, v3=v3, v3_t=v3_t, idx=idx, box=box)
    return d, host


@pytest.mark.parametrize("B", [1, 3, 64, 1000])
def test_kernels_match_model_bit_for_bit(cuda_device, B):
    d, h = _kernel_inputs(B, cuda_device, B)
    box = (d["box"][:, 2], d["box"][:, 3])
    hbox = (h["box"][:, 2], h["box"][:, 3])
    groups = [PM._Group(d["lm"], d["lm_t"], presence=d["pres"], box=box, pred_scale=256.0, target_scale=256.0),
              PM._Group(d["full"], d["full_t"], index=d["idx"], box=box),
              PM._Group(d["v3"], d["v3_t"], index=d["idx"], normalize=True),
              PM._Group(d["v3"], d["v3_t"], box=box)]
    mgroups = [M.group(h["lm"], h["lm_t"], presence=h["pres"], box=hbox, pred_scale=256.0, target_scale=256.0),
               M.group(h["full"], h["full_t"], index=h["idx"], box=hbox),
               M.group(h["v3"], h["v3_t"], index=h["idx"], normalize=True),
               M.group(h["v3"], h["v3_t"], box=hbox)]
    rec = PM._keypoint_errors(groups, B, cuda_device)
    want_rec = M.keypoint_errors(mgroups)
    assert _same(rec, want_rec)
    g = torch.Generator().manual_seed(B)
    for C, H, W in ((4, 16, 16), (3, 5, 7)):
        o = torch.rand(B, C, H, W, generator=g)
        tf = torch.rand(B, C, H, W, generator=g)
        tu = (torch.rand(B, C, H, W, generator=g) * 255).to(torch.uint8)
        for t in (tf, tu):
            stats = PM._iou_stats(o.to(cuda_device), t.to(cuda_device), logits=False)
            want_stats = M.iou_stats(o.numpy().reshape(B * C, -1), t.numpy().reshape(B * C, -1))
            assert _same(stats, want_stats), (C, H, W, t.dtype)
            per_head = torch.empty(B, 4, device=cuda_device)
            epoch = (torch.full((1 + 4 * 3 + 1,), 0.5, dtype=torch.float64, device=cuda_device),
                     torch.empty(1 + 4 * 3, device=cuda_device))
            vals = PM._reduce(cuda_device, 1 + 4 * 3, stats=stats, records=rec, nme_scale=100.0, thresholds=THR,
                              per_head=per_head, epoch=epoch, weight=float(B))
            wv, wph, wep = M.reduce(stats=want_stats, records=want_rec, nme_scale=100.0, thresholds=THR,
                                    epoch=np.full(1 + 4 * 3 + 1, 0.5), weight=float(B))
            assert _same(vals, wv) and _same(per_head, wph) and _same(epoch[0], wep)
            assert _same(epoch[1], M.epoch_values(wep))
    for below in (True, False):
        vals = PM._reduce(cuda_device, 2, records=rec[:, 1:2].contiguous(), thresholds=(0.05,), below=below)
        assert _same(vals, M.reduce(records=want_rec[:, 1:2], thresholds=(0.05,), below=below)[0])


def test_record_isolation_and_permutation(cuda_device):
    B = 64
    d, h = _kernel_inputs(B, cuda_device, 7)
    box = (d["box"][:, 2], d["box"][:, 3])

    def run(d):
        groups = [PM._Group(d["lm"], d["lm_t"], presence=d["pres"], box=(d["box"][:, 2], d["box"][:, 3]),
                            pred_scale=256.0, target_scale=256.0),
                  PM._Group(d["v3"], d["v3_t"], index=d["idx"], normalize=True)]
        rec = PM._keypoint_errors(groups, B, cuda_device)
        return rec, PM._reduce(cuda_device, 6, records=rec, nme_scale=100.0, thresholds=THR)

    rec, vals = run(d)
    perm = torch.from_numpy(np.random.default_rng(0).permutation(B)).to(cuda_device)
    dp = {k: (v if k == "idx" else v[perm].contiguous()) for k, v in d.items()}
    rec_p, vals_p = run(dp)
    assert _same(rec_p, rec[perm])
    for i in (1, 2, 4, 5):                                     # the counts; the fp64 sums may differ in the last bit
        assert vals_p[i].item() == vals[i].item()
    assert abs(vals_p[0].item() - vals[0].item()) <= 1e-6 * abs(vals[0].item())
    dn = {k: v.clone() for k, v in d.items()}
    dn["lm"][5, 3, 0] = float("nan")
    dn["v3"][9, int(d["idx"][4]), 2] = float("inf")
    rec_n, vals_n = run(dn)
    keep = torch.ones(B, dtype=torch.bool)
    keep[[5, 9]] = False
    assert _same(rec_n[keep.to(cuda_device)], rec[keep.to(cuda_device)])
    assert torch.isnan(rec_n[5, 0, 0]) and not torch.isfinite(rec_n[9, 1, 0])
    assert torch.isnan(vals_n[0]) and torch.isnan(vals_n[3])


# ---------------------------------------------------------------------------------------------- the step
def _config(tmp_path):
    from tests.test_targets_model_cpu import dataset_config
    return dataset_config(str(tmp_path), "68")


def _batch(tmp_path, B, seed, dev):
    from tests.test_targets_gpu import synthetic_records
    return FlameBatchBuilder(_config(tmp_path), dev)(collate_records(synthetic_records(B, seed)))


def _outputs(batch, seed, dev):
    from oracle.flame_oracle import sample_params
    B = batch[TARGET_2D_LANDMARKS].shape[0]
    g = torch.Generator().manual_seed(seed)
    lm = batch[TARGET_2D_LANDMARKS].cpu() + 0.03 * torch.randn(B, 68, 2, generator=g)
    return {OUTPUT_3DMM_PARAMS: sample_params(B, seed).to(dev), OUTPUT_2D_LANDMARKS: lm.to(dev),
            OUTPUT_LANDMARKS_HEATMAP: (3 * torch.randn(B, 68, 64, 64, generator=g) - 2).to(dev)}


def _mixin_form(batch):
    """KeypointsDataMixin.get_input's conversions (train/mixins.py:45-51), with the reference's own uint8_to_float32."""
    from dad_3dheads_b200.training_data import INPUT_BBOX_KEY as K
    out = dict(batch)
    out[TARGET_LANDMARKS_HEATMAP] = batch[TARGET_LANDMARKS_HEATMAP].div(255.0).to(dtype=torch.float32)
    out[K] = torch.stack(batch[K]).T
    return out


def _select(batch, outputs, keep):
    k = torch.as_tensor(keep)
    b = {key: ([c[k.to(c.device)] for c in v] if key == INPUT_BBOX_KEY else v[k.to(v.device)])
         for key, v in batch.items() if isinstance(v, torch.Tensor) or key == INPUT_BBOX_KEY}
    return b, {key: v[k.to(v.device)] for key, v in outputs.items()}


def _reference_block(batch, outputs, img_size=256):
    """FlameLightningModel._step_fn's metric block (train/flame_lightning_model.py:304-357) from the reference's own
    pieces, in fp64 on the CPU: soft_iou (metrics/iou.py:15-31), keypoints_nme and percentage_of_errors_below_IOD
    (metrics/keypoints.py:19-52, KeypointsNME's weight 100), HeadMesh (head_mesh.py:28-46), normalize_to_cube
    (model/utils.py:55-68) and the face indices of config flame_indices (flame_lightning_model.py:61-63).  Returns the
    ten values and the per-head err / norm of the three keypoint groups."""
    from tests.test_metrics_model_cpu import _ref
    _ref()
    from model_training.head_mesh import HeadMesh
    from model_training.metrics.iou import soft_iou
    from model_training.metrics.keypoints import keypoints_nme, percentage_of_errors_below_IOD
    from model_training.model.flame import FLAME_CONSTS, uint8_to_float32
    from model_training.model.utils import normalize_to_cube
    face = np.load(os.path.join(R.root(), "model_training", "model", "static", "flame_indices", "face.npy"))
    B = outputs[OUTPUT_3DMM_PARAMS].shape[0]
    hm = HeadMesh(flame_config=FLAME_CONSTS, batch_size=B, image_size=img_size)
    hm.to(torch.float64)
    hm.flame.dtype = torch.float64
    t = {k: (v.cpu() if isinstance(v, torch.Tensor) else [c.cpu() for c in v]) for k, v in batch.items()
         if isinstance(v, torch.Tensor) or k == INPUT_BBOX_KEY}
    o = {k: v.detach().cpu().double() for k, v in outputs.items()}
    t[TARGET_LANDMARKS_HEATMAP] = uint8_to_float32(t[TARGET_LANDMARKS_HEATMAP]).double()         # mixins.py:50
    bbox = torch.stack(t[INPUT_BBOX_KEY]).T if isinstance(t[INPUT_BBOX_KEY], list) else t[INPUT_BBOX_KEY]  # :51
    pres = t[TARGET_2D_LANDMARKS_PRESENCE][..., None]
    out = {"heatmap_iou": soft_iou(o[OUTPUT_LANDMARKS_HEATMAP].sigmoid(), t[TARGET_LANDMARKS_HEATMAP])}       # :307-313
    groups = {}
    lm = o[OUTPUT_2D_LANDMARKS] * img_size * pres                                                         # :316
    lm_t = t[TARGET_2D_LANDMARKS].double() * pres * img_size                                              # :317-319
    groups["2d"] = (lm, lm_t, bbox)
    params = o[OUTPUT_3DMM_PARAMS].clone()
    pj = hm.reprojected_vertices(params_3dmm=params, to_2d=True)                                          # :329
    groups["reproject_2d"] = (pj[:, face], t[TARGET_2D_FULL_LANDMARKS].double()[:, face], bbox)           # :330-333
    v3 = hm.vertices_3d(params_3dmm=params, zero_rotation=True)                                           # :344
    groups["3d"] = (normalize_to_cube(v3[:, face]),
                    normalize_to_cube(t[TARGET_3D_MODEL_VERTICES].double()[:, face]), None)               # :345-351
    per_head = {}
    for name, (p, q, bb) in groups.items():
        prefix, dim = ("reproject_", "2d") if name == "reproject_2d" else ("", name)
        out[f"{prefix}nme_{dim}"] = 100 * keypoints_nme(p, q, bb)
        for thr in THR:
            out[f"{prefix}fr_{dim}_{str(thr).replace('.', '')}"] = percentage_of_errors_below_IOD(p, q, bb, threshold=thr)
        per_head[name] = keypoints_nme(p, q, bb, reduce="none")
    return out, per_head


def _clear_heads(per_head):
    ok = None
    for q in per_head.values():
        q = q.numpy()
        c = np.ones(q.shape, bool)
        for thr in THR:
            c &= np.abs(q / thr - 1) > GAP
        ok = c if ok is None else ok & c
    return ok


def test_functions_and_step_match_reference(tmp_path, cuda_device):
    batch = _batch(tmp_path, 48, 21, cuda_device)
    outputs = _outputs(batch, 22, cuda_device)
    _, per_head = _reference_block(batch, outputs)
    keep = _clear_heads(per_head)
    assert keep.sum() >= 24, keep.sum()
    batch, outputs = _select(batch, outputs, keep)
    want, _ = _reference_block(batch, outputs)
    params_before = outputs[OUTPUT_3DMM_PARAMS].clone()
    got = PM.FlameStepMetrics().step(outputs, batch, loader_name="valid")
    assert torch.equal(outputs[OUTPUT_3DMM_PARAMS], params_before)          # the caller's parameters are not modified
    assert set(got) == {f"valid/metrics/{k}" for k in want}
    for k, w in want.items():
        g, w = got[f"valid/metrics/{k}"].item(), w.item()
        assert got[f"valid/metrics/{k}"].shape == () and got[f"valid/metrics/{k}"].is_cuda
        if "fr_" in k:
            assert np.float32(g) == np.float32(w), (k, g, w)
        else:
            assert abs(g - w) <= 1e-5 * abs(w), (k, g, w)
    # translation z changes no value (the reference zeroes it in place before reading the vertices)
    o2 = dict(outputs)
    o2[OUTPUT_3DMM_PARAMS] = outputs[OUTPUT_3DMM_PARAMS].clone()
    o2[OUTPUT_3DMM_PARAMS][:, 411] = 0.0
    got2 = PM.FlameStepMetrics().step(o2, batch)
    assert all(_same(got[k], got2[k]) for k in got)
    # the functions on the same inputs
    from model_training.metrics.keypoints import keypoints_nme, percentage_of_errors_below_IOD
    from model_training.metrics.iou import soft_iou
    bbox = torch.stack(batch[INPUT_BBOX_KEY]).T
    p = outputs[OUTPUT_2D_LANDMARKS] * 256
    q = batch[TARGET_2D_LANDMARKS] * 256
    w = keypoints_nme(p.cpu().double(), q.cpu().double(), bbox.cpu()).item()
    assert abs(PM.keypoints_nme(p, q, bbox).item() - w) <= 1e-5 * abs(w)
    wh = keypoints_nme(p.cpu().double(), q.cpu().double(), bbox.cpu(), reduce="none").numpy()
    gh = PM.keypoints_nme(p, q, list(batch[INPUT_BBOX_KEY]), reduce="none")
    assert gh.shape == (p.shape[0],) and np.allclose(gh.cpu().numpy(), wh, rtol=1e-5, atol=0)
    for thr in THR:
        for below in (True, False):
            w = percentage_of_errors_below_IOD(p.cpu().double(), q.cpu().double(), bbox.cpu(), threshold=thr, below=below)
            ok = np.abs(wh / thr - 1) > GAP
            if ok.all():
                assert PM.percentage_of_errors_below_IOD(p, q, bbox, threshold=thr, below=below).item() == \
                    np.float32(w.item())
    o = torch.sigmoid(outputs[OUTPUT_LANDMARKS_HEATMAP])
    t = batch[TARGET_LANDMARKS_HEATMAP].float() / 255
    w = soft_iou(o.cpu().double(), t.cpu().double()).item()
    assert abs(PM.soft_iou(o, t).item() - w) <= 1e-5 * abs(w)


def test_step_properties(tmp_path, cuda_device):
    batch = _batch(tmp_path, 64, 5, cuda_device)
    outputs = _outputs(batch, 6, cuda_device)
    m = PM.FlameStepMetrics()
    a = m.step(outputs, batch)
    b = m.step(outputs, batch)
    c = m.step(outputs, _mixin_form(batch))                       # both batch forms give the same bits
    assert all(_same(a[k], b[k]) and _same(a[k], c[k]) for k in a)
    assert all(torch.isfinite(v) for v in a.values())
    # no host synchronisation
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m.step(outputs, batch)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    # a fixed launch count
    counts = []
    for B in (8, 256):
        bt = _batch(tmp_path, B, B, cuda_device)
        ot = _outputs(bt, B, cuda_device)
        before = _lib.launch_count()
        m.step(ot, bt)
        counts.append(_lib.launch_count() - before)
    assert counts[0] == counts[1] == m.launches_per_step, counts
    # a captured graph replays the eager values
    m.reset()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.step(outputs, batch)
    torch.cuda.current_stream().wait_stream(s)
    m.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = m.step(outputs, batch)
    graph.replay()
    torch.cuda.synchronize()
    assert all(_same(captured[k], a[k]) for k in a)


def test_epoch_values_are_batch_size_weighted(tmp_path, cuda_device):
    m = PM.FlameStepMetrics()
    sizes, per_batch = (64, 64, 17), []
    for i, B in enumerate(sizes):
        bt = _batch(tmp_path, B, 40 + i, cuda_device)
        per_batch.append(m.step(_outputs(bt, 50 + i, cuda_device), bt))
    epoch = m.compute()
    for k in epoch:
        vals = np.array([pb[k].item() for pb in per_batch], np.float64)
        want = np.float32((vals * np.array(sizes)).sum() / sum(sizes))
        assert np.float32(epoch[k].item()) == want, k
    m.reset()
    assert all(torch.isnan(v) for v in m.compute().values())
    bt = _batch(tmp_path, 5, 60, cuda_device)
    one = m.step(_outputs(bt, 61, cuda_device), bt)
    assert all(_same(m.compute()[k], one[k]) for k in one)


def test_training_chain_is_finite_and_sync_free(tmp_path, cuda_device):
    """FlameBatchBuilder -> Dad3dEncoder (synthetic weights) -> the reference's LossModule over the package losses ->
    FlameStepMetrics, at B = 8 with no host synchronisation."""
    from dad_3dheads_b200.encoder import Dad3dEncoder
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from tests.test_losses_gpu import _mine
    from tests.test_targets_gpu import synthetic_records
    B = 8
    builder = FlameBatchBuilder(_config(tmp_path), cuda_device)
    packed = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v)
              for k, v in collate_records(synthetic_records(B, 77)).items()}
    enc = Dad3dEncoder(synthetic_state_dict(0), cuda_device)
    K, module = _mine()
    metrics = PM.FlameStepMetrics()
    for sync_mode in ("default", "error"):
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode(sync_mode)
        try:
            batch = builder(packed)
            outputs = enc(batch["INPUT_IMAGE_KEY"])
            targets = _mixin_form(batch)
            total, _ = module(dict(outputs), targets, epoch=0)
            values = metrics.step(outputs, targets)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(total)
    assert all(torch.isfinite(v) for v in values.values()), values


_COMPAT_SCRIPT = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = [{root!r}, {compat!r}, {stub!r}]
from model_training.metrics import SoftIoUMetric, FailureRate, KeypointsNME
from torchmetrics import MetricCollection
d = np.load({data!r})
iou = SoftIoUMetric(compute_on_step=True)
coll = MetricCollection({{"fr_2d_005": FailureRate(compute_on_step=True, threshold=0.05, below=True),
                          "fr_2d_01": FailureRate(compute_on_step=True, threshold=0.1, below=True),
                          "nme_2d": KeypointsNME(compute_on_step=True),
                          "fr_3d_005": FailureRate(threshold=0.05, below=False)}})
steps = []
for i in range(2):
    f = lambda k: torch.from_numpy(d[f"{{k}}{{i}}"]).cuda()
    v = {{"iou": iou(f("o"), f("t")).item()}}
    out = coll(f("p"), {{"keypoints": f("q"), "bboxes": f("bb")}})
    v.update({{k: x.item() for k, x in out.items()}})
    steps.append(v)
final = {{"iou": iou.compute().item(), **{{k: x.item() for k, x in coll.compute().items()}}}}
print(json.dumps({{"steps": steps, "final": final, "states": sorted(n for n in iou._defaults)}}))
"""


def test_compat_classes_in_reference_metric_collection(tmp_path, cuda_device):
    from tests.test_metrics_model_cpu import _clear, _keypoints
    data = {}
    g = torch.Generator().manual_seed(3)
    for i, B in enumerate((12, 5)):
        data[f"o{i}"] = torch.rand(B, 4, 16, 16, generator=g).numpy()
        data[f"t{i}"] = torch.rand(B, 4, 16, 16, generator=g).numpy()
        p, q, bb = _keypoints(B, 68, 2, 30 + i)
        rec = M.keypoint_errors([M.group(p, q, box=(bb[:, 2], bb[:, 3]))])
        assert _clear(rec[:, 0, 0], rec[:, 0, 1], THR).all()
        data[f"p{i}"], data[f"q{i}"], data[f"bb{i}"] = p, q, bb
    path = str(tmp_path / "inputs.npz")
    np.savez(path, **data)
    script = _COMPAT_SCRIPT.format(root=ROOT, compat=os.path.join(ROOT, "compat"), stub=STUB, data=path)
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, cwd=str(tmp_path))
    assert res.returncode == 0, res.stderr[-3000:]
    got = json.loads(res.stdout.strip().splitlines()[-1])
    assert got["states"] == ["ious", "total"]
    # the reference's own classes, in the same collection, in fp64 on the CPU
    from tests.test_metrics_model_cpu import _ref
    iou_m, kp = _ref()
    from torchmetrics import MetricCollection
    iou = iou_m.SoftIoUMetric(compute_on_step=True)
    coll = MetricCollection({"fr_2d_005": kp.FailureRate(compute_on_step=True, threshold=0.05, below=True),
                             "fr_2d_01": kp.FailureRate(compute_on_step=True, threshold=0.1, below=True),
                             "nme_2d": kp.KeypointsNME(compute_on_step=True),
                             "fr_3d_005": kp.FailureRate(threshold=0.05, below=False)})
    want_steps = []
    for i in range(2):
        f = lambda k: torch.from_numpy(data[f"{k}{i}"]).double()
        v = {"iou": iou(f("o"), f("t")).item()}
        out = coll(f("p"), {"keypoints": f("q"), "bboxes": torch.from_numpy(data[f"bb{i}"])})
        v.update({k: x.item() for k, x in out.items()})
        want_steps.append(v)
    want_final = {"iou": iou.compute().item(), **{k: x.item() for k, x in coll.compute().items()}}
    for g_, w_ in list(zip(got["steps"], want_steps)) + [(got["final"], want_final)]:
        for k, w in w_.items():
            if "fr_" in k and g_ is not got["final"]:
                assert np.float32(g_[k]) == np.float32(w), (k, g_[k], w)
            else:
                assert abs(g_[k] - w) <= 1e-5 * abs(w), (k, g_[k], w)
