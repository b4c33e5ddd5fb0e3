"""-m gpu: the CUDA encoder (through the C ABI) against the CPU oracle's FlameRegression.forward, same seeded weights/inputs.

Tolerances (norm-wise relative L2 vs the fp64 oracle; north_star contract: 1e-4 relative to the fp32 reference path):
  "fp32"   (bf16 three-way split, 6 products, two-class accumulation)   < 3e-5   -- strict-operand parity mode
  "fp16x2" (fp16 hi/lo, 3 products, per-channel scaled weights)          < 5e-5   -- bench default, also under the 1e-4 contract
  "bf16x2" (bf16 hi/lo, 3 products)                                      < 1e-4
  "bf16"   (plain bf16 operands, throughput mode, BASELINE config 3)     < 2e-2   (NOT under the 1e-4 banner)
"""
import pytest
import torch

from dad_3dheads_b200.encoder_weights import synthetic_state_dict
from oracle.encoder_oracle import (OUTPUT_2D_LANDMARKS, OUTPUT_3DMM_PARAMS, OUTPUT_LANDMARKS_HEATMAP,
                                   flame_regression_forward)

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(scope="module")
def sd():
    return synthetic_state_dict(0)


@pytest.fixture(scope="module")
def ref5(sd):
    x = torch.randn(5, 3, 256, 256, generator=torch.Generator().manual_seed(42))
    with torch.no_grad():
        out = flame_regression_forward(x.double(), {k: v.double() for k, v in sd.items()})
    return x, out


@pytest.mark.parametrize("precision,tol", [("fp32", 3e-5), ("fp16x2", 5e-5), ("bf16x2", 1e-4), ("fp16", 5e-3), ("bf16", 2e-2)])
def test_encoder_matches_oracle(sd, ref5, cuda_device, precision, tol):
    from dad_3dheads_b200.encoder import Dad3dEncoder
    x, ref = ref5
    enc = Dad3dEncoder(sd, cuda_device, precision=precision)
    out = enc(x.to(cuda_device))
    assert out[OUTPUT_3DMM_PARAMS].shape == (5, 413) and out[OUTPUT_2D_LANDMARKS].shape == (5, 68, 2)
    assert out[OUTPUT_LANDMARKS_HEATMAP].shape == (5, 68, 64, 64)
    errs = {k: _rel(out[k], ref[k]) for k in ref}
    assert all(e < tol for e in errs.values()), errs


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_elementwise_contract(sd, ref5, cuda_device, precision):
    """|err| <= 1e-4 * |ref| + 1e-4 on every one of the 413 params (values span +-3), vs the fp32 oracle itself."""
    from dad_3dheads_b200.encoder import Dad3dEncoder
    x, _ = ref5
    with torch.no_grad():
        ref32 = flame_regression_forward(x, sd)
    out = Dad3dEncoder(sd, cuda_device, precision=precision)(x.to(cuda_device))
    p, r = out[OUTPUT_3DMM_PARAMS].cpu(), ref32[OUTPUT_3DMM_PARAMS]
    assert ((p - r).abs() <= 1e-4 * r.abs() + 1e-4).all(), (p - r).abs().max()


def test_per_layer_activations(sd, cuda_device):
    """Every named activation against the CPU executor of the folded graph: localises a regression to one kernel."""
    from dad_3dheads_b200.encoder import Dad3dEncoder, fold_state_dict
    from tests.folded_ref import run_folded
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(7))
    layers, fw = fold_state_dict(sd)
    with torch.no_grad():
        ref = run_folded(x, layers, fw)
    enc = Dad3dEncoder(sd, cuda_device, precision="fp32")
    enc.set_debug(True)
    enc.forward_raw(x.to(cuda_device))
    bad = {}
    for name in ["stem"] + [n for n, _, _ in layers if n != "stem"] + ["cat", "gap"]:
        a = enc.read_activation(name)
        r = ref[name]
        if name in ("gap", "mlp1", "mlp2"):
            got, want = a.reshape(a.shape[2], a.shape[3])[:, : r.shape[1]], r.flatten(1)
        else:
            got, want = a[..., : r.shape[1]].permute(0, 3, 1, 2), r
            pad = a[..., r.shape[1]:]
            if pad.numel() and name not in ("cat",):
                assert pad.abs().max().item() == 0.0, f"{name}: padded channels must stay zero"
        e = _rel(got, want)
        if e > 3e-5:
            bad[name] = e
    assert not bad, bad


def test_batch_independence_and_determinism(sd, cuda_device):
    """Eval-mode network: an image's outputs must not depend on its batch (bit-exact), nor on the run."""
    from dad_3dheads_b200.encoder import Dad3dEncoder
    enc = Dad3dEncoder(sd, cuda_device, precision="fp32", want_heatmap=False)
    x = torch.randn(7, 3, 256, 256, generator=torch.Generator().manual_seed(9)).to(cuda_device)
    p7, l7, _ = enc.forward_raw(x)
    p7b, _, _ = enc.forward_raw(x)
    assert torch.equal(p7, p7b)
    p1, l1, _ = enc.forward_raw(x[3:4])
    assert torch.equal(p7[3:4], p1) and torch.equal(l7[3:4], l1)
    p3, _, _ = enc.forward_raw(x[4:7])
    assert torch.equal(p7[4:7], p3)


def test_batch_64_matches_oracle_subset(sd, cuda_device):
    """BASELINE configs[1] size: batch 64; oracle checked on a subset (CPU time), the rest by batch independence."""
    from dad_3dheads_b200.encoder import Dad3dEncoder
    x = torch.randn(64, 3, 256, 256, generator=torch.Generator().manual_seed(64))
    enc = Dad3dEncoder(sd, cuda_device, precision="fp32", want_heatmap=False)
    p, l, _ = enc.forward_raw(x.to(cuda_device))
    sel = [0, 31, 63]
    with torch.no_grad():
        ref = flame_regression_forward(x[sel].double(), {k: v.double() for k, v in sd.items()})
    assert _rel(p[sel], ref[OUTPUT_3DMM_PARAMS]) < 3e-5 and _rel(l[sel], ref[OUTPUT_2D_LANDMARKS]) < 3e-5
    assert torch.isfinite(p).all()


@pytest.mark.parametrize("precision,tol", [("fp16x2", 5e-5), ("bf16", 2e-2)])
@pytest.mark.parametrize("halo", ["1", "0"])
def test_halo_and_per_tap_paths_match_oracle(sd, ref5, cuda_device, monkeypatch, precision, tol, halo):
    """Default (DAD3D_HALO unset / 1): the 3x3 stride-1 layers run on 8x16-pixel tiles whose nine taps read one shared halo
    patch through shifted wgmma descriptors (k order: channel block outer, tap inner); DAD3D_HALO=0: one TMA box per tap
    (tap outer).  Both against the oracle, with the 3x3 layers checked one by one."""
    from dad_3dheads_b200.encoder import Dad3dEncoder, fold_state_dict
    from tests.folded_ref import run_folded
    monkeypatch.setenv("DAD3D_HALO", halo)
    x, ref = ref5
    enc = Dad3dEncoder(sd, cuda_device, precision=precision)
    out = enc(x.to(cuda_device))
    errs = {k: _rel(out[k], ref[k]) for k in ref}
    if precision == "fp16x2":                      # localise a failure to the layer
        x2 = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(7))
        layers, fw = fold_state_dict(sd)
        with torch.no_grad():
            lref = run_folded(x2, layers, fw)
        enc.set_debug(True)
        enc.forward_raw(x2.to(cuda_device))
        bad = {}
        three = sorted({s["layer"] for s in enc.describe_plan()["steps"] if s["kind"] == "conv" and s["R"] == 3})
        assert len(three) >= 17, three                 # the sixteen ResNet 3x3 layers of stages 1-4 and the heat-map head
        for name in three:
            a = enc.read_activation(name)
            r = lref[name]
            e = _rel(a[..., : r.shape[1]].permute(0, 3, 1, 2), r)
            if e > 5e-5:
                bad[name] = e
        assert not bad, bad
    assert all(e < tol for e in errs.values()), errs


def test_td_parity_launches_match(sd, cuda_device, monkeypatch):
    """DAD3D_TD_PARITY=1: P3 / P4 top-down nodes as four launches, one per pixel parity (strided A view, half-resolution
    residual, parity store); every activation against the CPU executor of the folded graph."""
    from dad_3dheads_b200.encoder import Dad3dEncoder, fold_state_dict
    from tests.folded_ref import run_folded
    monkeypatch.setenv("DAD3D_TD_PARITY", "1")
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(11))
    layers, fw = fold_state_dict(sd)
    with torch.no_grad():
        ref = run_folded(x, layers, fw)
    enc = Dad3dEncoder(sd, cuda_device, precision="fp16x2")
    enc.set_debug(True)
    enc.forward_raw(x.to(cuda_device))
    bad = {}
    for name in [n for n, _, _ in layers if n.startswith("b0_") or n.startswith("b1_")]:
        a = enc.read_activation(name)
        r = ref[name]
        e = _rel(a[..., : r.shape[1]].permute(0, 3, 1, 2), r)
        if e > 5e-5:
            bad[name] = e
    assert not bad, bad


def test_encoder_reference_fixture(sd, cuda_device):
    """tests/golden/reference_encoder.npz: outputs of the UNMODIFIED reference FlameRegression.forward
    (tools/make_reference_golden.py; weight seed 0, image seed 777), fp64 run as the yard-stick."""
    import os
    import numpy as np
    from dad_3dheads_b200.encoder import Dad3dEncoder
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_encoder.npz"))
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(int(z["image_seed"])))
    for mode in ("fp32", "fp16x2"):
        out = Dad3dEncoder(sd, cuda_device, precision=mode)(x.to(cuda_device))
        assert _rel(out[OUTPUT_3DMM_PARAMS], torch.from_numpy(z["params_f64"])) < 3e-5, mode
        assert _rel(out[OUTPUT_2D_LANDMARKS], torch.from_numpy(z["landmarks_f64"])) < 3e-5, mode
        assert _rel(out[OUTPUT_LANDMARKS_HEATMAP].sum(dim=(2, 3)), torch.from_numpy(z["heatmap_sum_f64"])) < 3e-5, mode
        assert _rel(out[OUTPUT_LANDMARKS_HEATMAP][:, :, :4, :4], torch.from_numpy(z["heatmap_corner_f64"])) < 1e-4, mode


def test_create_rejects_invalid_weights(sd, cuda_device):
    """dad3d_encoder_create refuses malformed weights with DAD3D_ERR_INVALID (-1) and says why: a record with a null or
    non-positive field, a stem that is not 7x7 3->64, a layer the graph needs but no record carries, pieces or operand
    format out of range."""
    import ctypes as C
    import numpy as np
    from dad_3dheads_b200 import _lib
    from dad_3dheads_b200.encoder import Dad3dEncoder, _ConvWeights, fold_state_dict
    layers, fw = fold_state_dict(sd)
    layers = [(n, np.ascontiguousarray(w, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32))
              for n, w, b in layers]

    def rejected(ls):
        with pytest.raises(_lib.Dad3dError) as e:
            Dad3dEncoder.from_folded(ls, fw, cuda_device, precision="fp16x2")
        assert "(rc=-1)" in str(e.value), str(e.value)
        return str(e.value)

    stem = next(i for i, (n, _, _) in enumerate(layers) if n == "stem")
    assert "missing layer weights: lat4" in rejected([l for l in layers if l[0] != "lat4"])
    assert "missing layer weights: b1_p3td_u" in rejected([l for l in layers if l[0] != "b1_p3td_u"])
    assert "missing layer weights: stem" in rejected([l for l in layers if l[0] != "stem"])
    bad_stem = list(layers)
    bad_stem[stem] = ("stem", np.zeros((64, 5, 5, 3), np.float32), layers[stem][2])
    assert "stem must be 7x7 3->64" in rejected(bad_stem)
    bad_stem[stem] = ("stem", np.zeros((64, 7, 7, 4), np.float32), layers[stem][2])
    assert "stem must be 7x7 3->64" in rejected(bad_stem)
    empty = list(layers)
    empty.insert(3, ("lat4", np.zeros((0, 1, 1, 512), np.float32), np.zeros(0, np.float32)))
    assert "invalid layer record 3" in rejected(empty)

    lib = _lib.load()
    name, w, b = layers[stem]
    rec = (_ConvWeights * 1)()
    rec[0].name, rec[0].weight_h, rec[0].bias_h = name.encode(), w.ctypes.data, b.ctypes.data
    rec[0].cout, rec[0].R, rec[0].S, rec[0].cin = w.shape
    fwc = np.ascontiguousarray(fw, dtype=np.float32)
    for pieces, fmt, msg in [(0, 0, "pieces must be"), (4, 0, "pieces must be"), (3, 1, "operand_format must be"),
                             (2, 2, "operand_format must be"), (1, -1, "operand_format must be")]:
        h = C.c_void_p()
        assert lib.dad3d_encoder_create(C.byref(h), rec, 1, fwc.ctypes.data, pieces, fmt, cuda_device.index) == -1
        assert not h.value and msg in lib.dad3d_last_error().decode(), (pieces, fmt)
    null = (_ConvWeights * 1)()
    h = C.c_void_p()
    assert lib.dad3d_encoder_create(C.byref(h), null, 1, fwc.ctypes.data, 1, 0, cuda_device.index) == -1
    assert "invalid layer record 0" in lib.dad3d_last_error().decode()
