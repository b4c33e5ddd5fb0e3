"""-m gpu: ping-pong launches of the tile engine.  The plan matches the CPU restatement (tests/pingpong_model.py) step for
step; the steps that cover each ping-pong schedule and launch kind run alone against tests/engine_model.py bit for bit;
and the whole predictor, graphed and streamed, is bit-identical to the eager call."""
import numpy as np
import pytest
import torch

from tests import pingpong_model as pm
from tests.test_encoder_steps_gpu import _designed_encoder, check_conv_steps, folded  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

FIELDS = ("tw", "th", "tn", "tiles_w", "tiles_h", "tiles_n", "block_n", "n_tiles", "stages", "halo", "res_kb", "pingpong",
          "grid", "cta_tiles_min", "cta_tiles_max")


def _covering(plan):
    """Indices of ping-pong steps that together cover: a CTA with one tile, an odd tile count above one, and every launch
    kind (tensor-core stem, 1x1 stride 2, second source, identity residual on K, up2, parity, gate, plain 1x1)."""
    want = {
        "one_tile": lambda s: s["cta_tiles_min"] == 1,
        "odd": lambda s: any(n % 2 == 1 and n > 1 for n in (s["cta_tiles_min"], s["cta_tiles_max"])),
        "stem": lambda s: s["stem"] == 1,
        "stride2": lambda s: s["R"] == 1 and s["stride"] == 2 and not s["parity"],
        "src2": lambda s: s["res_mode"] == 4,
        "identity": lambda s: s["res_mode"] == 1 and s["res_kb"] > 0 and not s["parity"],
        "up2": lambda s: s["up2"] == 1,
        "gate": lambda s: s["res_mode"] == 2,
        "plain1x1": lambda s: s["R"] == 1 and s["res_mode"] == 0 and not s["up2"] and s["stride"] == 1,
    }
    if any(s.get("parity") for s in plan["steps"]):
        want["parity"] = lambda s: s["parity"] > 0
    picked, missing = set(), []
    for what, pred in want.items():
        hits = [i for i, s in enumerate(plan["steps"]) if s["kind"] == "conv" and s["pingpong"] and pred(s)]
        if not hits:
            missing.append(what)
        else:
            picked.add(hits[0])
    return picked, missing


@pytest.mark.parametrize("mode", ["fp16x2", "fp32", "bf16"])
@pytest.mark.parametrize("B", [2, 5, 64, 129])
def test_plan_matches_restatement(folded, cuda_device, mode, B):  # noqa: F811
    enc, _, _ = _designed_encoder(folded, mode, cuda_device)
    enc.forward_raw(torch.randn(B, 3, 256, 256, device=cuda_device), want_heatmap=True)
    plan = enc.describe_plan()
    steps = [s for s in plan["steps"] if s["kind"] == "conv"]
    model = pm.network(B)
    assert [s["layer"] for s in steps] == [ln.layer for ln in model]
    P = pm.MODES[mode]
    for s, ln in zip(steps, model):
        g = pm.geometry(ln, P)
        got = {k: s[k] for k in FIELDS}
        assert got == {k: g[k] for k in FIELDS}, (s["layer"], got, g)
    pp = {s["layer"] for s in steps if s["pingpong"]}
    if P == 1:                                                    # one product per k-block: cooperative throughout
        assert not pp
        return
    assert "heat" not in pp and "mlp2" not in pp
    assert {"stem", "s1u1c1", "s1u1c3", "s2u1c1", "b0_p3td", "b0_p3td_u", "fusion", "mlp1"} <= pp
    assert not {"lat6", "s4u1c2"} & pp                            # more than 32 k-blocks per tile
    if P == 2:
        assert not {f"s2u{u}c2" for u in range(1, 5)} & pp       # halo layers stay cooperative
    _, missing = _covering(plan)
    assert missing == (["odd"] if B == 2 else []), missing       # at batch 2 no CTA has more than two tiles


@pytest.mark.parametrize("env,mode,B", [({}, "fp16x2", 64), ({}, "fp32", 5), ({}, "bf16x2", 129),
                                        ({"DAD3D_TD_PARITY": "1"}, "fp16x2", 5)])
def test_pingpong_steps_match_model(folded, cuda_device, monkeypatch, env, mode, B):  # noqa: F811
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    enc, weights, kws = _designed_encoder(folded, mode, cuda_device)
    enc.set_debug(True)
    enc.forward_raw(torch.randn(B, 3, 256, 256, device=cuda_device), want_heatmap=True)
    plan = enc.describe_plan()
    picked, missing = _covering(plan)
    assert not missing, missing
    # check_conv_steps offers the conv steps to `only` once each, in plan order
    conv_idx = [i for i, s in enumerate(plan["steps"]) if s["kind"] == "conv"]
    sel = {conv_idx.index(i) for i in picked}
    seen = iter(range(len(conv_idx)))
    _, bad = check_conv_steps(enc, weights, kws, mode, B, cuda_device, only=lambda st: next(seen) in sel)
    assert not bad, bad


def _outputs_equal(a, b):
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, torch.Tensor) and not torch.equal(x.cpu(), y.cpu()):
            return k
    return None


@pytest.mark.parametrize("B", [64, 512])
def test_graphed_and_streamed_match_eager(cuda_device, B):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    pred = FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0), precision="fp16x2", cuda_id=cuda_device.index or 0)
    x = torch.randint(0, 256, (B, 256, 256, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(B))
    eager = pred.predict_batch(x.to(cuda_device), landmark_subset="445")
    eager = {k: v.clone() for k, v in eager.items() if isinstance(v, torch.Tensor)}
    graphed = pred.predict_batch_graphed(x, landmark_subset="445")
    assert _outputs_equal(eager, {k: graphed[k] for k in eager}) is None
    keys = ("3dmm_params", "points", "3d_vertices", "landmarks_445")
    st = pred.open_stream(tuple(x.shape), keys=keys)
    st.submit(x.pin_memory())
    res = st.collect()
    for k in keys:
        assert np.array_equal(res[k].numpy(), eager[k].cpu().numpy()), k
