"""-m gpu: the regression-head kernels (csrc/heads.cu) against the exact model (tests/heads_model.py), bit for bit through the
C ABI with every output between NaN-payload guard bands; Dad3dEncoder.features; dropout; and the fine-tuning step over a
frozen backbone (determinism, no host synchronisation, fixed launches, graph capture, training progress, checkpoints)."""
import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from dad_3dheads_b200.encoder import OUTPUT_2D_LANDMARKS, OUTPUT_3DMM_PARAMS, Dad3dEncoder
from dad_3dheads_b200.encoder_weights import synthetic_state_dict
from dad_3dheads_b200.heads import FlameHeads, FrozenBackboneRegression
from tests import heads_model as H
from tests.test_losses_exact_gpu import Guarded, _dev_input

pytestmark = pytest.mark.gpu
f32 = np.float32


def _ulp_close(a, b, ulps):
    a, b = np.asarray(a, f32), np.asarray(b, np.float64)
    return np.abs(a.astype(np.float64) - b) <= ulps * np.spacing(np.abs(b).astype(f32)).astype(np.float64)


def _inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.rand(B, 2048, generator=g).numpy()
    w1 = (torch.randn(1536, 2048, generator=g) * 0.03).numpy()
    b1 = (torch.randn(1536, generator=g) * 0.1).numpy()
    w2 = (torch.randn(549, 512, generator=g) * 0.05).numpy()
    b2 = (torch.randn(549, generator=g) * 0.1).numpy()
    b2[:40] = np.where(np.arange(40) % 2, 40.0, -40.0)          # designed shape logits where tanh is exactly +-1
    dparams = torch.randn(B, 413, generator=g).numpy()
    dparams[:, 7] = 0.0
    dlms = torch.randn(B, 136, generator=g).numpy()
    return f, w1, b1, w2, b2, dparams, dlms


@pytest.mark.parametrize("B,train", [(1, True), (3, True), (64, True), (65, True), (257, True), (3, False), (65, False)])
def test_kernels_match_model(B, train, cuda_device):
    lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream
    f, w1, b1, w2, b2, dparams, dlms = _inputs(B, 100 + B)
    p, seed, ctr0 = 0.3, 0xC0FFEE123, 7
    dev = [_dev_input(a, (i * 3) % 8, cuda_device) for i, a in enumerate((f, w1, b1, w2, b2, dparams, dlms))]
    counter = torch.tensor([ctr0], dtype=torch.int64, device=cuda_device)
    shapes = dict(params=B * 413, lms=B * 136, h=B * 1536, d=B * 1536, mask=B * 48, y=B * 403, obits=B * 18)
    out = {k: Guarded(n, (i * 5) % 8, cuda_device) for i, (k, n) in enumerate(shapes.items())}
    ws = torch.empty(int(lib.dad3d_heads_workspace_bytes(B)), dtype=torch.uint8, device=cuda_device)
    _lib.check(lib.dad3d_heads_forward(dev[0].data_ptr(), B, *(t.data_ptr() for t in dev[1:5]), 3.0, int(train), p, seed,
                                       counter.data_ptr(), *(o.ptr() for o in out.values()), ws.data_ptr(), ws.numel(), st),
               "forward")
    got = {k: o.check() for k, o in out.items()}
    m = H.forward(f, w1, b1, w2, b2, train, p, seed, ctr0)
    assert int(counter.item()) == ctr0 + (1 if train else 0)
    bits = lambda a: a.view(np.int32)      # noqa: E731
    for k in ("h", "d"):
        assert (bits(got[k]) == bits(m[k].reshape(-1))).all(), k
    assert (got["mask"].view(np.uint32) == m["mask"].reshape(-1)).all()
    assert (got["obits"].view(np.uint32) == m["obits"].reshape(-1)).all()
    y = got["y"].reshape(B, 403)
    assert _ulp_close(y, np.tanh(m["o"][:, :403].astype(np.float64)), 2).all()
    assert (y[:, :40] == np.where(np.arange(40) % 2, 1.0, -1.0)).all()
    assert (bits(got["params"]) == bits(H.params(y, m["o"]).reshape(-1))).all()
    assert (bits(got["lms"]) == bits(m["landmarks"].reshape(-1))).all()

    saved = [_dev_input(got[k], 0, cuda_device) for k in ("h", "d", "mask", "y", "obits")]
    gshapes = dict(dw1=1536 * 2048, db1=1536, dw2=549 * 512, db2=549)
    gout = {k: Guarded(n, (i * 3 + 1) % 8, cuda_device) for i, (k, n) in enumerate(gshapes.items())}
    _lib.check(lib.dad3d_heads_backward(dev[5].data_ptr(), dev[6].data_ptr(), dev[0].data_ptr(), B, dev[3].data_ptr(), 3.0,
                                        int(train), p, *(t.data_ptr() for t in saved), *(o.ptr() for o in gout.values()),
                                        ws.data_ptr(), ws.numel(), st), "backward")
    want = H.backward(dparams, dlms, f, w2, m["h"], m["d"], m["mask"], y, m["obits"], train, p)
    for k, o in gout.items():
        assert (bits(o.check()) == bits(want[k].reshape(-1))).all(), k


@pytest.fixture(scope="module")
def sd():
    return synthetic_state_dict(0)


def _images(B, seed):
    return torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(seed)).cuda()


def test_features_are_the_pool(sd, cuda_device):
    from oracle.encoder_oracle import flame_regression_forward
    x = _images(3, 5)
    enc = Dad3dEncoder(sd, cuda_device, precision="fp32")
    enc.set_debug(True)
    want_params, want_lms, want_heat = enc.forward_raw(x, want_heatmap=True)
    feats, heat = enc.features(x, want_heatmap=True)
    gap = enc.read_activation("gap").reshape(3, 2048)
    assert torch.equal(feats, gap)
    assert torch.equal(heat, want_heat)
    params, lms, heat2 = enc.forward_raw(x, want_heatmap=True)
    assert torch.equal(params, want_params) and torch.equal(lms, want_lms) and torch.equal(heat2, want_heat)
    _, inter = flame_regression_forward(x.cpu().double(), {k: v.double() for k, v in sd.items()},
                                        return_intermediates=True)
    ref = inter["stage4"].mean(dim=(2, 3))
    err = ((feats.cpu().double() - ref).norm() / ref.norm()).item()
    assert err < 1e-4, err


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_eval_heads_agree_with_encoder(sd, precision, cuda_device):
    x = _images(4, 6)
    enc = Dad3dEncoder(sd, cuda_device, precision=precision)
    heads = FlameHeads.from_state_dict(sd).cuda().eval()
    feats, _ = enc.features(x, want_heatmap=False)
    with torch.no_grad():
        params, lms = heads(feats)
    want = enc(x)
    for got, w in ((params, want[OUTPUT_3DMM_PARAMS]), (lms, want[OUTPUT_2D_LANDMARKS])):
        assert ((got - w).norm() / w.norm()).item() < 1e-4


def _module_mask(heads, f):
    """the keep bits [B, 48] the module's own training forward saved for its backward"""
    params, _ = heads(f)
    return params.grad_fn.saved_tensors[4].clone()


def test_dropout_statistics_and_streams(cuda_device):
    heads = FlameHeads(seed=3).cuda().train()
    f = torch.rand(700, 2048, generator=torch.Generator().manual_seed(8)).cuda()
    m0, m1 = _module_mask(heads, f), _module_mask(heads, f)
    assert heads.counter.item() == 2
    keep = H.unpack_bits(m0.cpu().numpy().view(np.uint32), 1536)
    assert keep.size >= 10 ** 6 and abs(keep.mean() - 0.7) <= 5 * (0.21 / keep.size) ** 0.5
    assert not torch.equal(m0, m1)                                        # consecutive steps draw fresh masks
    for c, m in ((0, m0), (1, m1)):                                       # the module's masks are the Philox model's
        assert (m.cpu().numpy().view(np.uint32) == H.pack_bits(H.keep_mask(700, 3, c, 0.3))).all()
    heads.counter.zero_()
    assert torch.equal(_module_mask(heads, f[:3]), m0[:3])               # equal (seed, counter): equal mask


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_heads_run_on_their_tensors_device():
    """Heads on cuda:1 while cuda:0 is current launch on cuda:1 and give cuda:0's bits."""
    torch.cuda.set_device(0)
    f = torch.rand(5, 2048, generator=torch.Generator().manual_seed(2))
    sd = synthetic_state_dict(1)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        heads = FlameHeads.from_state_dict(sd, seed=4).to(dev).train()
        params, lms = heads(f.to(dev))
        (params.sum() + lms.sum()).backward()
        outs.append([t.detach().cpu() for t in (params, lms, heads.w1.grad, heads.b1.grad, heads.w2.grad, heads.b2.grad)])
    assert torch.cuda.current_device() == 0
    assert all(torch.equal(a, b) for a, b in zip(*outs))


# ---- the fine-tuning step ------------------------------------------------------------------------------------------------
def _setup(tmp_path, B, cuda_device, sd):
    from tests.test_losses_gpu import _mine
    from tests.test_metrics_gpu import _batch, _mixin_form
    batch = _batch(tmp_path, B, 41, cuda_device)
    enc = Dad3dEncoder(sd, cuda_device, precision="fp16x2")
    heads = FlameHeads.from_state_dict(sd, seed=5).cuda().train()
    model = FrozenBackboneRegression(enc, heads)
    K, module = _mine()
    return batch["INPUT_IMAGE_KEY"], _mixin_form(batch), model, module


def _step(model, module, opt, images, targets):
    total, _ = module(model(images), targets, epoch=0)
    opt.zero_grad(set_to_none=False)
    total.backward()
    opt.step()
    return total.detach()


def test_step_deterministic_sync_free_fixed_launches(tmp_path, sd, cuda_device):
    runs = []
    for B in (8, 8, 3):
        images, targets, model, module = _setup(tmp_path, B, cuda_device, sd)
        assert [n for n, _ in model.named_parameters()] == ["heads.w1", "heads.b1", "heads.w2", "heads.b2"]
        opt = torch.optim.Adam(model.parameters())
        _step(model, module, opt, images, targets)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            l0 = _lib.launch_count()
            total = _step(model, module, opt, images, targets)
            launches = _lib.launch_count() - l0
        finally:
            torch.cuda.set_sync_debug_mode("default")
        runs.append((B, total.cpu(), [p.detach().cpu() for p in model.parameters()], launches, model.heads.counter.item()))
    (_, t0, p0, n0, c0), (_, t1, p1, n1, c1), (_, _, _, n2, _) = runs
    assert torch.equal(t0, t1) and all(torch.equal(a, b) for a, b in zip(p0, p1))
    assert n0 == n1 == n2 and c0 == c1 == 2


def test_captured_step_replays_to_eager(tmp_path, sd, cuda_device):
    images, targets, model, module = _setup(tmp_path, 8, cuda_device, sd)
    eager = FrozenBackboneRegression(model.encoder, FlameHeads.from_state_dict(sd, seed=5).cuda().train())
    opt_e = torch.optim.Adam(eager.parameters(), capturable=True)
    opt = torch.optim.Adam(model.parameters(), capturable=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):                            # warm-up: the optimizer state and every workspace
            _step(model, module, opt, images, targets)
            _step(eager, module, opt_e, images, targets)
    torch.cuda.current_stream().wait_stream(s)
    saved = {}
    stash = lambda name: lambda mod, inp, out: saved.__setitem__(name, out[0].grad_fn.saved_tensors[4])  # noqa: E731
    model.heads.register_forward_hook(stash("graph"))
    eager.heads.register_forward_hook(stash("eager"))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        total = _step(model, module, opt, images, targets)
    counters, masks = [], []
    for _ in range(3):
        g.replay()
        want = _step(eager, module, opt_e, images, targets)
        assert torch.equal(total, want)
        assert torch.equal(saved["graph"], saved["eager"])                # the replay drew the eager step's mask
        counters.append(model.heads.counter.item())
        masks.append(saved["graph"].clone())
    assert counters == [3, 4, 5] and eager.heads.counter.item() == 5
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])
    for a, b in zip(model.parameters(), eager.parameters()):
        assert torch.equal(a, b)


def test_forty_steps_lower_the_objective_and_export(tmp_path, sd, cuda_device):
    from dad_3dheads_b200.metrics import FlameStepMetrics
    images, targets, model, module = _setup(tmp_path, 8, cuda_device, sd)
    opt = torch.optim.Adam(model.parameters())
    losses = [_step(model, module, opt, images, targets) for _ in range(40)]
    first, last = losses[0].item(), losses[-1].item()
    assert np.isfinite(last) and last < first, (first, last)
    model.heads.eval()
    with torch.no_grad():
        out = model(images)
    trained = dict(sd)
    trained.update(model.heads.reference_state_dict())
    enc = Dad3dEncoder(trained, cuda_device, precision="fp16x2")
    want = enc(images)
    for k in (OUTPUT_3DMM_PARAMS, OUTPUT_2D_LANDMARKS):
        assert ((out[k] - want[k]).norm() / want[k].norm()).item() < 1e-4, k
    values = FlameStepMetrics().step(out, targets)
    assert all(torch.isfinite(v) for v in values.values())


def test_invalid_inputs_raise(cuda_device):
    heads = FlameHeads().cuda()
    with pytest.raises(TypeError):
        heads(torch.zeros(2, 2048, device=cuda_device, dtype=torch.float16))
    with pytest.raises(ValueError):
        heads(torch.zeros(2, 1024, device=cuda_device))
    with pytest.raises(ValueError):
        heads(torch.zeros(0, 2048, device=cuda_device))
