"""-m "not gpu": the exact model of csrc/heads.cu (tests/heads_model.py): Philox against Random123's known answers, the
model's forward and gradients against fp64 autograd of the reference's ClassificationHead, the torch arithmetic the kernels
restate, and the packed weights' round trip through the reference keys."""
import numpy as np
import pytest
import torch

from oracle import ref_harness as R
from tests import heads_model as H
from tests.metrics_model import fma32

f32 = np.float32


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = H.philox4x32_10([np.array([c]) for c in ctr], [np.array([k]) for k in key])
    assert tuple(int(x[0]) for x in got) == want


def test_keep_fraction_and_streams():
    m = H.keep_mask(700, 11, 5, 0.3)
    n = m.size
    assert abs(m.mean() - 0.7) <= 5 * (0.21 / n) ** 0.5
    assert (H.keep_mask(3, 11, 5, 0.3) == m[:3]).all()
    assert (H.keep_mask(3, 11, 6, 0.3) != m[:3]).any() and (H.keep_mask(3, 12, 5, 0.3) != m[:3]).any()
    assert (H.unpack_bits(H.pack_bits(m[:5]), 1536) == m[:5]).all()


def test_fast_fma_matches_fma32():
    g = np.random.default_rng(0)
    a, b, c = (g.standard_normal(200000).astype(f32) * f32(s) for s in (1, 3e-3, 1))
    got = H._fma_acc(a.astype(np.float64) * b.astype(np.float64), c.astype(np.float64)).astype(f32)
    assert (got.view(np.int32) == fma32(a, b, c).view(np.int32)).all()


def test_torch_dropout_and_tanh_arithmetic():
    """Kept values are h * fp32(1 / (1 - p)) with the reciprocal in fp64; tanh_backward is g * fma(-y, y, 1)."""
    torch.manual_seed(0)
    h = torch.rand(400000) * 10 + 1e-3
    for p in (0.3, 0.1, 0.77):
        out = torch.nn.functional.dropout(h, p, True)
        kept = out != 0
        want = h.numpy() * H.dropout_scale(True, p)
        assert (out.numpy()[kept.numpy()] == want[kept.numpy()]).all(), p
    g = torch.randn(400000)
    y = torch.tanh(torch.randn(400000) * 2)
    got = torch.ops.aten.tanh_backward(g, y).numpy()
    gn, yn = g.numpy(), y.numpy()
    assert (got.view(np.int32) == (gn * fma32(-yn, yn, np.ones_like(yn))).view(np.int32)).all()


def test_keep_test_probability_against_torch_dropout():
    """torch's CPU dropout draws its keep bits from another generator, so the bits cannot be pinned; the keep test's
    probability can: over every 24-bit draw, fp32(k) * 2^-24 < fp32(1 - p) holds for exactly ceil(fp32(1 - p) * 2^24)
    of 2^24, within 2^-24 of 1 - p, and torch's CPU keep fraction lies within 5 sigma of it."""
    k = np.arange(1 << 24, dtype=np.uint32)
    u = k.astype(f32) * f32(2.0 ** -24)
    torch.manual_seed(1)
    ones = torch.ones(1 << 22)
    for p in (0.3, 0.1, 0.5, 0.77):
        q = H.keep_prob(p)
        n = int((u < q).sum())
        assert n == int(np.ceil(np.float64(q) * 2 ** 24))
        prob = n / 2 ** 24
        assert abs(prob - (1 - p)) <= 2 ** -24
        frac = (torch.nn.functional.dropout(ones, p, True) != 0).double().mean().item()
        assert abs(frac - prob) <= 5 * (prob * (1 - prob) / ones.numel()) ** 0.5, p


def _weights(seed, scale2=1.0):
    g = torch.Generator().manual_seed(seed)
    w1 = (torch.randn(1536, 2048, generator=g) * 0.03).numpy()
    b1 = (torch.randn(1536, generator=g) * 0.1).numpy()
    w2 = (torch.randn(549, 512, generator=g) * 0.05 * scale2).numpy()
    b2 = (torch.randn(549, generator=g) * 0.1).numpy()
    return w1, b1, w2, b2


def _ref_heads():
    if not R.available():
        pytest.skip("reference harness not available")
    R.activate()
    from model_training.model.flame_regression import ClassificationHead
    return ClassificationHead


@pytest.mark.parametrize("train", [True, False])
def test_model_against_fp64_autograd_of_the_reference(train):
    """The model's forward and all four gradients against the reference's ClassificationHead (+ flame_regression.py:96-100)
    in fp64 under autograd, with the model's keep mask in place of nn.Dropout."""
    CH = _ref_heads()
    B, p = 5, 0.3
    f = torch.rand(B, 2048, generator=torch.Generator().manual_seed(1)).numpy()
    w1, b1, w2, b2 = _weights(2)
    m = H.forward(f, w1, b1, w2, b2, train, p, seed=9, counter=4)
    y = np.tanh(m["o"][:, :403].astype(np.float64)).astype(f32)
    g = torch.Generator().manual_seed(3)
    dparams = torch.randn(B, 413, generator=g).numpy()
    dlms = torch.randn(B, 68, 2, generator=g).numpy()
    gm = H.backward(dparams, dlms, f, w2, m["h"], m["d"], m["mask"], y, m["obits"], train, p)

    keep = torch.from_numpy(H.unpack_bits(m["mask"], 1536)).double()
    scale = float(H.dropout_scale(train, p))
    heads, r = [], 0
    for i, n in enumerate(H.HEAD_ROWS):
        ch = CH(2048, n).double()
        lin1, lin2 = ch.logit_image[0], ch.logit_image[3]
        with torch.no_grad():
            lin1.weight.copy_(torch.from_numpy(w1[i * 512:(i + 1) * 512]))
            lin1.bias.copy_(torch.from_numpy(b1[i * 512:(i + 1) * 512]))
            lin2.weight.copy_(torch.from_numpy(w2[r:r + n]))
            lin2.bias.copy_(torch.from_numpy(b2[r:r + n]))
        kp = keep[:, i * 512:(i + 1) * 512] * scale
        ch.logit_image[2] = _Mask(kp)
        heads.append(ch)
        r += n
    x = torch.from_numpy(f).double().reshape(B, 2048, 1, 1)
    shape = heads[0](x).tanh() * 3.0
    pose = heads[1](x)
    lms = torch.relu(heads[2](x).reshape(B, 68, 2))
    params = torch.cat([shape, pose], 1)
    (params * torch.from_numpy(dparams).double()).sum().add((lms * torch.from_numpy(dlms).double()).sum()).backward()

    def close(a, b, tol):
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        return np.linalg.norm(a - b) <= tol * max(np.linalg.norm(b), 1e-30)

    assert close(H.params(y, m["o"]), params.detach().numpy(), 1e-5)
    assert close(m["landmarks"], lms.detach().reshape(B, -1).numpy(), 1e-5)
    want = {"dw1": torch.cat([h.logit_image[0].weight.grad for h in heads]),
            "db1": torch.cat([h.logit_image[0].bias.grad for h in heads]),
            "dw2": torch.cat([h.logit_image[3].weight.grad for h in heads]),
            "db2": torch.cat([h.logit_image[3].bias.grad for h in heads])}
    for k, w in want.items():
        assert close(gm[k], w.numpy(), 1e-4), k


class _Mask(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, x):
        return x * self.m


def test_state_dict_round_trip():
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.heads import FlameHeads
    sd = synthetic_state_dict(0)
    heads = FlameHeads.from_state_dict(sd)
    back = heads.reference_state_dict()
    keys = {k for k in sd if ".logit_image." in k}
    assert set(back) == keys and len(keys) == 12
    for k in keys:
        assert torch.equal(back[k], sd[k].float()), k
    assert [n for n, _ in heads.named_parameters()] == ["w1", "b1", "w2", "b2"]
    with pytest.raises(ValueError):
        FlameHeads(dropout=1.0)
    with pytest.raises(TypeError):
        heads(torch.zeros(2, 2048))                  # CPU tensors: there is no CPU path
