"""-m "not gpu": the exact engine model (tests/engine_model.py) and its designed operands.

The model's own premises (canonical splits, exact accumulator classes) are asserted, and for every layer kind each
deliberate fault of the model must change at least one output on designed data: that is what lets the GPU tests
(tests/test_encoder_steps_gpu.py), which compare the kernels with this model bit for bit, see such a fault in a kernel."""
import numpy as np
import pytest

from tests import engine_model as em

MODES = list(em.MODES)


def cout_pad(cout):
    bn = 128 if cout % 128 == 0 else 64 if cout % 64 == 0 else 80 if cout <= 80 else 96
    return -(-cout // bn) * bn


# layer kinds at small sizes: (spec, input shape [N,H,W,C], weight shape [cout,R,S,cin], residual shape, second source)
KINDS = {
    "stem": (em.ConvSpec("stem", 4, 4, pad_h=2, pad_w=0, Ho=8, Wo=8, relu=True, stem=True), (2, 8, 12, 16),
             (64, 7, 7, 3), None, None),
    "1x1": (em.ConvSpec("s1u1c1", 1, 1, Ho=8, Wo=8, relu=True), (2, 8, 8, 128), (64, 1, 1, 128), None, None),
    "strided_1x1": (em.ConvSpec("s2u1c1", 1, 1, stride=2, Ho=4, Wo=4, relu=True), (2, 8, 8, 256), (128, 1, 1, 256),
                    None, None),
    "halo_3x3": (em.ConvSpec("s2u2c2", 3, 3, pad_h=1, pad_w=1, Ho=8, Wo=16, relu=True), (2, 8, 16, 128),
                 (128, 3, 3, 128), None, None),
    "residual_in_k": (em.ConvSpec("s1u2c3", 1, 1, Ho=8, Wo=8, relu=True, res_mode=1), (2, 8, 8, 64), (256, 1, 1, 64),
                      (2, 8, 8, 256), None),
    "projection_shortcut": (em.ConvSpec("s2u1c3", 1, 1, Ho=4, Wo=4, relu=True, res_mode=4, res_stride=2),
                            (2, 4, 4, 128), (512, 1, 1, 128 + 256), None, (2, 8, 8, 256)),
    "up2": (em.ConvSpec("b0_p6td_u", 1, 1, Ho=4, Wo=4, up2=True), (2, 4, 4, 256), (256, 1, 1, 256), None, None),
    "parity": (em.ConvSpec("b0_p3td", 1, 1, stride=2, Ho=4, Wo=4, relu=True, res_mode=1, parity=2), (2, 8, 8, 256),
               (256, 1, 1, 256), (2, 4, 4, 256), None),
    "gate": (em.ConvSpec("fusion", 1, 1, Ho=4, Wo=4, res_mode=2), (2, 4, 4, 192), (128, 1, 1, 192), (2, 4, 4, 128),
             None),
    "sparse_heat": (em.ConvSpec("heat", 3, 3, pad_h=1, pad_w=1, Ho=8, Wo=8, f32_out=True), (2, 8, 8, 256),
                    (68, 3, 3, 256), None, None),
    "mlp1": (em.ConvSpec("mlp1", 1, 1, Ho=1, Wo=5, relu=True), (1, 1, 5, 256), (192, 1, 1, 256), None, None),
    "mlp2": (em.ConvSpec("mlp2", 1, 1, Ho=1, Wo=5, f32_out=True), (1, 1, 5, 192), (90, 1, 1, 192), None, None),
}


def _design(kind, mode, seed=0, saturate=False):
    spec, xs, ws, rs, s2 = KINDS[kind]
    P, fp16 = em.MODES[mode]
    rng = np.random.default_rng(seed)
    (_, w, b), = em.design_network(rng, [(spec.name, ws)], mode, saturate)[0]
    kw = em.design_network(np.random.default_rng(seed), [(spec.name, ws)], mode, saturate)[1][spec.name]
    cp = cout_pad(ws[0])
    bias = np.zeros(cp, np.float32)
    bias[:ws[0]] = b
    valid_c = 12 if spec.stem else None
    x, xp = em.design_tensor(rng, xs, P, fp16, valid_c=valid_c)
    if spec.stem:                                    # the s2d tensor's two zero columns on each side
        for a in [x] + xp:
            a[:, :, :2] = 0
            a[:, :, -2:] = 0
    res = src2 = None
    if rs is not None:
        if spec.res_mode == 2:
            res, _ = em.design_tensor(rng, rs, P, fp16, k=-3)
        else:
            kr = np.zeros(rs[-1], np.int64)
            kr[:ws[0]] = em.residual_exponent(fp16, kw)
            kr[ws[0]:] = kr[0]
            res, _ = em.design_tensor(rng, rs, P, fp16, k=kr)
    if s2 is not None:
        src2, _ = em.design_tensor(rng, s2, P, fp16)
    rows = [0, 1, 4, 5] if kind == "sparse_heat" else None
    pix = em.sample_pixels(xs[0], spec.Ho, spec.Wo, 8, 8, 1, rows=rows)
    return spec, w, bias, x, res, src2, pix


def _run(kind, mode, mut=em.Mutation(), saturate=False):
    spec, w, bias, x, res, src2, pix = _design(kind, mode, saturate=saturate)
    P, fp16 = em.MODES[mode]
    packed = em.pack(spec.name, w, P, fp16, trunc=mut.trunc_split)
    return em.conv_step(spec, packed, bias, x, pix, P, fp16, res=res, src2=src2, mut=mut)


def test_rounding_helpers():
    x = np.array([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 70000.0, -1e6, 2 ** -20], np.float32)
    assert list(em.rn_bf16(x)[:3]) == [1.0, 1.0 + 2 ** -6, -1.0]          # ties to even
    assert list(em.rn_f16_sat(x)[3:5]) == [65504.0, -65504.0]              # satfinite
    assert em.rz_bf16(np.float32(1.0 + 3 * 2 ** -8)) == 1.0 + 2 ** -7
    v = np.float32(np.pi)
    for mode in MODES:                               # P pieces keep 8P (bf16) / 11P (fp16) bits: the rest is rounded off
        P, fp16 = em.MODES[mode]
        ps = em.split(v, P, fp16)
        err = abs(float(em.sum_pieces(ps)) - float(v))
        half_ulp_last = 2.0 ** (np.frexp(abs(float(ps[-1])))[1] - (11 if fp16 else 8) - 1)
        assert len(ps) == P and all(p != 0 for p in ps) and err <= half_ulp_last
        assert err == 0 if P == 3 else err > 0
    assert em.grid_of([3.0, 0.5, 0.0]) == 0.5 and em.grid_of([-12.0]) == 4.0


@pytest.mark.parametrize("mode", MODES)
def test_designed_values_are_canonical_and_complete(mode):
    P, fp16 = em.MODES[mode]
    rng = np.random.default_rng(1)
    x, pieces = em.design_tensor(rng, (2, 4, 4, 64), P, fp16)
    for p in pieces:
        assert (p != 0).mean() > 0.99
    w, kw = em.design_weights(rng, "s1u1c2", 64, 3, 3, 64, P, fp16)
    packed = em.pack("s1u1c2", w, P, fp16)
    for q in packed.pieces:                          # every piece of every non-zero weight is present
        assert ((q != 0) == (w != 0)).all()
    if fp16:                                         # the per-row scale is the designed one: scaled rows in [2^14, 2^15)
        amax = np.abs(packed.pieces[0].reshape(64, -1)).max(1)
        assert ((amax >= 2 ** 14) & (amax < 2 ** 15)).all()
        assert np.array_equal(packed.up, np.ldexp(1.0, 11 - kw).astype(np.float32))


def test_stem_4x4_is_the_7x7_stride_2_conv():
    """The 4x4/1 conv over the 2x2 space-to-depth image equals the 7x7/2 pad-3 conv (products are exact)."""
    rng = np.random.default_rng(2)
    w7 = rng.integers(-4, 5, size=(64, 7, 7, 3)).astype(np.float32)
    img = rng.integers(-8, 9, size=(1, 16, 16, 3)).astype(np.float64)
    s2d = np.zeros((1, 8, 12, 16))
    for py in range(2):
        for px in range(2):
            s2d[0, :, 2:10, (py * 2 + px) * 3:(py * 2 + px) * 3 + 3] = img[0, py::2, px::2]
    spec = em.ConvSpec("stem", 4, 4, pad_h=2, pad_w=0, Ho=8, Wo=8, stem=True, f32_out=True)
    pix = em.sample_pixels(1, 8, 8, 8, 8, 1)
    packed = em.Packed([em.stem_to_4x4(w7)], np.ones(64, np.float32), np.ones(64, np.float32), None)
    got = em.conv_step(spec, packed, np.zeros(64, np.float32), s2d.astype(np.float32), pix, 1, False)
    pad = np.pad(img[0], ((3, 3), (3, 3), (0, 0)))
    want = np.zeros((8, 8, 64))
    for oy in range(8):
        for ox in range(8):
            want[oy, ox] = np.einsum("rsc,orsc->o", pad[2 * oy:2 * oy + 7, 2 * ox:2 * ox + 7], w7)
    assert np.array_equal(got.reshape(8, 8, 64), want.astype(np.float32))


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("mode", MODES)
def test_model_premises_hold_on_designed_data(kind, mode):
    """conv_step asserts the exactness premise itself; here: outputs are finite, ReLU clips some and keeps others."""
    out = _run(kind, mode)
    assert np.isfinite(out).all()
    spec = KINDS[kind][0]
    real = out[:, :KINDS[kind][2][0]]
    if spec.relu:
        assert (real == 0).mean() > 0.05 and (real > 0).mean() > 0.05
    else:
        assert (real < 0).mean() > 0.05


@pytest.mark.parametrize("mode", ["fp16x2", "fp16"])
def test_fp16_outputs_saturate(mode):
    out = _run("1x1", mode, saturate=True)
    assert np.isfinite(out).all()
    P, _ = em.MODES[mode]
    top = out[:, ::8].max()
    assert top >= 65504.0 and (P == 2 or top == 65504.0)


MUTATIONS = {
    "trunc_acc_sum": em.Mutation(trunc_acc_sum=True),
    "trunc_split": em.Mutation(trunc_split=True),
    "bias_before_scale": em.Mutation(bias_before_scale=True),
    "skip_last_kblock": em.Mutation(skip_last_kblock=True),
    "shift_tap": em.Mutation(shift_tap=True),
}


@pytest.mark.parametrize("kind", list(KINDS))
def test_mutations_change_a_checked_output(kind):
    """Each mutation must change at least one output in at least one mode where it means something (a bias/scale swap
    needs the fp16 scale, a truncated acc0 + acc1 needs two accumulators)."""
    base = {m: _run(kind, m) for m in MODES}
    missed = []
    for mname, mut in MUTATIONS.items():
        if not any(not np.array_equal(_run(kind, m, mut), base[m]) for m in MODES):
            missed.append(mname)
    for m in MODES:                                   # every single product, in every mode
        for i in range(len(em.products(em.MODES[m][0]))):
            if np.array_equal(_run(kind, m, em.Mutation(drop_product=i)), base[m]):
                missed.append(f"{m}: drop product {em.products(em.MODES[m][0])[i]}")
    if KINDS[kind][3] is not None and KINDS[kind][0].res_mode == 1:
        for m in MODES:
            if np.array_equal(_run(kind, m, em.Mutation(no_identity=True)), base[m]):
                missed.append(f"{m}: residual blocks dropped")
    assert not missed, missed


def test_sample_covers_partial_tiles_and_borders():
    pix = em.sample_pixels(64, 64, 64, 8, 16, 1, n_random=64)
    s = set(map(tuple, pix.tolist()))
    assert (63, 63, 63) in s and (0, 0, 0) in s and (0, 63, 17) in s and (63, 60, 60) in s
    assert all((0, h, 0) in s and (63, h, 63) in s for h in range(64))
    assert len(pix) < 6144
    rows = [0, 1, 4, 5]
    assert set(em.sample_pixels(2, 8, 8, 8, 2, 1, rows=rows)[:, 1]) == set(rows)
