"""CPU checks of the premises of tests/backward_model.py, the exact model the decoder backward's GPU tests compare against,
and proof that each modelled error (`Mutation`) changes an output those tests compare, on exactly their designed inputs."""
import dataclasses
import fractions
import math

import numpy as np
import pytest
import torch

from tests import backward_model as bm
from tests import decode_model as dm

F = fractions.Fraction


def test_lowbit_matches_fractions():
    g = np.random.default_rng(3)
    x = (g.standard_normal(2000) * 2.0 ** g.integers(-140, 100, 2000)).astype(np.float32)
    x[:5] = [0.0, 1.0, -3.0 * 2.0 ** -149, 2.0 ** 127, 6.0]
    got = bm.lowbit(torch.from_numpy(x))
    for i, v in enumerate(x):
        if v == 0:
            assert got[i] == math.inf
            continue
        q = abs(F(float(v)))
        low = F(1, q.denominator) if q.denominator > 1 else F(q.numerator & -q.numerator)
        assert F(got[i].item()) == low, (i, v)


def test_exact_sum_accepts_only_exact_sums():
    t = lambda *v: torch.tensor(v, dtype=torch.float64)
    assert bm.exact_sum([t(1.0), t(2.0 ** -23)], "ok").item() == 1.0 + 2.0 ** -23
    for terms in ([t(1.0), t(2.0 ** -24)],                     # needs 25 bits
                  [t(2.0 ** -150), t(2.0 ** -150)],             # below fp32's subnormal grid
                  [t(2.0 ** 23), t(2.0 ** 23), t(1.0)]):        # sum |terms| reaches 2^24 grid
        with pytest.raises(AssertionError):
            bm.exact_sum(terms, "inexact")
    # the premise is per element: heads on grids 2^-120 and 2^40 side by side
    a = t(3.0 * 2.0 ** -120, 5.0 * 2.0 ** 40)
    assert torch.equal(bm.exact_sum([a, a], "per element").double(), 2 * a)


def test_sigma_and_exponent_cap():
    """sigma lifts max |g| into [512, 1024); all-zero and non-finite maxima give 1; NaN entries are ignored (fmaxf)."""
    B, nv = 6, 5
    gv = torch.zeros(B, nv, 3)
    gv[0, 1, 2] = 3.0                       # 3 = 0.75 * 2^2 -> 2^8
    gv[1, 4, 0] = -2.0 ** -100              # -> 2^109
    gv[3, 0, 0] = float("inf")
    gv[4, 0, 0], gv[4, 1, 1] = float("nan"), 1.0
    gv[5, 2, 2] = 2.0 ** -115               # below 2^(10 - 118): capped at 2^117 for basis_scale 2^10
    xf = torch.zeros(B, 68)
    xf[:, 63] = 1.0
    s = bm.sigma(gv, None, xf, 256.0, True, 1024.0)
    assert s.tolist() == [2.0 ** 8, 2.0 ** 109, 1.0, 1.0, 2.0 ** 9, 2.0 ** 117]
    assert bm.sigma_emax(1024.0) == 117 and bm.sigma_emax(2.0 ** -8) == 127
    assert math.isfinite(s[5].item() * 1024.0)


def test_sigma_defect_at_a_threshold_head():
    """A head with max |g| just below 2^(k - 118) (k = log2 basis_scale = 10 for the designed static): without the cap its
    lift is infinite: D's hi plane is +-inf (NaN where dp = 0), its lo plane NaN (inf - inf), and so is every dcoef of the
    head; with the cap D is finite."""
    nv = 40
    st = bm.designed_static(nv, seed=1)
    pk = dm.pack(st)
    k = bm.log2_scale(pk.scale)
    assert k == 10
    g = torch.Generator().manual_seed(0)
    vposed, xf, gv, gp = bm.designed_vertex_inputs(2, nv, 128, pk.scale, [k - 129, 0], g)
    # |g| <= |gV| + sc (image / 2) |gP| with sc < 2 and |gP| <= 7 2^E
    assert 7 * 2.0 ** (k - 129) * (1 + 2 * 128) < 2.0 ** (k - 118)
    s_bad, hi_bad, lo_bad, _ = bm.vertex_stage(vposed, xf, gv, gp, pk.w2, 256.0, True, pk.scale,
                                               bm.Mutation(no_sigma_cap=True), check=True)
    assert torch.isinf(s_bad[0] * torch.tensor(pk.scale, dtype=torch.float32))
    assert torch.isinf(hi_bad[0, :3 * nv]).any() and torch.isnan(lo_bad[0, :3 * nv]).all()
    assert torch.isnan(bm.dense_stage(hi_bad, lo_bad, pk, bm.Mutation(no_sigma_cap=True))[0]).all()
    s, hi, lo, part = bm.vertex_stage(vposed, xf, gv, gp, pk.w2, 256.0, True, pk.scale)
    assert s[0].item() == 2.0 ** 117 and torch.isfinite(hi).all() and torch.isfinite(lo).all()
    assert (hi[0] != 0).any()
    assert torch.equal(hi[1], hi_bad[1]) and s[1] == s_bad[1]


# ----------------------------------------------------------------------------------------------- designed operands
VERTEX_EXPS = [-100, -60, -20, -3, 0, 7, 20, 40, None, -120]


def test_designed_vertex_inputs_are_exact_and_fill_the_lo_plane():
    """The model's exactness assertions hold on the designed vertex operands for every head magnitude (2^-120 ... 2^40);
    every non-zero head gets its own sigma, the all-zero head sigma = 1, and a good share of D's lo plane is non-zero."""
    for nv in (97, 256, 300):
        pk = dm.pack(bm.designed_static(nv, seed=nv))
        npad = (3 * nv + 127) // 128 * 128
        for to_2d, image in ((True, 256.0), (False, 224.0), (True, 512.0)):
            g = torch.Generator().manual_seed(nv)
            vposed, xf, gv, gp = bm.designed_vertex_inputs(len(VERTEX_EXPS), nv, npad, pk.scale, VERTEX_EXPS, g,
                                                           to_2d=to_2d)
            s, hi, lo, part = bm.vertex_stage(vposed, xf, gv, gp, pk.w2, image, to_2d, pk.scale)
            nz = [i for i, e in enumerate(VERTEX_EXPS) if e is not None]
            assert len(set(s[nz].tolist())) == len(nz)
            assert s[VERTEX_EXPS.index(None)].item() == 1.0
            assert s[VERTEX_EXPS.index(-120)].item() == 2.0 ** bm.sigma_emax(pk.scale)        # the capped head
            share = (lo[nz, :3 * nv] != 0).double().mean().item()
            assert share > 0.4, share
            assert (hi[:, 3 * nv:] == 0).all() and (lo[:, 3 * nv:] == 0).all()
            assert hi.abs().max().item() < 2048 and torch.isfinite(part).all()


def test_designed_d_planes_keep_the_dense_product_exact():
    for nv in (97, 5023):
        pk = dm.pack(bm.designed_static(nv, seed=nv))
        npad = (3 * nv + 127) // 128 * 128
        d_hi, d_lo = bm.designed_d_planes(4, nv, npad, torch.Generator().manual_seed(1))
        out = bm.dense_stage(d_hi, d_lo, pk)                   # asserts the exactness premise
        assert (out[:, :436] != 0).float().mean().item() > 0.9


# ---------------------------------------------------------------------------------------------------------- mutations
def _differs(a, b):
    return not torch.equal(a.view(torch.int32), b.view(torch.int32))


def _vertex_outputs(mut, nv=300):
    pk = dm.pack(bm.designed_static(nv, seed=nv))
    npad = (3 * nv + 127) // 128 * 128
    g = torch.Generator().manual_seed(nv)
    vposed, xf, gv, gp = bm.designed_vertex_inputs(len(VERTEX_EXPS), nv, npad, pk.scale, VERTEX_EXPS, g, to_2d=False)
    return bm.vertex_stage(vposed, xf, gv, gp, pk.w2, 224.0, False, pk.scale, mut)


def _dense_outputs(mut, nv=97):
    pk = dm.pack(bm.designed_static(nv, seed=nv))
    npad = (3 * nv + 127) // 128 * 128
    d_hi, d_lo = bm.designed_d_planes(16, nv, npad, torch.Generator().manual_seed(2))
    return (bm.dense_stage(d_hi, d_lo, pk, mut),)


def _finalize_outputs(mut, nv=97):
    """Linear parts (exact) of the designed finalize inputs, and the fp64 reference's excess over the GPU test's bound
    relative to the unmutated reference."""
    st = bm.designed_static(nv, seed=nv)
    pk = dm.pack(st)
    jt, jd = bm.joint_constants(st)
    params, dcoef, partial, sig = bm.designed_finalize_inputs(8, nv, torch.Generator().manual_seed(3))
    lin, mask = bm.finalize_linear(params, dcoef, partial, sig, pk.scale, 0, mut)
    ref, mag = bm.finalize_f64(params, dcoef, partial, sig, jt, jd, pk.scale, 0, mut)
    ref0, mag0 = bm.finalize_f64(params, dcoef, partial, sig, jt, jd, pk.scale, 0)
    excess = ((ref - ref0).abs() > bm.finalize_bound(params, mag0)).any()
    return lin[mask].contiguous(), torch.tensor([1.0 if excess else 0.0])


STAGES = {"vertex": _vertex_outputs, "dense": _dense_outputs, "finalize": _finalize_outputs}
SEEN_BY = {"sigma_head0": "vertex", "no_sigma_cap": "vertex", "drop_d_lo": "vertex", "drop_lohi": "dense",
           "drop_hilo": "dense", "swap_w": "vertex", "swap_a": "vertex", "partial_next_block": "finalize",
           "half_img_twice": "vertex", "tz_nonzero": "finalize", "jaw_cols_first": "finalize"}


def test_every_mutation_is_listed():
    assert set(SEEN_BY) == {f.name for f in dataclasses.fields(bm.Mutation)}


@pytest.mark.parametrize("name", sorted(SEEN_BY))
def test_every_mutation_changes_a_compared_output(name):
    run = STAGES[SEEN_BY[name]]
    base = run(bm.NONE)
    got = run(bm.Mutation(**{name: True}))
    assert any(_differs(a, b) for a, b in zip(base, got)), name
    if name == "drop_d_lo":                                     # also visible in the dense stage
        assert _differs(_dense_outputs(bm.NONE)[0], _dense_outputs(bm.Mutation(drop_d_lo=True))[0])
