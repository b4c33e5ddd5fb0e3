"""CPU checks of the premises of tests/decode_model.py, the exact model the decoder's GPU tests compare against."""
import fractions
import math
import struct

import numpy as np
import pytest
import torch

from tests import decode_model as dm

F = fractions.Fraction


def _round_f32(q: F) -> float:
    """Round a rational to binary32, ties to even (normal and subnormal results)."""
    if q == 0:
        return 0.0
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = max(math.floor(math.log2(q.numerator) - math.log2(q.denominator)), -126)
    while F(2) ** e > q:
        e -= 1
    while F(2) ** (e + 1) <= q:
        e += 1
    e = max(e, -126)
    ulp = F(2) ** (e - 23)
    m = q / ulp
    n = m.numerator // m.denominator
    r = m - n
    if r > F(1, 2) or (r == F(1, 2) and n % 2 == 1):
        n += 1
    return sign * float(n * ulp)


def _f32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", x))[0]


def _fmaf(a, b, c) -> float:
    t = lambda v: torch.tensor([v], dtype=torch.float32)
    return dm.fmaf(t(a), t(b), t(c)).item()


def test_fmaf_emulation_is_correctly_rounded_on_random_values():
    g = np.random.default_rng(0)
    n = 4000
    a = (g.standard_normal(n) * 2.0 ** g.integers(-30, 30, n)).astype(np.float32)
    b = (g.standard_normal(n) * 2.0 ** g.integers(-30, 30, n)).astype(np.float32)
    c = (g.standard_normal(n) * 2.0 ** g.integers(-60, 60, n)).astype(np.float32)
    c[: n // 4] = (-(a[: n // 4].astype(np.float64) * b[: n // 4])).astype(np.float32)    # heavy cancellation
    got = dm.fmaf(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c)).numpy()
    for i in range(n):
        want = _round_f32(F(float(a[i])) * F(float(b[i])) + F(float(c[i])))
        assert got[i] == np.float32(want), (i, a[i], b[i], c[i])


def test_fmaf_emulation_on_midpoints_and_double_rounding_cases():
    u = 2.0 ** -23
    cases = [
        (2.0 ** -12, 2.0 ** -12, 1.0),                        # exact midpoint 1 + 2^-24: ties to even -> 1
        (2.0 ** -12, 2.0 ** -12, 1.0 + u),                    # midpoint above an odd value: ties to even -> 1 + 2^-22
        (1.0 + u, _f32(2.0 ** -24 * (1.0 - u)), 1.0 + u),     # fp64 rounding lands on the midpoint: naive double rounding errs
        (-(1.0 + u), _f32(2.0 ** -24 * (1.0 - u)), -(1.0 + u)),
        (1.0 + u, 1.0 - u, -1.0),                             # exact -2^-46
        (3.0, _f32(1.0 / 3.0), -1.0),
    ]
    naive_wrong = 0
    for a, b, c in cases:
        want = _round_f32(F(a) * F(b) + F(c))
        assert _fmaf(a, b, c) == want, (a, b, c)
        naive = float(np.float32(np.float64(a) * np.float64(b) + np.float64(c)))
        naive_wrong += naive != want
    assert naive_wrong >= 2          # the constructed cases do defeat a plain fp64 evaluation


def test_dec_phys_row_and_head_of_are_inverse():
    h = torch.arange(4 * 256)
    r = dm.dec_phys_row(h)
    assert torch.equal(torch.sort(r).values, h)                   # a permutation of every 256-block
    m_tile, wq, lane = r // 128, (r % 128) // 32, r % 32
    assert torch.equal(dm.dec_head_of(m_tile, wq, lane), h)
    assert torch.equal((h % 8)[r // 32 == (r // 32)], h % 8)
    for q in range(r.numel() // 32):                             # one warp = heads equal mod 8 (one sector phase)
        heads = h[(r // 32) == q]
        assert (heads % 8 == heads[0] % 8).all()


def test_packing_premises_on_the_real_asset(flame_static):
    nv = flame_static["v_template"].shape[0]
    sd = np.asarray(flame_static["shapedirs"], np.float32).reshape(3 * nv, -1)
    pd = np.asarray(flame_static["posedirs"], np.float32)
    vt = np.asarray(flame_static["v_template"], np.float32).reshape(-1)
    s = dm.basis_scale(sd, pd, vt)
    amax = max(np.abs(sd).max(), np.abs(pd).max()) * s
    assert math.log2(s) == int(math.log2(s))
    assert 512 <= amax < 1024 or np.abs(vt).max() * s * 2 >= 2 ** 15          # the basis rule or the template clamp
    assert np.abs(vt).max() * s < 2 ** 15
    pk = dm.pack(flame_static)
    tmpl = pk.hi[:, dm.TMPL].double() + pk.hi[:, dm.TMPL + 1].double() + pk.lo[:, dm.TMPL].double() + pk.lo[:, dm.TMPL + 1].double()
    # four pieces carry the template up to fp16 underflow of the last piece (half the smallest subnormal, 2^-25)
    err = (tmpl - torch.from_numpy(vt).double() * s).abs()
    assert err.max().item() <= 2.0 ** -25 and (err == 0).float().mean() > 0.99
    x = torch.from_numpy(sd).double() * s
    assert ((pk.hi[:, :400].double() + pk.lo[:, :400].double() - x).abs() <= x.abs() * 2.0 ** -22 + 2.0 ** -25).all()
    w = np.asarray(flame_static["lbs_weights"], np.float32)
    assert np.array_equal(pk.w2[:, 1].numpy(), w[:, 2])


def test_designed_operands_are_exact_and_packed_as_designed():
    st = dm.designed_static(97, seed=1)
    pk = dm.pack(st)
    assert pk.scale == 1024.0
    assert dm.grid_of(pk.hi[:, :436]) == 1.0 and dm.grid_of(pk.lo[:, :436]) == 2.0 ** -12
    assert (pk.lo[:, :436] != 0).float().mean() > 0.5
    assert (pk.w2[:, 0] != pk.w2[:, 1]).all() and len(set(pk.w2[:, 0].tolist())) == 97
    g = torch.Generator().manual_seed(0)
    hi, lo = dm.designed_rows(40, g)
    xf = dm.designed_xf(40, g, pk.scale)
    for path in ("dedicated", "lbs", "blend"):
        dm.decode(path, hi, lo, xf, pk)                            # asserts the exactness premise for every output
    assert (dm.product("lbs", hi, lo, pk, dm.Mutation(add_lolo=True)) != dm.product("lbs", hi, lo, pk)).any()
    assert (pk.lo[:, dm.TMPL].abs() == 2.0 ** -10).sum() > 10 and dm.grid_of(pk.hi[:, dm.TMPL:dm.TMPL + 2]) == 0.5
    assert (pk.lo[:, dm.TMPL + 1] == 0).all()                     # a fourth piece cannot fit an exact design


def _design(nv=37, B=24, seed=3):
    pk = dm.pack(dm.designed_static(nv, seed=seed))
    g = torch.Generator().manual_seed(seed)
    hi, lo = dm.designed_rows(B, g)
    return pk, hi, lo, dm.designed_xf(B, g, pk.scale)


MUTATIONS = {
    "lbs": [dm.Mutation(drop_lohi=True), dm.Mutation(drop_hilo=True), dm.Mutation(add_lolo=True),
            dm.Mutation(drop_tmpl_piece=0), dm.Mutation(drop_tmpl_piece=1), dm.Mutation(drop_tmpl_piece=2),
            dm.Mutation(drop_col437=True), dm.Mutation(swap_w=True), dm.Mutation(neighbour_w=True), dm.Mutation(swap_rj=True),
            dm.Mutation(no_z_offset=True), dm.Mutation(image_size_for_hs=True), dm.Mutation(tz_nonzero=True)],
    "dedicated": [dm.Mutation(drop_tmpl_piece=0), dm.Mutation(drop_tmpl_piece=1), dm.Mutation(drop_col437=True),
                  dm.Mutation(swap_w=True), dm.Mutation(neighbour_w=True), dm.Mutation(swap_rj=True),
                  dm.Mutation(carry_shift=True), dm.Mutation(carry_prev_row=True), dm.Mutation(no_z_offset=True),
                  dm.Mutation(image_size_for_hs=True), dm.Mutation(tz_nonzero=True)],
    "blend": [dm.Mutation(drop_lohi=True), dm.Mutation(drop_hilo=True), dm.Mutation(add_lolo=True),
              dm.Mutation(drop_tmpl_piece=2), dm.Mutation(drop_col437=True), dm.Mutation(no_z_offset=True),
              dm.Mutation(image_size_for_hs=True)],
}


@pytest.mark.parametrize("path", sorted(MUTATIONS))
def test_every_mutation_changes_a_compared_output(path):
    """On the designed operands each modelled error changes at least one output the GPU tests compare bit for bit (both
    outputs, 3-component projection, and for the store mutations every sector phase of the base offset)."""
    pk, hi, lo, xf = _design()
    for base in range(8) if path == "dedicated" else (0,):
        ref = dm.decode(path, hi, lo, xf, pk, to_2d=False, base_v=base, base_p=base)
        for mut in MUTATIONS[path]:
            if base and not (mut.carry_shift or mut.carry_prev_row):
                continue
            got = dm.decode(path, hi, lo, xf, pk, to_2d=False, mut=mut, base_v=base, base_p=base)
            changed = sum(int((a.view(torch.int32) != b.view(torch.int32)).sum()) for a, b in zip(ref, got))
            assert changed > 0 or (base == 0 and (mut.carry_shift or mut.carry_prev_row)), (path, mut, base)


def test_carry_mask_covers_every_phase():
    """The carried floats of a row are the c floats in front of every pass start, c = the row's phase mod 8."""
    m = dm.carry_mask(8, 40, 3, 0)
    n = 120
    for h in range(8):
        c = (h * n) % 8
        want = [any(g0 - c <= j < g0 for g0 in range(24, n, 24)) for j in range(n)]
        assert m[h].tolist() == want
