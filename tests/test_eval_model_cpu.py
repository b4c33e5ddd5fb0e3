"""CPU checks of tests/eval_model.py, the exact model the evaluator's GPU tests compare against: it agrees with the oracle's
calc_zn and with a float64 chamfer, and each modelled error changes an output on the inputs those GPU tests use."""
import itertools
from fractions import Fraction as F

import pytest
import torch

from oracle.evaluator_oracle import calc_zn
from tests import eval_model as em


def test_sqrtf_and_divf_are_correctly_rounded():
    """Checked with exact rationals, on random values and on values where torch's fp32 CPU sqrt is one ulp off."""
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.tensor([36.67272186279297, 10.630736351013184, 1.9728565216064453]),
                   torch.rand(3000, generator=g) * 40, torch.rand(1000, generator=g) * 1e-3])
    y = torch.randint(1, 65536, (x.numel(),), generator=g)
    r, q = em.sqrtf(x), em.divf(x, 1.0)
    for xi, ri, yi in zip(x.tolist(), r.tolist(), y.tolist()):
        lo, hi = F(torch.tensor(ri).nextafter(torch.tensor(0.0)).item()), F(torch.tensor(ri).nextafter(torch.tensor(99.0)).item())
        mid_lo, mid_hi = (lo + F(ri)) / 2, (hi + F(ri)) / 2
        assert mid_lo ** 2 <= F(xi) <= mid_hi ** 2, xi
        qi = em.divf(torch.tensor([xi]), yi).item()
        exact = F(xi) / yi
        qlo = F(torch.tensor(qi).nextafter(torch.tensor(-1.0)).item())
        qhi = F(torch.tensor(qi).nextafter(torch.tensor(99.0)).item())
        assert (qlo + F(qi)) / 2 <= exact <= (qhi + F(qi)) / 2, (xi, yi)
    assert torch.equal(q, x)


@pytest.mark.parametrize("K", [64, 1000, 3669])
def test_zn_model_matches_oracle_calc_zn(K):
    """On points without near-ties the model's count is the reference's: this pins the column quirk (columns 1..top_k of
    the column-sorted gt distance matrix)."""
    g = torch.Generator().manual_seed(K)
    for top_k in (1, 5, 16):
        gt = em.separated_points(K, top_k, seed=K + top_k)
        pred = gt + 0.3 * torch.randn(K, 3, generator=g)
        got = int(em.zn_counts(pred[None], gt[None], top_k).sum())
        want = round(calc_zn(pred, gt, top_k) * K * top_k)
        assert got == want, (K, top_k, got, want)


def test_separated_points_are_separated():
    gt = em.separated_points(1000, 5, seed=3).double()
    for c in range(1, 6):
        s = torch.sort(((gt - gt[c]) ** 2).sum(1)).values
        assert (s[1:] - s[:-1]).min() > 3e-5


@pytest.mark.parametrize("na,nb", [(1, 1), (31, 1025), (257, 1024), (2094, 5023)])
def test_chamfer_model_matches_float64(na, nb):
    a, b = em.chamfer_inputs(na, nb, 2, seed=na + nb)
    total = em.chamfer_terms(a, b).double().sum(1)
    want = (torch.cdist(a.double(), b.double()) ** 2).min(2).values.mean(1)
    assert ((total - want).abs() <= 1e-5 * want).all(), (total, want)


def test_chamfer_block_sum_is_the_kernel_tree():
    """The butterfly is a fixed tree: with values whose fp32 sums depend on the order, the model's block term differs
    from a sequential sum, and equals the tree written out by hand."""
    v = torch.tensor([1.0, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24] * 8)
    a = torch.zeros(1, 32, 3)
    a[0, :, 0] = v.sqrt()
    b = torch.zeros(1, 1, 3)
    term = em.chamfer_terms(a, b)[0, 0].item()
    assert em.chamfer_minima(a, b)[0].tolist() == v.tolist()
    x = v.clone()
    for o in (16, 8, 4, 2, 1):
        x = x + x[torch.arange(32) ^ o]
    assert term == (x[0] / 32).item()


def test_align_and_gather_bary_models_round_once_per_fma():
    """fmaf chains, not fp32 products and sums: the models differ from the unfused evaluation on some element."""
    v, s, r, t = em.align_inputs(5023, 3, seed=0)
    got = em.align(v, s, r, t)
    unfused = s[:, None, None] * (v @ r) + t[:, None, :]
    assert not torch.equal(got, unfused)
    want64 = s.double()[:, None, None] * (v.double() @ r.double()) + t.double()[:, None, :]
    assert ((got.double() - want64).abs() <= 4 * em.U * (want64.abs() + 1e3)).all()
    src = torch.randn(2, 50, 3)
    tri = torch.randint(0, 50, (40, 3))
    bary = torch.randn(40, 3)
    gb = em.gather_bary(src, tri, bary)
    exact = (src.double()[:, tri] * bary.double()[None, :, :, None]).sum(2)
    assert ((gb.double() - exact).abs() <= 4 * em.U * (src.double()[:, tri].abs() * bary.double().abs()[None, :, :, None]).sum(2)).all()


# ------------------------------------------------------------------------------------------------ mutations are visible
def _zn_detects(mut):
    for K, top_k, kind in itertools.product(em.ZN_K, em.ZN_TOP_K, em.ZN_KINDS):
        K = em.zn_k(K, top_k)
        if K <= top_k:
            continue
        pred, gt = em.zn_case(kind, K, top_k)
        if not torch.equal(em.zn_counts(pred, gt, top_k, mut), em.zn_counts(pred, gt, top_k)):
            return kind, K, top_k
    return None


@pytest.mark.parametrize("mut", [em.Mutation(zn_rowwise=True), em.Mutation(zn_cols_from_0=True),
                                 em.Mutation(zn_ties_desc=True), em.Mutation(zn_strict=True)], ids=str)
def test_zn_mutation_changes_a_count(mut):
    """The GPU test requires the recovered count to equal the model's exactly, so any changed count is seen."""
    assert _zn_detects(mut) is not None, mut


def test_zn_self_key_is_zero_without_forcing():
    """The key formula gives exactly 0 at k == c: n2 and dot are the same fmaf chain there, so n2 + cn - 2 dot =
    2 cn - 2 cn.  Forcing key[c] to 0 is therefore invisible in the kernel's output, and the model shows it on every
    input the GPU tests use (and on large, badly scaled points)."""
    mut = em.Mutation(zn_no_self_zero=True)
    assert _zn_detects(mut) is None
    g = torch.Generator().manual_seed(5)
    gt = torch.randn(2, 300, 3, generator=g) * torch.logspace(-6, 6, 300)[None, :, None]
    cols = torch.arange(1, 17)
    assert (em._keys(gt, cols, mut)[:, torch.arange(16), cols] == 0).all()


@pytest.mark.parametrize("mut", [em.Mutation(chamfer_drop_tail=True), em.Mutation(chamfer_div_nb=True)], ids=str)
def test_chamfer_mutation_escapes_the_gpu_tolerance(mut):
    """Some chamfer case of the GPU test moves out of the interval that test accepts (bit-exact for one block)."""
    for na, nb, B in itertools.product(em.CHAMFER_NA[:4], em.CHAMFER_NB, em.CHAMFER_B):
        a, b = em.chamfer_case(na, nb, B)
        total, bound = em.chamfer_bound(em.chamfer_terms(a, b))
        mtotal, mbound = em.chamfer_bound(em.chamfer_terms(a, b, mut))
        if ((mtotal - total).abs() > bound + mbound).any():
            return
    pytest.fail(str(mut))


def test_align_mutation_changes_an_output():
    mut = em.Mutation(align_transposed=True)
    for nv, B in itertools.product(em.ALIGN_NV, em.ALIGN_B):
        v, s, r, t = em.align_case(nv, B)
        if not torch.equal(em.align(v, s, r, t, mut).view(torch.int32), em.align(v, s, r, t).view(torch.int32)):
            return
    pytest.fail("align_transposed is invisible")
