"""-m gpu: the evaluator's kernels (csrc/evaluator.cu, and the landmark gathers of csrc/flame.cu) through the C ABI, against
the exact fp32 model in tests/eval_model.py -- bit for bit where the kernel's result has a fixed order, and within the
model's bound where atomics add per-block terms in any order -- and DADEvaluatorGPU head by head against the oracle."""
import json
from collections import defaultdict

import numpy as np
import pytest
import torch

from tests import eval_model as em

pytestmark = pytest.mark.gpu

INVALID = -1


def _lib():
    from dad_3dheads_b200 import _lib
    return _lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.detach().cpu().contiguous().view(torch.int32)


def _assert_bits(got: torch.Tensor, want: torch.Tensor, what):
    diff = _bits(got) != _bits(want)
    assert not diff.any(), (what, int(diff.sum()), got.cpu()[diff][:4], want[diff][:4])


def _chamfer(a, b):
    out = torch.empty(a.shape[0], device="cuda")
    rc = _lib().dad3d_eval_chamfer(a.data_ptr(), a.shape[1], b.data_ptr(), b.shape[1], a.shape[0], out.data_ptr(), _stream())
    assert rc == 0, _lib().dad3d_last_error()
    return out.cpu()


def _zn(pred, gt, top_k):
    B, K, _ = gt.shape
    out = torch.empty(B, device="cuda")
    rc = _lib().dad3d_eval_zn(pred.data_ptr(), gt.data_ptr(), K, B, top_k, out.data_ptr(), _stream())
    assert rc == 0, _lib().dad3d_last_error()
    return out.cpu()


def _check_zn(got: torch.Tensor, counts: torch.Tensor, K: int, what):
    """The count recovered from the output equals the model's, and the output lies within top_k - 1 ulps of the model's
    value: the columns' non-negative terms are added by atomics in any order."""
    top_k = counts.shape[1]
    total = counts.sum(1)
    rec = torch.round(got.double() * K * top_k).long()
    bad = rec != total
    assert not bad.any(), (what, int(bad.sum()), rec[bad][:4], total[bad][:4])
    want = em.zn_value(counts, K)
    err = (got.double() - want.double()).abs()
    assert (err <= (top_k - 1) * em.ulp(torch.maximum(got, want))).all(), (what, err.max().item())


# ---------------------------------------------------------------------------------------------------------------- align
@pytest.mark.parametrize("B", em.ALIGN_B)
@pytest.mark.parametrize("nv", em.ALIGN_NV)
def test_align_exact(cuda_device, nv, B):
    """Zero and negative scales, reflections, translations around 1e3: bit-exact."""
    v, s, r, t = em.align_case(nv, B)
    dv, ds, dr, dt = (x.to(cuda_device).contiguous() for x in (v, s, r, t))
    out = torch.empty_like(dv)
    assert _lib().dad3d_eval_align(dv.data_ptr(), nv, B, ds.data_ptr(), dr.data_ptr(), dt.data_ptr(), out.data_ptr(),
                                   _stream()) == 0
    _assert_bits(out, em.align(v, s, r, t), (nv, B))


# -------------------------------------------------------------------------------------------------------------- gathers
@pytest.mark.parametrize("ncomp", [2, 3])
def test_gathers_exact(cuda_device, ncomp):
    """First and last vertex, repeated indices, negative barycentric weights; one head next to many; L = 0."""
    lib = _lib()
    nv = 97
    g = torch.Generator().manual_seed(ncomp)
    idx = torch.cat([torch.tensor([0, nv - 1, 5, 5, 0, nv - 1], dtype=torch.int32),
                     torch.randint(0, nv, (40,), generator=g, dtype=torch.int32)])
    tri = torch.randint(0, nv, (30, 3), generator=g, dtype=torch.int32)
    tri[0] = torch.tensor([0, nv - 1, 0])
    tri[1] = torch.tensor([7, 7, 7])
    bary = torch.randn(30, 3, generator=g)
    bary[2] = torch.tensor([1.5, -0.25, -0.25])
    di, dtri, dbary = idx.cuda(), tri.cuda(), bary.cuda()
    for B in (1, 300):
        src = torch.randn(B, nv, ncomp, generator=g) * 100.0
        ds = src.cuda()
        out = torch.empty(B, idx.numel(), ncomp, device="cuda")
        assert lib.dad3d_gather_landmarks(ds.data_ptr(), B, nv, ncomp, di.data_ptr(), idx.numel(), out.data_ptr(),
                                          _stream()) == 0
        _assert_bits(out, em.gather(src, idx), ("gather", B))
        out = torch.empty(B, tri.shape[0], ncomp, device="cuda")
        assert lib.dad3d_gather_landmarks_bary(ds.data_ptr(), B, nv, ncomp, dtri.data_ptr(), dbary.data_ptr(), tri.shape[0],
                                               out.data_ptr(), _stream()) == 0
        _assert_bits(out, em.gather_bary(src, tri, bary), ("gather_bary", B))
    sentinel = torch.full((4,), 7.0, device="cuda")
    assert lib.dad3d_gather_landmarks(ds.data_ptr(), 300, nv, ncomp, di.data_ptr(), 0, sentinel.data_ptr(), _stream()) == 0
    assert lib.dad3d_gather_landmarks_bary(ds.data_ptr(), 300, nv, ncomp, dtri.data_ptr(), dbary.data_ptr(), 0,
                                           sentinel.data_ptr(), _stream()) == 0
    assert (sentinel.cpu() == 7.0).all()


# -------------------------------------------------------------------------------------------------------------- chamfer
@pytest.mark.parametrize("nb", em.CHAMFER_NB)
@pytest.mark.parametrize("na", em.CHAMFER_NA)
def test_chamfer_exact(cuda_device, na, nb):
    """One block (na <= 256): bit-exact, a single atomicAdd onto zero.  More blocks: within the model's bound for adding
    its per-block terms in any order."""
    for B in em.CHAMFER_B:
        a, b = em.chamfer_case(na, nb, B)
        got = _chamfer(a.to(cuda_device), b.to(cuda_device))
        terms = em.chamfer_terms(a, b)
        if terms.shape[1] == 1:
            _assert_bits(got, terms[:, 0], (na, nb, B))
        else:
            total, bound = em.chamfer_bound(terms)
            assert ((got.double() - total).abs() <= bound).all(), (na, nb, B, got, total, bound)


@pytest.mark.parametrize("na", [31, 2094])
def test_chamfer_coincident_points_give_zero(cuda_device, na):
    g = torch.Generator().manual_seed(na)
    b = torch.randn(3, 5023, 3, generator=g) * 30.0
    a = torch.gather(b, 1, torch.randint(0, 5023, (3, na, 1), generator=g).expand(-1, -1, 3)).contiguous()
    got = _chamfer(a.to(cuda_device), b.to(cuda_device))
    assert torch.equal(_bits(got), torch.zeros(3, dtype=torch.int32))


# ------------------------------------------------------------------------------------------------------------------ Z_n
@pytest.mark.parametrize("kind", em.ZN_KINDS)
@pytest.mark.parametrize("top_k", em.ZN_TOP_K)
@pytest.mark.parametrize("K", em.ZN_K)
def test_zn_exact(cuda_device, K, top_k, kind):
    """Random points; small-integer lattices (exact distances, ties and equal depths everywhere: the index tie-break,
    the self key and '>='); a copy of a centre point at a lower index.  K around the bitonic sort's 4096 padding."""
    K = em.zn_k(K, top_k)
    pred, gt = em.zn_case(kind, K, top_k)
    got = _zn(pred.to(cuda_device), gt.to(cuda_device), top_k)
    _check_zn(got, em.zn_counts(pred, gt, top_k), K, (K, top_k, kind))


def test_zn_rejects_invalid_arguments(cuda_device):
    lib = _lib()
    buf = torch.zeros(4097 * 3, device="cuda")
    out = torch.zeros(1, device="cuda")
    for K, top_k in ((4097, 5), (10, 10), (10, 11), (10, 0)):
        assert lib.dad3d_eval_zn(buf.data_ptr(), buf.data_ptr(), K, 1, top_k, out.data_ptr(), _stream()) == INVALID, (K, top_k)
    assert out.item() == 0.0


# ------------------------------------------------------------------------------------------------------------ many heads
def test_more_heads_than_one_grid_dimension(cuda_device):
    """Both batched kernels put the head on grid.y (at most 65535 blocks): larger batches must still give every head."""
    B = 65535 + 7
    g = torch.Generator().manual_seed(11)
    a, b = torch.randn(B, 3, 3, generator=g), torch.randn(B, 2, 3, generator=g)
    _assert_bits(_chamfer(a.to(cuda_device), b.to(cuda_device)), em.chamfer_terms(a, b)[:, 0], "chamfer")
    gt = torch.randn(B, 4, 3, generator=g)
    pred = torch.randn(B, 4, 3, generator=g)
    _check_zn(_zn(pred.to(cuda_device), gt.to(cuda_device), 2), em.zn_counts(pred, gt, 2), 4, "zn")


# ---------------------------------------------------------------------------------------------------------- end to end
N_HEADS = 40


@pytest.fixture(scope="module")
def heads():
    """40 heads, the GPU evaluator's per-head metrics, the oracle's, and the model's Z5 counts on the model's own aligned
    and gathered inputs."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from dad_3dheads_b200.evaluator import DADEvaluatorGPU
    from dad_3dheads_b200.flame import load_flame_static
    from oracle.evaluator_oracle import EvaluatorOracle
    from tests.eval_fixtures import make_pairs
    gts, sub = make_pairs(N_HEADS, seed=9)
    st = load_flame_static()
    ev = DADEvaluatorGPU(static=st)
    res = ev.metrics(gts, [sub[a["id"]] for a in gts])
    orc = EvaluatorOracle(st, st["head_indices"], st["flame_indices_face"])
    want = [orc.sample(a, sub[a["id"]]) for a in gts]
    f32 = lambda key, src: torch.from_numpy(np.asarray([s[key] for s in src], dtype=np.float32))
    verts, mv = f32("vertices", gts), f32("model_view_matrix", gts)
    pred_v = f32("N_landmarks_3d", [sub[a["id"]] for a in gts]).reshape(N_HEADS, -1, 3)
    head = torch.from_numpy(np.asarray(st["head_indices"], dtype=np.int64))
    world = em.align(verts, torch.ones(N_HEADS), mv[:, :3, :3].transpose(1, 2), mv[:, :3, 3])
    z5 = em.zn_counts(em.gather(pred_v, head), em.gather(world, head) * -1.0, 5)
    return gts, sub, st, res, want, z5, head.numel()


TOL = {"pose_error": (1e-4, 1e-5), "nme": (1e-4, 1e-6), "chamfer": (1e-4, 1e-6)}      # relative, absolute
ORACLE = {"pose_error": "pose_error", "nme": "nme_reprojection", "z5": "z5_accuracy", "chamfer": "chamfer"}


def test_metrics_per_head(heads):
    """Pose error, NME and chamfer head by head against the oracle; Z5 head by head exactly against the model (the
    oracle's torch.cdist reorders near-equal distances, so Z5 against it is only comparable as a mean)."""
    gts, _, _, res, want, z5, K = heads
    for n, (rt, at) in TOL.items():
        got = np.asarray(res[n], np.float64)
        w = np.array([r[ORACLE[n]] for r in want])
        err = np.abs(got - w)
        assert (err <= rt * np.abs(w) + at).all(), (n, int(np.argmax(err - rt * np.abs(w))), err.max())
    _check_zn(torch.from_numpy(res["z5"]), z5, K, "z5")


def test_call_batches_and_skips_missing_ids(heads, tmp_path, capsys):
    """batch=16 over 37 of the 40 heads (3 ids missing from the submission): chunks of 16, 16 and 5 in ground-truth
    order; every head's values land in the overall and per-attribute means under its own keys."""
    from dad_3dheads_b200.evaluator import DADEvaluatorGPU
    gts, sub, st, _, want, z5, K = heads
    missing = {"item003", "item016", "item039"}
    sub = {k: v for k, v in sub.items() if k not in missing}
    json.dump(gts, open(tmp_path / "gt.json", "w"))
    json.dump(sub, open(tmp_path / "sub.json", "w"))
    ev = DADEvaluatorGPU(str(tmp_path / "gt.json"), str(tmp_path / "sub.json"), static=st)
    chunks = []
    inner = ev.metrics

    def spy(annotations, predictions):
        r = inner(annotations, predictions)
        chunks.append(([a["id"] for a in annotations], r))
        return r
    ev.metrics = spy
    capsys.readouterr()
    overall, attrs = ev(batch=16)
    printed = capsys.readouterr().out
    assert sorted(l for l in printed.splitlines() if l.startswith("No prediction")) == \
        sorted(f"No prediction with ID: {i}." for i in missing)
    kept = [i for i, a in enumerate(gts) if a["id"] not in missing]
    assert [len(ids) for ids, _ in chunks] == [16, 16, 5]
    assert [i for ids, _ in chunks for i in ids] == [gts[i]["id"] for i in kept]
    # the chunked per-head values are the ones the means are made of, exactly
    per = {n: np.concatenate([r[n] for _, r in chunks]).astype(np.float64) for n in ORACLE}
    # ... and each is the head's own: pose / NME / chamfer against the oracle, Z5 against the model
    ref = {n: np.array([want[i][ORACLE[n]] for i in kept]) for n in TOL}
    ref["z5"] = (z5.sum(1).double() / (K * 5)).numpy()[kept]
    tol = dict(TOL, z5=(1e-6, 0.0))
    for n, out in ORACLE.items():
        rt, at = tol[n]
        assert overall[out] == np.mean([float(v) for v in per[n]]), n
        assert abs(overall[out] - ref[n].mean()) <= rt * abs(ref[n].mean()) + at, (n, overall[out], ref[n].mean())
        groups = defaultdict(lambda: defaultdict(list))
        for j, i in enumerate(kept):
            for name, value in gts[i]["attributes"].items():
                groups[name][value].append(j)
        assert {k: set(v) for k, v in attrs[out].items()} == {k: set(v) for k, v in groups.items()}
        for name, d in groups.items():
            for value, js in d.items():
                assert attrs[out][name][value] == np.mean([float(per[n][j]) for j in js]), (n, name, value)
                w = ref[n][js].mean()
                assert abs(attrs[out][name][value] - w) <= rt * abs(w) + at, (n, name, value)
