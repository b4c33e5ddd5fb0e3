"""-m "not gpu": the training losses' host side (dad_3dheads_b200.losses) and the gradient formulas csrc/loss.cu implements.

- ``from model_training.losses import ...`` resolves through compat/ to the package classes;
- the constructors validate like the reference's;
- the subset tables hold what the reference's ``indices_reweighing`` reads from its own flame_indices files;
- the backward formulas of the kernels, restated in fp64, equal torch autograd of the reference's expressions: the heat-map
  IoU, and normalize_to_cube (model/utils.py:55-68) with exact ties at each of its three reductions, where torch routes the
  gradient to the first extreme."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["Vertices3DLoss", "ReprojectionLoss", "LandmarksLossWVisibility", "IoULoss"]       # losses/__init__.py:6-7


def test_compat_losses_resolve_to_the_package():
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from model_training.losses import Vertices3DLoss, ReprojectionLoss, LandmarksLossWVisibility, IoULoss\n"
        "import model_training.losses as L, dad_3dheads_b200.losses as P\n"
        "assert L.__all__ == %r\n"
        "assert all(getattr(L, n) is getattr(P, n) for n in L.__all__)\n"
        "from model_training.utils import indices_reweighing\n"
        "from dad_3dheads_b200.flame_assets import indices_reweighing as ir\n"
        "assert indices_reweighing is ir\n"
        "print('ok')\n" % (ROOT, os.path.join(ROOT, "compat"), NAMES))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]


def _index_folder(tmp_path):
    np.save(tmp_path / "a.npy", np.array([3, 1, 4, 1, 5], dtype=np.int64))
    np.save(tmp_path / "b.npy", np.array([9, 2, 6], dtype=np.int64))
    return {"flame_indices": {"folder": str(tmp_path), "files": {"a": "a.npy", "b": "b.npy", "c": "c.npy"}},
            "weights": {"b": 0.25, "a": 2.0}}


def test_constructors_validate_like_the_reference(tmp_path):
    from dad_3dheads_b200.flame import FLAME_CONSTS
    from dad_3dheads_b200.losses import IoULoss, LandmarksLossWVisibility, ReprojectionLoss, Vertices3DLoss
    wi = _index_folder(tmp_path)
    makers = [lambda c: LandmarksLossWVisibility(c), lambda c: Vertices3DLoss(c, 4, FLAME_CONSTS, wi),
              lambda c: ReprojectionLoss(c, 4, FLAME_CONSTS, 256, wi)]
    for make in makers:
        with pytest.raises(ValueError, match="^Unsupported discrepancy loss type huber$"):
            make("huber")
        for c in ("l1", "l2", "smooth_l1"):
            make(c)
    IoULoss()
    r = ReprojectionLoss("l1", 4, FLAME_CONSTS, 224, wi)
    assert r.weights == [2.0, 0.25] and [list(i) for i in r.indices] == [[3, 1, 4, 1, 5], [9, 2, 6]]
    assert r.head_mesh._image_size == 224
    assert r.subsets.sizes == [5, 3] and list(r.subsets._off) == [0, 5, 8]


def test_constructor_errors_match_the_reference_classes(tmp_path):
    from oracle import ref_harness as R
    if not R.available():
        pytest.skip("reference tree not available")
    R.activate()
    import model_training.losses as ref
    from dad_3dheads_b200 import losses as mine
    from dad_3dheads_b200.flame import FLAME_CONSTS
    wi = _index_folder(tmp_path)
    cases = {"LandmarksLossWVisibility": ("x",), "Vertices3DLoss": ("x", 4, FLAME_CONSTS, wi),
             "ReprojectionLoss": ("x", 4, FLAME_CONSTS, 256, wi)}
    for name, args in cases.items():
        msgs = []
        for mod in (ref, mine):
            with pytest.raises(ValueError) as e:
                getattr(mod, name)(*args)
            msgs.append(str(e.value))
        assert msgs[0] == msgs[1], (name, msgs)


def test_subset_tables_match_the_reference_reweighing():
    from oracle import ref_harness as R
    if not R.available():
        pytest.skip("reference tree not available")
    R.activate()
    from model_training.utils import indices_reweighing as ref_reweighing
    from dad_3dheads_b200.losses import VertexSubsets
    from dad_3dheads_b200.flame_assets import indices_reweighing
    folder = os.path.join(R.root(), "model_training", "model", "static", "flame_indices")
    files = {"head": "head.npy", "face_w_ears": "face_w_ears.npy", "face": "face.npy"}           # config/dataset/dad_3d_heads.yaml
    for weights in ({"head": .5, "face_w_ears": .75, "face": 1.}, {"face": .5, "face_w_ears": .5}):   # train_loss.yaml
        wi = {"flame_indices": {"folder": folder, "files": files}, "weights": weights}
        rw, ri = ref_reweighing(wi)
        w, i = indices_reweighing(wi)
        assert w == rw and len(i) == len(ri) and all(np.array_equal(a, b) for a, b in zip(i, ri))
        sub = VertexSubsets(i, w, 5023)
        assert np.array_equal(sub._idx, np.concatenate(ri).astype(np.int32))
        assert list(sub._off) == list(np.cumsum([0] + [len(a) for a in ri]))
        assert np.array_equal(sub._w, np.asarray(rw, dtype=np.float32))


def test_subset_tables_reject_bad_sets():
    from dad_3dheads_b200.losses import VertexSubsets
    with pytest.raises(IndexError):
        VertexSubsets([np.array([0, 10])], [1.0], 10)
    with pytest.raises(ValueError):
        VertexSubsets([np.array([], dtype=np.int64)], [1.0], 10)
    with pytest.raises(ValueError):
        VertexSubsets([np.array([1])], [1.0, 2.0], 10)
    assert list(VertexSubsets([np.array([-1, 0])], [1.0], 10)._idx) == [9, 0]


# ---- the kernels' gradient formulas, restated in fp64 ----------------------------------------------------------------------
def _iou_loss(x, t, eps=1e-6):
    """keypoint_losses.py:12-31."""
    s = torch.sigmoid(x)
    op = lambda a: a.reshape(a.shape[0], a.shape[1], -1).sum(2)
    return 1 - ((op(t * s) + eps) / (op(t ** 2) + op(s ** 2) - op(t * s) + eps)).mean()


def _iou_backward(x, t, g, eps=1e-6):
    """iou_backward_kernel: -g / P (t D - N (2 s - t)) / D^2 s (1 - s), N = I + eps, D = T + S - I + eps."""
    B, C = x.shape[:2]
    s = torch.sigmoid(x)
    op = lambda a: a.reshape(B, C, -1).sum(2)[:, :, None, None]
    I, T, S = op(s * t), op(t * t), op(s * s)
    N, D = I + eps, T + S - I + eps
    return -g / (B * C) * (t * D - N * (2 * s - t)) / D ** 2 * s * (1 - s)


def test_iou_backward_formula():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(3, 5, 8, 8, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    t = torch.rand(3, 5, 8, 8, generator=g, dtype=torch.float64)
    t[0, 1] = 0                                                                 # an empty target plane
    (_iou_loss(x, t) * 0.7).backward()
    want = x.grad
    assert torch.allclose(_iou_backward(x.detach(), t, 0.7), want, rtol=1e-12, atol=1e-15)


def _normalize_to_cube(v):
    """model/utils.py:55-68 for [B, N, 3]."""
    v = v - v.min(1, True)[0]
    v = v - 0.5 * v.max(1, True)[0]
    return v / v.max(-1, True)[0].max(-2, True)[0]


def _first(mask, dim):
    return mask.to(torch.int64).argmax(dim)            # first True along dim


def _normalize_backward(v, G):
    """vsub_backward_kernel's routing for one set: d/dv of sum(G * normalize_to_cube(v)), each reduction's gradient going
    to its first extreme (positions, then coordinates within a position for the overall maximum)."""
    B, n, K = v.shape
    mn = v.min(1, True)[0]
    amin = _first(v == mn, 1)                                                   # [B, K]
    v1 = v - mn
    mx = v1.max(1, True)[0]
    amax = _first(v1 == mx, 1)
    v2 = v1 - 0.5 * mx
    flat = v2.reshape(B, -1)
    M = flat.max(1)[0]
    star = _first(flat == M[:, None], 1)
    nstar, cstar = star // K, star % K
    u = v2 / M[:, None, None]
    sco = (G * u).sum((1, 2))
    sg = G.sum(1)                                                               # [B, K]
    dM = -sco / M
    gv = G / M[:, None, None]
    A = -0.5 * (sg / M[:, None] + torch.nn.functional.one_hot(cstar, K) * dM[:, None])
    b = torch.arange(B)
    gv[b, nstar, cstar] += dM
    for c in range(K):
        gv[b, amax[:, c], c] += A[:, c]
        gv[b, amin[:, c], c] += A[:, c]
    return gv


def _tied_vertices():
    g = torch.Generator().manual_seed(1)
    v = torch.randint(-8, 9, (3, 30, 3), generator=g).double() / 8
    # x and y span [-1.5, 2.5], z [-1, 1]: ties at the minima and maxima of every coordinate, and at the overall maximum
    # across vertices (1, 5) and across coordinates (x, y of vertex 1)
    v[:, :6] = torch.tensor([[-1.5, -1.5, -1.0], [2.5, 2.5, 1.0], [-1.5, 2.5, 1.0], [2.5, -1.5, -1.0], [0.0, 0.0, 0.0],
                             [2.5, 2.5, 1.0]], dtype=torch.float64)
    v[2] = v[2].roll(7, dims=0)                                                 # the tied vertices elsewhere in one head
    return v


def test_normalize_backward_formula_with_ties():
    g = torch.Generator().manual_seed(2)
    for v0 in (_tied_vertices(), torch.randn(4, 50, 3, generator=g, dtype=torch.float64)):
        G = torch.randn(v0.shape, generator=g, dtype=torch.float64)
        v = v0.clone().requires_grad_(True)
        (G * _normalize_to_cube(v)).sum().backward()
        assert torch.allclose(_normalize_backward(v0, G), v.grad, rtol=1e-12, atol=1e-13)


def test_tied_vertices_tie_at_every_reduction():
    """The constructed input does exercise all three tie rules."""
    v = _tied_vertices()
    mn = v.min(1, True)[0]
    assert ((v == mn).sum(1) >= 2).all()
    v1 = v - mn
    assert ((v1 == v1.max(1, True)[0]).sum(1) >= 2).all()
    v2 = v1 - 0.5 * v1.max(1, True)[0]
    M = v2.reshape(3, -1).max(1)[0]
    hits = (v2 == M[:, None, None])
    assert (hits.any(2).sum(1) >= 2).all() and (hits.sum(2).max(1)[0] >= 2).all()
