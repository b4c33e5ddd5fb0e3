"""-m gpu: the training losses (dad_3dheads_b200.losses, csrc/loss.cu) against the reference's own loss classes and
LossModule, loaded from the pinned harness (oracle/ref_harness.py) and run on the CPU in fp64 under autograd.

Bounds: loss values relative <= 1e-5; heat-map and landmark gradients relL2 <= 1e-5; 3DMM parameter gradients relL2 < 1e-4 per
parameter group (the bound of test_backward_gpu.py).  Targets come from other seeded parameters plus noise, so differences
fall on both smooth-L1 branches.  Two things would make an fp32 / fp64 comparison flaky rather than wrong, and the inputs are
built so they cannot happen: an l1 difference within rounding of its kink at 0 (targets are nudged until every difference is
clear of it), and near-ties at normalize_to_cube's reductions (heads are drawn until every head has a relative gap of at least
1e-4 between its first and second extreme at each reduction; the tie rule itself is checked on exact ties)."""
import functools
import os

import pytest
import torch

from oracle import ref_harness as R
from oracle.flame_oracle import FLAME_CONSTS, sample_params

pytestmark = pytest.mark.gpu

GROUPS = {"shape": (0, 300), "expression": (300, 400), "jaw": (400, 403), "rotation": (403, 409), "translation": (409, 412),
          "scale": (412, 413)}
FILES = {"head": "head.npy", "face_w_ears": "face_w_ears.npy", "face": "face.npy"}
V_WEIGHTS = {"head": .5, "face_w_ears": .75, "face": 1.}        # config/loss/train_loss.yaml
P_WEIGHTS = {"face": .5, "face_w_ears": .5}
CRITERIA = ("l1", "l2", "smooth_l1")
GAP = 1e-4


def _weights_and_indices(weights):
    if not R.available():
        pytest.skip("reference harness not available")
    folder = os.path.join(R.root(), "model_training", "model", "static", "flame_indices")
    return {"flame_indices": {"folder": folder, "files": dict(FILES)}, "weights": dict(weights)}


def _ref():
    R.activate()
    import model_training.losses as L
    return L


def _fp64(loss):
    loss.head_mesh.to(torch.float64)
    loss.head_mesh.flame.dtype = torch.float64
    return loss


def _rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return ((a - b).norm() / b.norm()).item()


def _check_param_grad(got, want):
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    for name, (a, b) in GROUPS.items():
        w, q = want[:, a:b], got[:, a:b]
        if w.norm().item() == 0:
            assert q.norm().item() == 0, name
        else:
            assert ((q - w).norm() / w.norm()).item() < 1e-4, (name, ((q - w).norm() / w.norm()).item())


def _normalize(v):
    """normalize_to_cube (model/utils.py:55-68) in fp64, with the centred values and the reductions' winners."""
    mn, amin = v.min(1, True)
    v1 = v - mn
    mx, amax = v1.max(1, True)
    v2 = v1 - 0.5 * mx
    return v2, amin, amax


def _gaps(v, sets):
    """Per head, the smallest relative gap between first and second extreme over every reduction of every set."""
    out = torch.full((v.shape[0],), float("inf"), dtype=torch.float64)
    for idx in sets:
        x = v[:, idx]
        rng = (x.max(1)[0] - x.min(1)[0])                                             # [B, 3]
        lo = x.topk(2, dim=1, largest=False)[0]
        out = torch.minimum(out, ((lo[:, 1] - lo[:, 0]) / rng).min(1)[0])
        v1 = x - lo[:, :1]
        hi = v1.topk(2, dim=1)[0]
        out = torch.minimum(out, ((hi[:, 0] - hi[:, 1]) / rng).min(1)[0])
        v2 = (v1 - 0.5 * hi[:, :1]).reshape(v.shape[0], -1)
        top = v2.topk(2, dim=1)[0]
        out = torch.minimum(out, (top[:, 0] - top[:, 1]) / top[:, 0])
    return out


def _clear_l1_kinks(pred, target, sets, normalize, delta):
    """Nudge fp32 target entries until every per-set difference of ``pred`` (fp64) and ``target`` is at least ``delta`` away
    from 0 (the l1 kink), so a rounding-sized difference between fp32 and fp64 cannot flip a sign.  A vertex in several
    sets is normalised differently in each, so the nudges have random sizes and signs: a fixed rule can oscillate."""
    g = torch.Generator().manual_seed(0)
    t = target.clone()
    for _ in range(50):
        bad = torch.zeros_like(t, dtype=torch.bool)
        size = torch.zeros_like(t, dtype=torch.float64)
        for idx in sets:
            u, w = pred[:, idx], t.double()[:, idx]
            if normalize:
                (u, _, _), (w2, _, _) = _normalize(u), _normalize(w)
                M = u.reshape(u.shape[0], -1).max(1)[0][:, None, None]
                Mt = w2.reshape(w2.shape[0], -1).max(1)[0][:, None, None]
                u, w = u / M, w2 / Mt
                scale = Mt.expand_as(w)
            else:
                scale = torch.ones_like(w)
            # where both operands are normalised to exactly +-1 (an extreme of the overall-max coordinate in both), d is
            # exact in either precision
            near = ((u - w).abs() < delta) & ~((u.abs() == 1) & (w.abs() == 1))
            bad[:, idx] |= near
            size[:, idx] = torch.maximum(size[:, idx], torch.where(near, delta * scale, 0.0))
        if not bad.any():
            return t
        step = (3 + 7 * torch.rand(t.shape, generator=g, dtype=torch.float64)) * size
        sign = torch.where(torch.rand(t.shape, generator=g) < 0.5, -1.0, 1.0).double()
        t = (t.double() + sign * step).float()
    raise AssertionError("could not clear the l1 kinks")


@functools.lru_cache(maxsize=None)
def _heads(B, seed):
    """B heads whose fp64 zero-rotation vertices have every normalize_to_cube reduction separated by GAP, over the loss
    subsets; and fp64 vertices / 2D projections of other (seeded, nearby) parameters for targets."""
    L = _ref()
    from model_training.model.flame import FLAME_CONSTS as C
    wi = _weights_and_indices(V_WEIGHTS)
    vl = _fp64(L.Vertices3DLoss("l2", B, C, wi))
    sets = [torch.as_tensor(i) for i in vl.indices]
    keep, n, s = [], 0, seed
    while n < B:
        p = sample_params(max(B, 8) * 2, seed=s)
        s += 1000
        with torch.no_grad():
            v = vl.head_mesh.vertices_3d(p.double(), zero_rotation=True)
        ok = _gaps(v, sets) >= GAP
        keep.append(p[ok])
        n += int(ok.sum())
    p = torch.cat(keep)[:B]
    with torch.no_grad():
        v = vl.head_mesh.vertices_3d(p.double(), zero_rotation=True)
        assert (_gaps(v, sets) >= GAP).all()
        g = torch.Generator().manual_seed(seed + 1)
        other = p + 0.3 * torch.randn(p.shape, generator=g)
        hm = _fp64(L.ReprojectionLoss("l2", B, C, 256, _weights_and_indices(P_WEIGHTS))).head_mesh
        tv = hm.vertices_3d(other.double(), zero_rotation=True)
        tp = hm.reprojected_vertices(other.double().clone(), to_2d=True)
        big = (torch.rand(tv.shape, generator=g) < 0.05).double()
        tv = (tv + 0.002 * torch.randn(tv.shape, generator=g, dtype=torch.float64) * (1 + 20 * big)).float()
        tp = (tp + 1.5 * torch.randn(tp.shape, generator=g, dtype=torch.float64)).float()
    return p, tv, tp


def _subsets(loss):
    return [torch.as_tensor(i) for i in loss.indices]


@pytest.mark.parametrize("criterion", CRITERIA)
@pytest.mark.parametrize("B", [1, 3, 64, 4133])
def test_vertices3d_loss_matches_reference(cuda_device, B, criterion):
    from dad_3dheads_b200.losses import Vertices3DLoss
    L = _ref()
    wi = _weights_and_indices(V_WEIGHTS)
    ref = _fp64(L.Vertices3DLoss(criterion, B, FLAME_CONSTS, wi))
    p, tv, _ = _heads(B, 11)
    if criterion == "l1":
        with torch.no_grad():
            v = ref.head_mesh.vertices_3d(p.double(), zero_rotation=True)
        tv = _clear_l1_kinks(v, tv, _subsets(ref), True, 1e-4)
    q = p.double().clone().requires_grad_(True)
    want = ref(q * 1.0, tv.double())
    want.backward()
    mine = Vertices3DLoss(criterion, B, FLAME_CONSTS, wi)
    x = p.to(cuda_device).requires_grad_(True)
    got = mine(x * 1.0, tv.to(cuda_device))
    got.backward()
    assert abs(got.item() - want.item()) <= 1e-5 * abs(want.item()), (got.item(), want.item())
    _check_param_grad(x.grad, q.grad)


@pytest.mark.parametrize("criterion", CRITERIA)
@pytest.mark.parametrize("B", [1, 3, 64, 4133])
def test_reprojection_loss_matches_reference(cuda_device, B, criterion):
    from dad_3dheads_b200.losses import ReprojectionLoss
    L = _ref()
    wi = _weights_and_indices(P_WEIGHTS)
    ref = _fp64(L.ReprojectionLoss(criterion, B, FLAME_CONSTS, 256, wi))
    p, _, tp = _heads(B, 11)
    if criterion == "l1":
        with torch.no_grad():
            pj = ref.head_mesh.reprojected_vertices(p.double().clone(), to_2d=True)
        tp = _clear_l1_kinks(pj, tp, _subsets(ref), False, 1e-2)
    q = p.double().clone().requires_grad_(True)
    qa = q * 1.0
    if B == 3:
        # the reference's rot_mat_from_6dof takes torch.cross over the first axis of size 3, the batch axis when B == 3;
        # the package takes it over the last axis for every B (DESIGN.md).  A mean over heads is the mean of one-head means.
        want = torch.stack([ref(qa[b:b + 1], [tp.double()[b:b + 1]]) for b in range(B)]).mean()
    else:
        want = ref(qa, [tp.double()])
    want.backward()
    mine = ReprojectionLoss(criterion, B, FLAME_CONSTS, 256, wi)
    x = p.to(cuda_device).requires_grad_(True)
    xa = x * 1.0
    got = mine(xa, [tp.to(cuda_device)])
    got.backward()
    assert abs(got.item() - want.item()) <= 1e-5 * abs(want.item()), (got.item(), want.item())
    _check_param_grad(x.grad, q.grad)
    assert (xa[:, 411] == 0).all() and (qa[:, 411] == 0).all()                   # translation z zeroed in place, as in the reference


def _heatmaps(B, seed, C=68, H=64):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, H, generator=g) * 3
    cy, cx = torch.rand(B, C, 1, 1, generator=g) * H, torch.rand(B, C, 1, 1, generator=g) * H
    yy, xx = torch.arange(H).view(1, 1, H, 1).float(), torch.arange(H).view(1, 1, 1, H).float()
    t = torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * 2.0 ** 2))
    return x, t


@pytest.mark.parametrize("B", [1, 3, 64])
def test_iou_loss_matches_reference(cuda_device, B):
    from dad_3dheads_b200.losses import IoULoss
    x, t = _heatmaps(B, 5 + B)
    q = x.double().requires_grad_(True)
    want = _ref().IoULoss()(q, t.double())
    want.backward()
    xd = x.to(cuda_device).requires_grad_(True)
    got = IoULoss()(xd, t.to(cuda_device))
    got.backward()
    assert abs(got.item() - want.item()) <= 1e-5 * abs(want.item()), (got.item(), want.item())
    assert _rel(xd.grad, q.grad) <= 1e-5


def _landmarks(B, seed, N=68):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(B, N, 2, generator=g) * 64
    t = p + torch.randn(B, N, 2, generator=g) * 1.5
    pm = (torch.rand(B, N, generator=g) < 0.8).float()
    tm = torch.where(torch.rand(B, N, generator=g) < 0.9, pm, 1 - pm)
    return p, pm, t, tm


@pytest.mark.parametrize("criterion", CRITERIA)
@pytest.mark.parametrize("B", [1, 3, 64])
def test_landmarks_loss_matches_reference(cuda_device, B, criterion):
    from dad_3dheads_b200.losses import LandmarksLossWVisibility
    p, pm, t, tm = _landmarks(B, 21 + B)
    q = p.double().requires_grad_(True)
    want = _ref().LandmarksLossWVisibility(criterion)([q, pm.double()], [t.double(), tm.double()])
    want.backward()
    pd = p.to(cuda_device).requires_grad_(True)
    got = LandmarksLossWVisibility(criterion)([pd, pm.to(cuda_device)], [t.to(cuda_device), tm.to(cuda_device)])
    got.backward()
    assert abs(got.item() - want.item()) <= 1e-5 * abs(want.item()), (got.item(), want.item())
    assert _rel(pd.grad, q.grad) <= 1e-5


@pytest.mark.parametrize("criterion", CRITERIA)
def test_normalize_ties_go_to_the_first_extreme(cuda_device, criterion):
    """Exact ties at all three reductions of normalize_to_cube (min, max, and the overall max over vertex then coordinate),
    on vertex-space inputs through nested sets with a repeated index: loss and gradient match the reference's function in
    fp64 autograd, which routes each reduction's gradient to the first extreme."""
    from dad_3dheads_b200.losses import VertexSubsets, vertex_subset_loss
    R.activate()
    from model_training.model.utils import normalize_to_cube
    g = torch.Generator().manual_seed(3)
    B, V = 2, 40
    v = (torch.randint(-8, 9, (B, V, 3), generator=g).float() / 8)
    # x and y both span [-1.5, 2.5], z spans [-1, 1]: ties at the minima (vertices 0, 2 in x; 0, 3 in y; many in z), at the
    # maxima (1, 3, 5 in x; 1, 2, 5 in y), and at the overall maximum across vertices (1, 5) and coordinates (x, y of 1 and 5)
    v[:, :6] = torch.tensor([[-1.5, -1.5, -1.0], [2.5, 2.5, 1.0], [-1.5, 2.5, 1.0], [2.5, -1.5, -1.0], [0.0, 0.0, 0.0],
                             [2.5, 2.5, 1.0]])
    t = torch.randn(B, V, 3, generator=g) * 0.7
    sets = [torch.arange(0, 40), torch.tensor([0, 1, 2, 3, 5, 6, 7, 1]), torch.arange(0, 12)]    # nested, index 1 twice
    weights = [0.5, 0.75, 1.0]
    sub = VertexSubsets([s.numpy() for s in sets], weights, V)
    crit = {"l1": torch.nn.L1Loss(), "l2": torch.nn.MSELoss(), "smooth_l1": torch.nn.SmoothL1Loss()}[criterion]
    q = v.double().requires_grad_(True)
    want = torch.stack([crit(*map(normalize_to_cube, (q[:, i], t.double()[:, i]))) * w for w, i in zip(weights, sets)]).sum()
    want.backward()
    vd = v.to(cuda_device).requires_grad_(True)
    got = vertex_subset_loss(vd, t.to(cuda_device), sub, criterion, normalize=True)
    got.backward()
    assert abs(got.item() - want.item()) <= 1e-5 * abs(want.item())
    assert _rel(vd.grad, q.grad) <= 1e-5, _rel(vd.grad, q.grad)


# ---- the whole objective: train_loss.yaml through the reference's LossModule ------------------------------------------
def _objective_inputs(B, seed):
    p, tv, tp = _heads(B, seed)
    x, th = _heatmaps(B, seed)
    lm, pres, lt, _ = _landmarks(B, seed)
    return p, tv, tp, x, th, lm, lt, pres


def _loss_module(classes, to_fp64=None):
    R.activate()
    from model_training.data import config as K
    from model_training.train.loss_module import LossModule
    vl = classes.Vertices3DLoss("l2", 8, FLAME_CONSTS, _weights_and_indices(V_WEIGHTS))
    rl = classes.ReprojectionLoss("smooth_l1", 8, FLAME_CONSTS, 256, _weights_and_indices(P_WEIGHTS))
    if to_fp64:
        vl, rl = to_fp64(vl), to_fp64(rl)
    crits = [classes.IoULoss(), vl, rl, classes.LandmarksLossWVisibility("smooth_l1")]
    return K, LossModule(names=["heatmap_loss", "vertices3d_loss", "reprojection_loss", "landmarks_loss"],
                         output_keys=[K.OUTPUT_LANDMARKS_HEATMAP, K.OUTPUT_3DMM_PARAMS, K.OUTPUT_3DMM_PARAMS,
                                      [K.OUTPUT_2D_LANDMARKS, K.TARGET_2D_LANDMARKS_PRESENCE]],
                         target_keys=[K.TARGET_LANDMARKS_HEATMAP, K.TARGET_3D_MODEL_VERTICES, K.TARGET_2D_FULL_LANDMARKS,
                                      [K.TARGET_2D_LANDMARKS, K.TARGET_2D_LANDMARKS_PRESENCE]],
                         criterions=crits, weights=[1., 50., 0.05, 100.], schedule=[0, 0, 0, 0], reduction="sum")


def _run(module, K, p, tv, tp, x, th, lm, lt, pres, device, dtype):
    cast = lambda a: a.to(device=device, dtype=dtype)
    leaves = [cast(a).requires_grad_(True) for a in (x, p, lm)]
    params = leaves[1] * 1.0                                   # a network output: not a leaf
    preds = {K.OUTPUT_LANDMARKS_HEATMAP: leaves[0], K.OUTPUT_3DMM_PARAMS: params, K.OUTPUT_2D_LANDMARKS: leaves[2]}
    targets = {K.TARGET_LANDMARKS_HEATMAP: cast(th), K.TARGET_3D_MODEL_VERTICES: cast(tv), K.TARGET_2D_FULL_LANDMARKS: cast(tp),
               K.TARGET_2D_LANDMARKS: cast(lt), K.TARGET_2D_LANDMARKS_PRESENCE: cast(pres)}
    total, parts = module(preds, targets, epoch=0)
    grads = torch.autograd.grad(total, leaves)
    return total, parts, grads, params


def _mine():
    import dad_3dheads_b200.losses as M
    return _loss_module(M)


def test_loss_module_drop_in(cuda_device):
    B = 8
    inputs = _objective_inputs(B, 41)
    K, ref = _loss_module(_ref(), _fp64)
    want, want_parts, want_g, want_p = _run(ref, K, *inputs, "cpu", torch.float64)
    K, mine = _mine()
    got, got_parts, got_g, got_p = _run(mine, K, *inputs, cuda_device, torch.float32)
    assert list(got_parts) == list(want_parts)
    for k in want_parts:
        assert abs(got_parts[k].item() - want_parts[k].item()) <= 1e-5 * abs(want_parts[k].item()), k
    assert abs(got.item() - want.item()) <= 1e-5 * abs(want.item())
    assert _rel(got_g[0], want_g[0]) <= 1e-5 and _rel(got_g[2], want_g[2]) <= 1e-5
    _check_param_grad(got_g[1], want_g[1])
    assert (got_p[:, 411] == 0).all() and (want_p[:, 411] == 0).all()


def _bits(*ts):
    return [t.detach().cpu().view(torch.int32) if t.dtype == torch.float32 else t.detach().cpu() for t in ts]


def test_determinism_and_head_permutation(cuda_device):
    B = 64
    K, mine = _mine()
    inputs = _objective_inputs(B, 43)
    a = _run(mine, K, *inputs, cuda_device, torch.float32)
    b = _run(mine, K, *inputs, cuda_device, torch.float32)
    assert torch.equal(*_bits(a[0], b[0]))
    for ga, gb in zip(a[2], b[2]):
        assert torch.equal(*_bits(ga, gb))
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(0))
    c = _run(mine, K, *[t[perm] for t in inputs], cuda_device, torch.float32)
    for ga, gc in zip(a[2], c[2]):
        assert torch.equal(*_bits(ga[perm.to(ga.device)], gc))


def test_non_finite_head_is_isolated(cuda_device):
    B = 16
    K, mine = _mine()
    inputs = list(_objective_inputs(B, 47))
    clean = _run(mine, K, *inputs, cuda_device, torch.float32)
    p, x = inputs[0].clone(), inputs[3].clone()
    x[2, 5, 10, 10] = float("nan")
    p[5, 17] = float("nan")
    inputs[0], inputs[3] = p, x
    dirty = _run(mine, K, *inputs, cuda_device, torch.float32)
    others = [h for h in range(B) if h not in (2, 5)]
    for gc, gd in zip(clean[2], dirty[2]):
        assert torch.equal(*_bits(gc[others], gd[others]))
    assert not torch.isfinite(dirty[2][0][2]).all() and not torch.isfinite(dirty[2][1][5]).all()


def test_graph_capture_matches_eager(cuda_device):
    B = 16
    K, mine = _mine()
    first, second = _objective_inputs(B, 51), _objective_inputs(B, 53)
    static = [a.to(cuda_device) for a in first]

    def step():
        total, _, grads, _ = _run(mine, K, *static, cuda_device, torch.float32)
        return (total,) + tuple(grads)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    with torch.no_grad():
        for s, n in zip(static, second):
            s.copy_(n)
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    for a, b in zip(out, eager):
        assert torch.equal(*_bits(a, b))
