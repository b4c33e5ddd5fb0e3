"""Exact fp32 model of the benchmark evaluator's kernels (csrc/evaluator.cu, and the landmark gathers of csrc/flame.cu), in
torch on the CPU, plus the seeded inputs the GPU tests feed both of them.

What it restates, in kernel order:
- align_kernel: out[c] = fmaf(s, fmaf(x, R[c], fmaf(y, R[3+c], z * R[6+c])), t[c]).  Bit-exact.
- gather_kernel / gather_bary_kernel: a copy, and acc = fmaf(bary[3l+k], src[tri[3l+k]], acc) for k = 0, 1, 2 from
  acc = 0.  Bit-exact.
- chamfer_kernel: per point of a, the fminf of fmaf(dx, dx, fmaf(dy, dy, dz * dz)) over b, dx = ax - bx in fp32; per
  256-point block the xor-butterfly over 32 lanes (lanes past na add 0), the 8 warp sums added in order from 0, then
  s / (float)na.  The blocks' atomicAdd onto out[head] has no fixed order, so the model returns the per-block terms.
- zn_kernel, per column c = j + 1: key[k] = sqrtf(fmaxf(n2 + cn - 2 * dot, 0)) with n2, cn, dot fmaf chains and
  key[c] = 0; (key, index) sorted ascending (the kernel's padding keys are FLT_MAX, past every finite key); the count of
  i with (G[i].z >= G[order[i]].z) == (P[i].z >= P[order[i]].z).  2 * dot is exact, so it does not matter whether nvcc
  contracts the subtraction into an fma.  The library is built without --use_fast_math (csrc/Makefile), so sqrtf and
  the divisions are IEEE correctly rounded on the device.  torch's fp32 sqrt on the CPU is not (it is off by one ulp
  on about 1 in 140 inputs), so the model takes sqrt and / in fp64 and rounds once to fp32: correctly rounded for
  binary32, as 53 >= 2 * 24 + 2.

fmaf is tests/decode_model.fmaf (correctly rounded).  `Mutation` switches in the errors the exact GPU tests must be able
to see (tests/test_eval_model_cpu.py shows that each one changes an output those tests compare).
"""
from __future__ import annotations

import dataclasses
import math
from typing import Tuple

import torch

from tests.decode_model import fmaf

FLT_MAX = 3.4028234663852886e38
U = 2.0 ** -24                     # fp32 unit roundoff
CHAMFER_BLOCK = 256
CHAMFER_TILE = 1024                # b points per shared-memory tile


@dataclasses.dataclass(frozen=True)
class Mutation:
    zn_rowwise: bool = False        # neighbours of point i (row-wise sort) instead of the column quirk
    zn_cols_from_0: bool = False    # columns 0..top_k-1 instead of 1..top_k
    zn_ties_desc: bool = False      # equal keys ordered by descending index
    zn_no_self_zero: bool = False   # key[c] left as computed instead of forced to 0
    zn_strict: bool = False         # '>' instead of '>='
    chamfer_drop_tail: bool = False  # the last partial 1024-point tile of b skipped
    chamfer_div_nb: bool = False    # block sum divided by nb instead of na
    align_transposed: bool = False  # R[3c + r] instead of R[3r + c]


NONE = Mutation()


def sqrtf(x: torch.Tensor) -> torch.Tensor:
    return torch.sqrt(x.double()).float()


def divf(x: torch.Tensor, y: float) -> torch.Tensor:
    return (x.double() / float(y)).float()


# --------------------------------------------------------------------------------------------------------------- align
def align(v: torch.Tensor, scale: torch.Tensor, rot: torch.Tensor, trans: torch.Tensor, mut: Mutation = NONE) -> torch.Tensor:
    """v [B,nv,3], scale [B], rot [B,3,3] (row-vector convention, row-major), trans [B,3] -> [B,nv,3]."""
    B = v.shape[0]
    R = (rot.transpose(1, 2) if mut.align_transposed else rot).reshape(B, 9)[:, None, :]
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    out = [fmaf(scale[:, None], fmaf(x, R[..., c], fmaf(y, R[..., 3 + c], z * R[..., 6 + c])), trans[:, None, c])
           for c in range(3)]
    return torch.stack(out, -1)


# ------------------------------------------------------------------------------------------------------------- gathers
def gather(src: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    return src[:, idx.long()].clone()


def gather_bary(src: torch.Tensor, tri: torch.Tensor, bary: torch.Tensor) -> torch.Tensor:
    """src [B,nv,nc], tri [L,3], bary [L,3] fp32 -> [B,L,nc]."""
    tri = tri.long()
    acc = torch.zeros(src.shape[0], tri.shape[0], src.shape[2])
    for k in range(3):
        acc = fmaf(bary[None, :, k, None].float(), src[:, tri[:, k]], acc)
    return acc


# ------------------------------------------------------------------------------------------------------------- chamfer
def chamfer_minima(a: torch.Tensor, b: torch.Tensor, mut: Mutation = NONE) -> torch.Tensor:
    """a [B,na,3], b [B,nb,3] -> [B,na] per-point minima (FLT_MAX when no b point is visited)."""
    B, na, _ = a.shape
    nb = b.shape[1]
    if mut.chamfer_drop_tail and nb % CHAMFER_TILE:
        nb -= nb % CHAMFER_TILE
    best = torch.full((B, na), FLT_MAX, dtype=torch.float32)
    if nb == 0:
        return best
    rows = max(1, (1 << 22) // (B * nb))
    bx, by, bz = (b[:, None, :nb, k] for k in range(3))
    for i0 in range(0, na, rows):
        ai = a[:, i0:i0 + rows]
        dx, dy, dz = (ai[:, :, None, k] - bb for k, bb in enumerate((bx, by, bz)))
        best[:, i0:i0 + rows] = fmaf(dx, dx, fmaf(dy, dy, dz * dz)).min(-1).values
    return best


def chamfer_terms(a: torch.Tensor, b: torch.Tensor, mut: Mutation = NONE) -> torch.Tensor:
    """[B, n_blocks]: what each 256-point block atomically adds onto out[head]."""
    B, na, _ = a.shape
    nblk = -(-na // CHAMFER_BLOCK)
    v = torch.zeros(B, nblk * CHAMFER_BLOCK)
    v[:, :na] = chamfer_minima(a, b, mut)
    v = v.view(B, nblk, CHAMFER_BLOCK // 32, 32)
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    s = torch.zeros(B, nblk)
    for w in range(CHAMFER_BLOCK // 32):
        s = s + v[..., w, 0]
    return divf(s, b.shape[1] if mut.chamfer_div_nb else na)


def chamfer_bound(terms: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(exact sum, bound) per head: an fp32 sum of n terms in any order lies within (n - 1) u sum|term| of the exact sum
    (Jeannerod & Rump, 2013).  One block gives bound 0: a single atomicAdd onto zero is exact."""
    t = terms.double()
    return t.sum(1), (terms.shape[1] - 1) * U * t.abs().sum(1)


# ----------------------------------------------------------------------------------------------------------------- Z_n
def _keys(G: torch.Tensor, cols: torch.Tensor, mut: Mutation) -> torch.Tensor:
    """[B, m, K]: key of every point k for each centre point cols[m]."""
    C = G[:, cols]
    cx, cy, cz = (C[..., k, None] for k in range(3))
    x, y, z = (G[:, None, :, k] for k in range(3))
    cn = fmaf(cx, cx, fmaf(cy, cy, cz * cz))
    n2 = fmaf(x, x, fmaf(y, y, z * z))
    dot = fmaf(x, cx, fmaf(y, cy, z * cz))
    key = sqrtf(torch.clamp_min((n2 + cn) - 2.0 * dot, 0.0))
    if not mut.zn_no_self_zero:
        key[:, torch.arange(cols.numel()), cols] = 0.0
    return key


def _order(key: torch.Tensor, mut: Mutation) -> torch.Tensor:
    """Indices sorted by (key, index) ascending, or by (key, -index) under zn_ties_desc."""
    if mut.zn_ties_desc:
        K = key.shape[-1]
        return K - 1 - torch.sort(key.flip(-1), dim=-1, stable=True).indices
    return torch.sort(key, dim=-1, stable=True).indices


def zn_counts(pred: torch.Tensor, gt: torch.Tensor, top_k: int, mut: Mutation = NONE) -> torch.Tensor:
    """pred, gt [B,K,3] -> [B, top_k] int64: the agreement count of each column's block."""
    B, K, _ = gt.shape
    cols = torch.arange(top_k) + (0 if mut.zn_cols_from_0 else 1)
    if mut.zn_rowwise:
        nbr = _order(_keys(gt, torch.arange(K), mut), mut)[:, :, cols].transpose(1, 2)      # [B, top_k, K]
    else:
        nbr = _order(_keys(gt, cols, mut), mut)
    cmp = torch.gt if mut.zn_strict else torch.ge
    gz, pz = gt[..., 2], pred[..., 2]
    g = cmp(gz[:, None, :].expand_as(nbr), torch.gather(gz[:, None, :].expand_as(nbr), 2, nbr))
    p = cmp(pz[:, None, :].expand_as(nbr), torch.gather(pz[:, None, :].expand_as(nbr), 2, nbr))
    return (g == p).sum(-1)


def zn_value(counts: torch.Tensor, K: int) -> torch.Tensor:
    """[B] fp32: the columns' terms float(count) / (float(K) * float(top_k)) added in column order.  The kernel adds them
    with atomics in any order; as every term is non-negative, two orders differ by at most top_k - 1 ulps."""
    top_k = counts.shape[1]
    t = divf(counts.float(), K * top_k)
    s = torch.zeros(counts.shape[0])
    for j in range(top_k):
        s = s + t[:, j]
    return s


def ulp(x: torch.Tensor) -> torch.Tensor:
    """fp32 ulp of |x| (x normal or zero)."""
    x = x.float().abs()
    return (torch.nextafter(x, torch.tensor(math.inf)) - x).double()


# -------------------------------------------------------------------------------------------------------------- inputs
# the shapes the GPU tests run; the CPU tests show every mutation is visible on exactly these inputs
ALIGN_NV, ALIGN_B = (1, 7, 5023), (1, 3, 257)
CHAMFER_NA = (1, 31, 255, 256, 257, 2094)          # one block up to 256 points
CHAMFER_NB = (1, 1023, 1024, 1025, 2048, 5023)     # around the 1024-point tiles
CHAMFER_B = (1, 5)
ZN_KINDS = ("random", "lattice", "duplicate")
ZN_K = ("top_k+1", 25, 26, 1023, 1024, 1025, 3669, 4095, 4096)   # 25 / 26: torch.cdist's switch to the mm formula
ZN_TOP_K = (1, 5, 16)


def zn_k(K, top_k: int) -> int:
    return top_k + 1 if K == "top_k+1" else K


def align_case(nv: int, B: int):
    return align_inputs(nv, B, seed=nv * 1000 + B)


def chamfer_case(na: int, nb: int, B: int):
    return chamfer_inputs(na, nb, B, seed=na * 10007 + nb * 10 + B)


def zn_case(kind: str, K: int, top_k: int, B: int = 2):
    return zn_inputs(kind, K, B, top_k, seed=K * 100 + top_k * 7 + ZN_KINDS.index(kind))


def align_inputs(nv: int, B: int, seed: int):
    """Vertices around 1, scales with a zero and a negative one, rotations and reflections, translations around 1e3."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(B, nv, 3, generator=g)
    scale = torch.randn(B, generator=g) * 2.0
    scale[0] = 0.0
    if B > 1:
        scale[1] = -abs(scale[1].item()) - 0.5
    q, _ = torch.linalg.qr(torch.randn(B, 3, 3, generator=g, dtype=torch.float64))
    q[0::2, :, 0] *= torch.where(torch.linalg.det(q[0::2]) > 0, -1.0, 1.0).to(q.dtype)[:, None]    # det -1: reflections
    rot = q.float()
    trans = torch.randn(B, 3, generator=g) * 1e3
    return v, scale, rot, trans


def chamfer_inputs(na: int, nb: int, B: int, seed: int):
    """Different points per head; every 7th point of a coincides with a point of b."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(B, na, 3, generator=g) * 10.0 + 5.0
    b = torch.randn(B, nb, 3, generator=g) * 10.0 + 5.0
    pick = torch.randint(0, nb, (B, (na + 6) // 7), generator=g)
    a[:, ::7] = torch.gather(b, 1, pick[..., None].expand(-1, -1, 3))
    return a, b


def zn_inputs(kind: str, K: int, B: int, top_k: int, seed: int):
    """'random': normal points, pred = gt + noise.  'lattice': small integers (fp32 distances exact, ties and equal z
    everywhere), pred an independent lattice.  'duplicate': random, with points 1 and top_k copied to indices 0 and
    top_k - 1, so each of those columns has a zero-distance twin at a lower index."""
    g = torch.Generator().manual_seed(seed)
    if kind == "lattice":
        gt = torch.randint(-3, 4, (B, K, 3), generator=g).float()
        pred = torch.randint(-3, 4, (B, K, 3), generator=g).float()
        return pred, gt
    gt = torch.randn(B, K, 3, generator=g)
    pred = gt + 0.3 * torch.randn(B, K, 3, generator=g)
    if kind == "duplicate":
        gt[:, 0] = gt[:, 1]
        if top_k >= 3:
            gt[:, top_k - 1] = gt[:, top_k]
    else:
        assert kind == "random", kind
    return pred, gt


def separated_points(K: int, top_k: int, seed: int, gap: float = 3e-5) -> torch.Tensor:
    """[K,3] normal points whose squared distances to each of the points 1..top_k differ pairwise by more than `gap`, so
    that any evaluation of the distances with fp32 rounding (torch.cdist's included, whose error in the squared distance
    is about 1e-6 here) orders them the same way."""
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(4 * K, 3, generator=g, dtype=torch.float32)
    keep = torch.ones(4 * K, dtype=torch.bool)
    changed = True
    while changed:
        changed = False
        p = pts[keep].double()
        idx = keep.nonzero()[:, 0]
        for c in range(1, top_k + 1):
            d2 = ((p - p[c]) ** 2).sum(1)
            s, o = torch.sort(d2)
            close = (s[1:] - s[:-1]) <= gap
            drop = torch.maximum(o[1:][close], o[:-1][close])       # the later point of each close pair: when that is
            if drop.numel():                                       # a centre, the next kept point takes its place
                keep[idx[drop]] = False
                changed = True
                break
    out = pts[keep][:K]
    assert out.shape[0] == K
    for c in range(1, top_k + 1):
        s = torch.sort(((out.double() - out[c].double()) ** 2).sum(1)).values
        assert (s[1:] - s[:-1]).min() > gap
    return out
