"""Exact model of the FLAME decode paths (csrc/flame.cu, csrc/flame_decode.cuh), in torch so that it runs on the CPU or on
the device, and designed operands on which every path is fully determined.

What it restates, in kernel order:
1. Packing (dad3d_flame_create): the power-of-two basis scale; fp16 round-to-nearest hi/lo split of scale * [shapedirs |
   posedirs^T]; the scaled template as four successive fp16 pieces in columns 436 / 437 as (hi, hi, lo, lo); w_rest = the
   fp32 sum of the lbs weights of joints 0, 1, 3, 4 in that order, w_jaw = the weight of joint 2.
2. Prep rows (flame_prep_kernel): fp16 RN of beta and of beta - hi, coefficient 1.0 in both template columns, zero padding,
   and the dec_phys_row permutation of the dedicated kernel.
3. The product: default path one product hi*hi; hi/lo path acc0 = hi*hi, acc1 = lo*hi + hi*lo (no lo*lo), then
   fp32(acc0 + acc1); SIMT path the sequential fmaf over k of fp32(hi + lo) products.  For the tensor-core paths the
   model asserts, for every output it returns, that each accumulator is summed exactly in fp32 whatever the order or
   truncation: all its terms lie on one power-of-two grid and sum |terms| < 2^24 grid.
4. The epilogues: two-transform skinning fmaf(wj, jx, fmaf(wr, rx, c)) over fmaf chains (dedicated kernel, EpiLbs), the
   five-joint skinning of lbs_project_kernel (joints with w == 0 skipped), and the projection (fmaf(x, sc, t) + 1) * hs
   (dedicated kernel, hs = 0.5 * image_size) or ((fmaf(x, sc, t) + 1) * 0.5) * image_size (EpiLbs, lbs_project_kernel).
fmaf is emulated exactly: the product is exact in fp64, the sum gets a TwoSum error term and is rounded to odd in fp64,
then rounded to fp32 -- correctly rounded for binary32 (53 >= 24 + 2).

`Mutation` switches in the errors the exact tests must be able to see (tests/test_decode_model.py shows that each of them
changes an output the GPU tests compare).
"""
from __future__ import annotations

import dataclasses
from typing import Dict, Optional

import numpy as np
import torch

K = 448                  # coefficient columns: 400 betas, 36 pose features, 2 template columns, padding
N_BETAS = 400
TMPL = 436               # template columns 436, 437
XF = 68                  # floats per transform record
MESH_OFFSET_Z = 0.05


# ------------------------------------------------------------------------------------------------------------ arithmetic
def fmaf(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """Correctly rounded fp32 fused multiply-add of fp32 tensors (any device)."""
    a64, b64, c64 = a.double(), b.double(), c.double()
    p = a64 * b64                                   # exact: 24 + 24 bits
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                 # TwoSum: p + c = s + e exactly
    odd = (s.view(torch.int64) & 1) == 1
    inf = torch.full_like(s, float("inf"))
    s = torch.where((e != 0) & ~odd, torch.nextafter(s, torch.where(e > 0, inf, -inf)), s)    # round to odd
    return s.float()


def grid_of(x: torch.Tensor) -> float:
    """Largest power of two that divides every non-zero element (inf for an all-zero tensor)."""
    a = x.double().abs()
    a = a[a != 0]
    if a.numel() == 0:
        return float("inf")
    m, e = torch.frexp(a)
    mi = (m * 2.0 ** 53).to(torch.int64)
    low = mi & -mi
    return float(torch.ldexp(low.double(), (e - 53).double()).min())


def f16(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> fp16 round-to-nearest-even, back as fp32."""
    return x.float().half().float()


# ---------------------------------------------------------------------------------------------------------------- packing
def basis_scale(shapedirs: np.ndarray, posedirs: np.ndarray, v_template: np.ndarray) -> float:
    """dad3d_flame_create: scaled basis amax in [512, 1024), exponent clamped to [-8, 24], scale * |T| < 2^15."""
    amax = max(float(np.abs(shapedirs).max()), float(np.abs(posedirs).max()))
    tmax = float(np.abs(v_template).max())
    e = 0
    if amax > 0:
        e = min(max(10 - int(np.frexp(np.float32(amax))[1]), -8), 24)
    if tmax > 0:
        e = min(e, 15 - int(np.frexp(np.float32(tmax))[1]))
    return float(2.0 ** e)


@dataclasses.dataclass
class Packed:
    scale: float
    hi: torch.Tensor         # [3 nv, 448] fp32 values of the fp16 hi plane
    lo: torch.Tensor         # [3 nv, 448] lo plane
    w2: torch.Tensor         # [nv, 2] (w_rest, w_jaw) fp32
    weights: torch.Tensor    # [nv, 5] fp32

    def to(self, device) -> "Packed":
        return Packed(self.scale, self.hi.to(device), self.lo.to(device), self.w2.to(device), self.weights.to(device))


def pack(static: Dict[str, np.ndarray]) -> Packed:
    sd = np.asarray(static["shapedirs"], np.float32)
    nv = sd.shape[0]
    sd = sd.reshape(3 * nv, -1)
    pd = np.asarray(static["posedirs"], np.float32)
    vt = np.asarray(static["v_template"], np.float32).reshape(-1)
    s = basis_scale(sd, pd, vt)
    x = torch.zeros(3 * nv, K)
    x[:, :N_BETAS] = torch.from_numpy(sd) * s                   # exact: power of two
    x[:, N_BETAS:TMPL] = torch.from_numpy(pd).T * s
    hi = f16(x)
    lo = f16(x - hi)
    hi[:, TMPL:], lo[:, TMPL:] = 0.0, 0.0
    r = torch.from_numpy(vt) * s
    pieces = []
    for _ in range(4):
        pieces.append(f16(r))
        r = r - pieces[-1]
    hi[:, TMPL], hi[:, TMPL + 1], lo[:, TMPL], lo[:, TMPL + 1] = pieces
    w = torch.from_numpy(np.asarray(static["lbs_weights"], np.float32))
    rest = torch.zeros(nv)
    for j in (0, 1, 3, 4):
        rest = rest + w[:, j]                                    # fp32, this order
    return Packed(s, hi, lo, torch.stack([rest, w[:, 2]], 1), w)


# --------------------------------------------------------------------------------------------------------- prep rows
def dec_phys_row(h):
    return (h & ~255) + ((h & 7) >> 2) * 128 + (h & 3) * 32 + ((h & 255) >> 3)


def dec_head_of(m_tile, wq, lane):
    return (m_tile >> 1) * 256 + lane * 8 + (m_tile & 1) * 4 + wq


def rows_padded(B: int) -> int:
    return (B + 255) // 256 * 256


def prep_rows(betas: torch.Tensor, pose_feat: torch.Tensor):
    """[B, 448] fp32 values of the hi / lo coefficient rows of flame_prep_kernel (unpermuted)."""
    B = betas.shape[0]
    x = torch.zeros(B, K, dtype=torch.float32, device=betas.device)
    x[:, :N_BETAS] = betas
    x[:, N_BETAS:TMPL] = pose_feat
    hi = f16(x)
    lo = f16(x - hi)
    hi[:, TMPL:TMPL + 2] = 1.0
    return hi, lo


def permute_rows(rows: torch.Tensor) -> torch.Tensor:
    """Unpermuted [B, 448] rows -> the [rows_padded(B), 448] physical layout of the dedicated kernel (padding rows zero)."""
    B = rows.shape[0]
    out = torch.zeros(rows_padded(B), rows.shape[1], dtype=rows.dtype, device=rows.device)
    out[dec_phys_row(torch.arange(B, device=rows.device))] = rows
    return out


# ----------------------------------------------------------------------------------------------------------- mutations
@dataclasses.dataclass(frozen=True)
class Mutation:
    drop_lohi: bool = False          # hi/lo path without lo_coef * hi_basis
    drop_hilo: bool = False          # ... without hi_coef * lo_basis
    add_lolo: bool = False           # ... with a lo * lo product
    drop_tmpl_piece: int = -1        # template piece 0..3 missing from the basis
    drop_col437: bool = False        # second template column missing
    swap_w: bool = False             # w_rest <-> w_jaw
    neighbour_w: bool = False        # weights of the next vertex pair
    swap_rj: bool = False            # rest <-> jaw transforms
    carry_shift: bool = False        # floats written from the carry shifted by one float
    carry_prev_row: bool = False     # floats written from the carry taken from the previous head's row
    no_z_offset: bool = False        # c = 0
    image_size_for_hs: bool = False  # projection scaled by image_size instead of image_size / 2
    tz_nonzero: bool = False         # third projected coordinate translated by tx instead of 0


NONE = Mutation()


# --------------------------------------------------------------------------------------------------------------- product
def _mutated_basis(pk: Packed, mut: Mutation):
    hi, lo = pk.hi, pk.lo
    if mut.drop_tmpl_piece >= 0 or mut.drop_col437:
        hi, lo = hi.clone(), lo.clone()
        planes = [(hi, TMPL), (hi, TMPL + 1), (lo, TMPL), (lo, TMPL + 1)]
        if mut.drop_tmpl_piece >= 0:
            t, c = planes[mut.drop_tmpl_piece]
            t[:, c] = 0.0
        if mut.drop_col437:
            hi[:, TMPL + 1], lo[:, TMPL + 1] = 0.0, 0.0
    return hi, lo


def _exact_class(terms, what: str, check: bool) -> torch.Tensor:
    """Sum over the (a, b) operand pairs of one accumulator class.  With `check` (an unmutated model), assert the exactness
    premise for every output; a mutated model makes no such claim and rounds the exact sum once."""
    acc = sum(a.double() @ b.double().T for a, b in terms)
    if check:
        grid = min(grid_of(a) * grid_of(b) for a, b in terms)
        bound = sum(a.double().abs() @ b.double().abs().T for a, b in terms)
        worst = bound.max().item() if bound.numel() else 0.0
        assert worst < 2.0 ** 24 * grid, f"{what}: accumulator not exact (sum |terms| = {worst / grid:.3g} grid)"
        assert torch.equal(acc.float().double(), acc), what
    return acc.float()


def product(path: str, a_hi: torch.Tensor, a_lo: torch.Tensor, pk: Packed, mut: Mutation = NONE) -> torch.Tensor:
    """[B, 3 nv] fp32 scaled v_posed of the path ("dedicated", "lbs", "blend", "simt", "blend_fast")."""
    b_hi, b_lo = _mutated_basis(pk, mut)
    if path in ("dedicated", "blend_fast"):
        return _exact_class([(a_hi, b_hi)], "hi*hi", mut == NONE)
    if path == "simt":
        a = (a_hi + a_lo).float()
        b = (b_hi + b_lo).float()
        acc = torch.zeros(a.shape[0], b.shape[0], device=a.device)
        for k in range(K):
            acc = fmaf(a[:, k:k + 1], b[:, k][None, :], acc)
        return acc
    acc0 = _exact_class([(a_hi, b_hi)], "acc0", mut == NONE)
    t1 = ([] if mut.drop_lohi else [(a_lo, b_hi)]) + ([] if mut.drop_hilo else [(a_hi, b_lo)])
    t1 += [(a_lo, b_lo)] if mut.add_lolo else []
    acc1 = _exact_class(t1, "acc1", mut == NONE) if t1 else torch.zeros_like(acc0)
    return acc0 + acc1                                            # fp32, one rounding


# ------------------------------------------------------------------------------------------------------------ epilogues
def _chain(A: torch.Tensor, p):
    """fmaf(A0, px, fmaf(A1, py, fmaf(A2, pz, A3))) for the three rows of one [.., 12] transform."""
    px, py, pz = p
    return [fmaf(A[..., 4 * r], px, fmaf(A[..., 4 * r + 1], py, fmaf(A[..., 4 * r + 2], pz, A[..., 4 * r + 3])))
            for r in range(3)]


def skin_fused(v: torch.Tensor, xf: torch.Tensor, pk: Packed, mut: Mutation = NONE) -> torch.Tensor:
    """Dedicated kernel / EpiLbs: [B, 3 nv] scaled v_posed -> [B, nv, 3] vertices."""
    B, nv = v.shape[0], v.shape[1] // 3
    p = v.view(B, nv, 3)
    p = (p[..., 0], p[..., 1], p[..., 2])
    R, J = xf[:, None, 0:12], xf[:, None, 24:36]
    if mut.swap_rj:
        R, J = J, R
    w2 = pk.w2
    if mut.neighbour_w:
        w2 = torch.cat([w2[2:], torch.zeros(2, 2, device=w2.device)])[:nv]
    wr, wj = (w2[:, 1], w2[:, 0]) if mut.swap_w else (w2[:, 0], w2[:, 1])
    c = torch.zeros_like(xf[:, 60:63]) if mut.no_z_offset else xf[:, 60:63]
    rx, jx = _chain(R, p), _chain(J, p)
    out = [fmaf(wj[None].expand(B, nv), jx[r], fmaf(wr[None].expand(B, nv), rx[r], c[:, r:r + 1].expand(B, nv)))
           for r in range(3)]
    return torch.stack(out, -1)


def skin_lbs5(v: torch.Tensor, xf: torch.Tensor, pk: Packed, mut: Mutation = NONE) -> torch.Tensor:
    """lbs_project_kernel: five joints, a joint with w == 0 is skipped."""
    B, nv = v.shape[0], v.shape[1] // 3
    p = v.view(B, nv, 3)
    p = (p[..., 0], p[..., 1], p[..., 2])
    c = torch.zeros_like(xf[:, 60:63]) if mut.no_z_offset else xf[:, 60:63]
    o = [c[:, r:r + 1].expand(B, nv).clone() for r in range(3)]
    for j in range(5):
        w = pk.weights[:, j][None].expand(B, nv)
        t = _chain(xf[:, None, 12 * j:12 * j + 12], p)
        for r in range(3):
            o[r] = torch.where(w != 0, fmaf(w, t[r], o[r]), o[r])
    return torch.stack(o, -1)


def project(verts: torch.Tensor, xf: torch.Tensor, image_size: float, to_2d: bool, dedicated: bool,
            mut: Mutation = NONE) -> torch.Tensor:
    sc, tx, ty = xf[:, 63:64], xf[:, 64:65], xf[:, 65:66]
    tz = tx if mut.tz_nonzero else torch.zeros_like(tx)
    img = torch.tensor(image_size, dtype=torch.float32, device=verts.device)
    out = []
    for r, t in enumerate((tx, ty, tz)[:2 if to_2d else 3]):
        x = fmaf(verts[..., r], sc.expand_as(verts[..., r]), t.expand_as(verts[..., r])) + 1.0
        if mut.image_size_for_hs:
            out.append(x * img)
        elif dedicated:
            out.append(x * (0.5 * img))
        else:
            out.append((x * 0.5) * img)
    return torch.stack(out, -1)


def carry_mask(B: int, nv: int, nc: int, base: int, device=None) -> torch.Tensor:
    """[B, nv * nc] bool: the floats in front of a pass window that the dedicated kernel writes from its carry (the c floats
    before every pass start, c = the row's sector phase; base = the output's offset in floats from a 32-byte boundary)."""
    step = 24 if nc == 3 else 16
    n = nv * nc
    j = torch.arange(n, device=device)
    phase = (base + torch.arange(B, device=device) * n) % 8
    dist = (-j) % step                                       # floats from j to the next pass start
    g0 = j + dist
    return (dist[None, :] > 0) & (dist[None, :] <= phase[:, None]) & (g0[None, :] < n)


def apply_store_mutation(out: torch.Tensor, nc: int, base: int, mut: Mutation) -> torch.Tensor:
    if not (mut.carry_shift or mut.carry_prev_row):
        return out
    B, nv = out.shape[0], out.shape[1]
    flat = out.reshape(B, nv * nc)
    m = carry_mask(B, nv, nc, base, out.device)
    src = torch.roll(flat, 1, dims=1) if mut.carry_shift else torch.roll(flat, 1, dims=0)
    return torch.where(m, src, flat).view_as(out)


def decode(path: str, a_hi, a_lo, xf, pk: Packed, image_size: float = 256.0, to_2d: bool = True,
           mut: Mutation = NONE, base_v: int = 0, base_p: int = 0):
    """(vertices [B, nv, 3], projected [B, nv, 2|3]) of `path` from unpermuted coefficient rows and transform records."""
    v = product(path, a_hi, a_lo, pk, mut)
    fused = path in ("dedicated", "lbs")
    verts = skin_fused(v, xf, pk, mut) if fused else skin_lbs5(v, xf, pk, mut)
    proj = project(verts, xf, image_size, to_2d, path == "dedicated", mut)
    if path == "dedicated":
        verts = apply_store_mutation(verts, 3, base_v, mut)
        proj = apply_store_mutation(proj, 2 if to_2d else 3, base_p, mut)
    return verts, proj


# ------------------------------------------------------------------------------------------------------ designed operands
FLAME_PARENTS = np.array([-1, 0, 1, 1, 1], np.int32)


def designed_static(nv: int, seed: int = 0) -> Dict[str, np.ndarray]:
    """FLAME-shaped constants with small dyadic entries.  Scaled by the packing's 2^10, every basis entry is h + b 2^-12 with
    an integer 2 <= |h| <= 1023 (the fp16 hi piece) and 0 <= b h <= 3 |h| (the lo piece, |b| <= 3: the same sign as h); the scaled template is an integer below 8 000
    in magnitude (one or, above 2 048, two fp16 hi pieces) or, at every seventh entry, three pieces whose third (in the
    lo plane) is +-2^-10; it is zero at every fifth vertex.  Every vertex gets its own
    lbs weights (jaw weight zero at every third vertex, where lbs_project_kernel skips the joint)."""
    g = np.random.default_rng(seed)
    n3 = 3 * nv

    def basis(shape):
        sign = g.choice([-1, 1], size=shape)
        return sign * (g.integers(2, 1024, size=shape) + g.integers(0, 4, size=shape) * 2.0 ** -12) / 1024.0

    sd = basis((n3, N_BETAS))
    sd.flat[0] = 1000.0 / 1024.0                                     # pins the scale: scaled amax in [512, 1024)
    pd = basis((36, n3))
    t0 = g.integers(-1000, 1000, size=n3) * 8.0
    t1 = g.integers(-3, 4, size=n3).astype(np.float64)
    ts = t0 + t1
    # every seventh entry has three pieces: p0 = 8 k with 2^13 < |p0| < 2^14 (p0 + p1 stays in that binade), p1 = m / 2
    # with 5 <= |m| <= 7 and a tail of +-2^-10, the exact midpoint of p1's fp16 spacing, which ties back to the even p1:
    # so p2 = +-2^-10 lands in the lo plane while the hi planes stay on a grid of 1/2 (acc0 remains exact)
    three = np.arange(n3) % 7 == 3
    n = int(three.sum())
    p0 = g.integers(1025, 2048, size=n) * 8.0 * g.choice([-1, 1], size=n)
    p1 = g.integers(5, 8, size=n) * 0.5 * g.choice([-1, 1], size=n)
    ts[three] = p0 + p1 + g.choice([-1, 1], size=n) * 2.0 ** -10
    vt = ts / 1024.0
    vt.reshape(nv, 3)[4::5] = 0.0
    w = (g.random((nv, 5)) * 0.4 + 0.01).astype(np.float32)    # not normalised: every (w_rest, w_jaw) pair differs
    w[::3, 2] = 0.0
    jr = np.zeros((5, nv), np.float32)
    for j in range(5):
        jr[j, g.integers(0, nv, size=min(nv, 4))] = 0.25
    return dict(shapedirs=sd.reshape(nv, 3, N_BETAS).astype(np.float32), posedirs=pd.astype(np.float32),
                v_template=vt.reshape(nv, 3).astype(np.float32), J_regressor=jr, parents=FLAME_PARENTS.copy(),
                lbs_weights=w)


def designed_rows(B: int, generator: torch.Generator, device=None):
    """Coefficient rows (hi, lo), fp32 values: hi = c 2^-4 with |c| <= 15, lo = d 2^-16 with |d| <= 7 (nonzero lo * lo
    products), 1.0 in both template columns.  Every fourth head is quiet: one nonzero beta, so that small terms show."""
    kw = dict(generator=generator, device=device)
    hi = torch.randint(-15, 16, (B, K), **kw).float() * 2.0 ** -4
    lo = torch.randint(-7, 8, (B, K), **kw).float() * 2.0 ** -16
    hi[:, TMPL + 2:], lo[:, TMPL:] = 0.0, 0.0
    quiet = torch.arange(B, device=device) % 4 == 3
    keep = torch.zeros(B, K, dtype=torch.bool, device=device)
    keep[torch.arange(B, device=device), torch.randint(0, N_BETAS, (B,), **kw)] = True
    hi = torch.where(quiet[:, None] & ~keep, torch.zeros_like(hi), hi)
    lo = torch.where(quiet[:, None] & ~keep, torch.zeros_like(lo), lo)
    hi[:, TMPL:TMPL + 2] = 1.0
    return hi, lo


def designed_xf(B: int, generator: torch.Generator, scale: float, device=None) -> torch.Tensor:
    """Transform records: five distinct [R | t] per head (rotation parts ~ 1 / basis scale), offset c, scale, tx, ty.
    Quiet heads (every fourth) have zero translations and offset."""
    kw = dict(generator=generator, device=device)
    xf = torch.zeros(B, XF, device=device)
    A = torch.randn(B, 5, 3, 4, **kw)
    A[..., :3] /= scale
    A[..., 3] *= 0.02
    quiet = torch.arange(B, device=device) % 4 == 3
    A[..., 3] = torch.where(quiet[:, None, None], torch.zeros_like(A[..., 3]), A[..., 3])
    xf[:, :60] = A.reshape(B, 60)
    xf[:, 60:63] = torch.where(quiet[:, None], torch.zeros(B, 3, device=device), torch.randn(B, 3, **kw) * 0.05)
    xf[:, 63] = torch.rand(B, **kw) + 0.5
    xf[:, 64:66] = torch.rand(B, 2, **kw) * 0.6 - 0.3
    return xf


# ------------------------------------------------------------------------------------------------ prep records (fp64)
def _rodrigues(r: torch.Tensor) -> torch.Tensor:
    """smplx batch_rodrigues as flame_prep_kernel computes it: the 1e-8 is added to the vector inside the norm."""
    angle = torch.linalg.norm(r + 1e-8, dim=-1, keepdim=True)
    x, y, z = (r / angle).unbind(-1)
    s, c1 = torch.sin(angle)[..., 0], 1.0 - torch.cos(angle)[..., 0]
    zero = torch.zeros_like(x)
    K = torch.stack([zero, -z, y, z, zero, -x, -y, x, zero], -1).view(*r.shape[:-1], 3, 3)
    eye = torch.eye(3, dtype=r.dtype, device=r.device)
    return eye + s[..., None, None] * K + c1[..., None, None] * (K @ K)


def prep_records(params: torch.Tensor, static: Dict[str, np.ndarray], scale: float, dtype=torch.float64):
    """Restatement of flame_prep_kernel for the released layout (300 shape, 100 expression, jaw, 6-D rotation,
    translation, scale; FLAME parents) in `dtype`.  The folded joint regressor is rounded to fp32 as dad3d_flame_create
    stores it.  Returns (pose features [B, 36] = R_j - I for joints 1..4, records [B, 68], cond [B] = 1 + |vy| / |b1 x vy|,
    the amplification of the 6-D Gram-Schmidt step)."""
    p = params.to(dtype)
    dev = p.device
    B = p.shape[0]
    jr = torch.from_numpy(np.asarray(static["J_regressor"], np.float64))
    vt = torch.from_numpy(np.asarray(static["v_template"], np.float64)).reshape(-1, 3)
    sd = torch.from_numpy(np.asarray(static["shapedirs"], np.float64))
    jt = (jr @ vt).float().to(dev, dtype)                                         # [5, 3]
    jd = torch.einsum("jv,vcl->jcl", jr, sd).float().to(dev, dtype)              # [5, 3, 400]
    J = jt + torch.einsum("jcl,bl->bjc", jd, p[:, :N_BETAS])                     # [B, 5, 3]
    pose = torch.zeros(B, 5, 3, dtype=dtype, device=dev)
    pose[:, 2] = p[:, 400:403]                                                   # jaw = joint 2
    R = _rodrigues(pose)                                                         # [B, 5, 3, 3]
    feats = (R[:, 1:] - torch.eye(3, dtype=dtype, device=dev)).reshape(B, 36)
    parents = FLAME_PARENTS
    GR, Gt = [R[:, 0]], [J[:, 0]]
    for i in range(1, 5):
        par = int(parents[i])
        GR.append(GR[par] @ R[:, i])
        Gt.append((GR[par] @ (J[:, i] - J[:, par])[..., None])[..., 0] + Gt[par])
    vx, vy = p[:, 403:406], p[:, 406:409]
    n1 = torch.linalg.norm(vx, dim=-1, keepdim=True).clamp_min(1e-12)
    b1 = vx / n1
    c3 = torch.linalg.cross(b1, vy, dim=-1)
    n3 = torch.linalg.norm(c3, dim=-1, keepdim=True).clamp_min(1e-12)
    b3 = c3 / n3
    b2 = -torch.linalg.cross(b1, b3, dim=-1)
    R6 = torch.stack([b1, b2, b3], -1)                                           # columns b1, b2, b3
    rec = torch.zeros(B, XF, dtype=dtype, device=dev)
    for i in range(5):
        t = Gt[i] - (GR[i] @ J[:, i, :, None])[..., 0]
        AR = R6 @ GR[i]
        At = (R6 @ t[..., None])[..., 0]
        rec[:, 12 * i:12 * i + 12] = torch.cat([AR / scale, At[..., None]], -1).reshape(B, 12)
    rec[:, 60:63] = R6[:, :, 2] * MESH_OFFSET_Z
    rec[:, 63] = (p[:, 412] + 1.0).clamp_min(1e-8)
    rec[:, 64:66] = p[:, 409:411]
    cond = 1.0 + torch.linalg.norm(vy, dim=-1) / n3[:, 0]
    return feats, rec, cond, J
