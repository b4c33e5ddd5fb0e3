"""Exact model of the FLAME decoder backward (csrc/flame.cu: flame_bwd_gmax_kernel, flame_bwd_vertex_kernel, the dense
EpiBlend product over the transposed basis, flame_bwd_finalize_kernel), in torch so that it runs on the CPU or on the device,
and designed operands on which every stage is fully determined.

What it restates, in kernel order:
1. sigma (gmax kernel): g = fmaf(sc * half_img, gP, gV); m = the fmaxf maximum of |g| (NaN entries ignored); sigma =
   2^min(10 - e, sigma_emax) for m = f 2^e, f in [0.5, 1), when m is finite and > 0, else 1.  sigma_emax = min(127, 127 -
   log2(basis_scale)) keeps sigma * basis_scale finite (without the cap a head with m < 2^(log2(basis_scale) - 118) got an
   infinite lift and a NaN gradient: `Mutation.no_sigma_cap`).
2. The vertex kernel: gq = half_img * gP, the forward value o = fmaf(wj, b, fmaf(wr, a, c)) over fmaf chains, the 30
   cotangent terms, g = fmaf(sc, gq, gV), dp = wr (A0'^T g) + wj (A2'^T g), the fp16 round-to-nearest hi/lo split of
   dp * lift (lift = sigma * basis_scale), and the reductions in kernel order: xor butterfly 16 ... 1 (lane 0's value),
   warps 0 ... 7 in order, then blocks 0 ... n-1 in order (finalize kernel).
3. The dense product: acc0 = hi*hi, acc1 = lo*hi + hi*lo (no lo*lo), then fp32(acc0 + acc1).  As in decode_model, every
   accumulator is asserted exact whatever the summation order: all terms on one power-of-two grid, sum |terms| < 2^24 grid.
4. The finalize kernel's linear parts: dcoef * unlift (unlift = 1 / lift, exact), the fmaf chain over the 15 joint
   directions, the placement of the shape / expression / jaw / rotation / translation / scale gradients, t_z = 0, the
   ZERO_ROT / ZERO_JAW zeros and the scale clamp (s + 1 > 1e-8 in fp32).  The 24-input transform function F is
   differentiated in dual numbers in the kernel; the model gives its fp64 autograd gradient and Jacobian instead
   (`transform_grads`), against which the GPU tests apply an error bound.

Kernel source that leaves rounding to the compiler -- plain `a*b + c` that nvcc may contract, in dp, acc[27] (d sc) and
the Dual ops -- is modelled bit-exactly only on designed operands that make every contraction exact: `exact_sum` asserts
that premise (one grid, sum |terms| < 2^24 grid, per output element) for dp and acc[27].  Where dp is exactly zero, its
sign still depends on the contraction (a fused multiply-add of two negative zeros gives -0, the model's sum +0), so
zeros of D are compared without their sign.  The Dual ops are never modelled bit for bit.

`Mutation` switches in the errors the exact tests must be able to see (tests/test_backward_model_cpu.py shows that each
of them changes an output the GPU tests compare)."""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, Optional

import numpy as np
import torch

from tests import decode_model as dm
from tests.decode_model import f16, fmaf

K = dm.K
N_BETAS = dm.N_BETAS
XF = dm.XF
PARTIAL = 32             # floats per (head, vertex block) partial record
BLOCK = 256              # vertices per vertex-kernel block
N_COT = 30
JAW_FEATS = slice(N_BETAS + 9, N_BETAS + 18)      # pose features of joint 2 (the jaw) in the coefficient columns
ZERO_ROT, ZERO_JAW = 1, 2
# released layout: shape 0..299, expression 300..399, jaw 400..402, rotation 403..408, translation 409..411, scale 412
OFF_JAW, OFF_ROT, OFF_TRANS, OFF_SCALE, N_PARAMS = 400, 403, 409, 412, 413


@dataclasses.dataclass(frozen=True)
class Mutation:
    sigma_head0: bool = False        # every head lifted by head 0's sigma
    no_sigma_cap: bool = False       # sigma's exponent not capped (the old defect)
    drop_d_lo: bool = False          # lo plane of D dropped
    drop_lohi: bool = False          # dense product without lo_D * hi_basis
    drop_hilo: bool = False          # ... without hi_D * lo_basis
    swap_w: bool = False             # w_rest <-> w_jaw
    swap_a: bool = False             # A0' <-> A2'
    partial_next_block: bool = False # finalize reads partial block b + 1 (zero past the last one)
    half_img_twice: bool = False     # gP scaled by half_img twice
    tz_nonzero: bool = False         # t_z gradient = d tx instead of 0
    jaw_cols_first: bool = False     # jaw pose features read from columns 400 + 0..8 instead of 400 + 9..17


NONE = Mutation()


# ------------------------------------------------------------------------------------------------------------ arithmetic
def lowbit(x: torch.Tensor) -> torch.Tensor:
    """Elementwise largest power of two dividing |x| (fp64; inf where x == 0)."""
    a = x.double().abs()
    m, e = torch.frexp(torch.where(a == 0, torch.ones_like(a), a))
    mi = (m * 2.0 ** 53).to(torch.int64)
    low = torch.ldexp((mi & -mi).double(), (e - 53).double())
    return torch.where(a == 0, torch.full_like(a, math.inf), low)


def exact_sum(terms, what: str) -> torch.Tensor:
    """fp32 value of a sum of fp64 terms that fp32 arithmetic computes exactly in any order and with any contraction:
    asserted per element (one grid = the smallest low bit of the terms, sum |terms| < 2^24 grid, grid >= 2^-149)."""
    terms = [t.double() for t in terms]
    grid = terms[0].new_full(terms[0].shape, math.inf)
    tot = torch.zeros_like(terms[0])
    s = torch.zeros_like(terms[0])
    for t in terms:
        grid = torch.minimum(grid, lowbit(t))
        tot = tot + t.abs()
        s = s + t
    ok = (tot == 0) | ((tot < 2.0 ** 24 * grid) & (grid >= 2.0 ** -149) & (tot < 2.0 ** 127))
    assert bool(ok.all()), f"{what}: not exact in fp32 at {(~ok).nonzero()[0].tolist()}"
    return s.float()


def log2_scale(scale: float) -> int:
    k = int(round(math.log2(scale)))
    assert 2.0 ** k == scale
    return k


def sigma_emax(scale: float) -> int:
    return min(127, 127 - log2_scale(scale))


# --------------------------------------------------------------------------------------------------------------- stage 1
def _grads(gv, gp, B, nv, pc, device):
    gv = gv if gv is not None else torch.zeros(B, nv, 3, device=device)
    gp3 = torch.zeros(B, nv, 3, device=device)
    if gp is not None:
        gp3[..., :pc] = gp
    return gv.float(), gp3.float(), gp is not None


def sigma(gv, gp, xf, image_size: float, to_2d: bool, scale: float, mut: Mutation = NONE) -> torch.Tensor:
    """[B] fp32: flame_bwd_gmax_kernel."""
    B = xf.shape[0]
    ref = gv if gv is not None else gp
    nv = ref.shape[1]
    half_img = torch.tensor(0.5 * image_size, dtype=torch.float32)
    g, gp3, has_p = _grads(gv, gp, B, nv, 2 if to_2d else 3, xf.device)
    if has_p:
        sc = (xf[:, 63] * half_img.to(xf.device))[:, None, None].expand_as(g)
        g = fmaf(sc.contiguous(), gp3, g)             # gP's missing third coordinate adds 0: g[2] = gV[2]
    a = g.abs()
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
    m = a.reshape(B, -1).amax(1).double()
    _, e = torch.frexp(torch.where(m > 0, m, torch.ones_like(m)))
    n = 10 - e
    if not mut.no_sigma_cap:
        n = torch.clamp(n, max=sigma_emax(scale))
    s = torch.ldexp(torch.ones_like(m).float(), n.float())
    s = torch.where((m > 0) & torch.isfinite(m), s, torch.ones_like(s))
    if mut.sigma_head0:
        s = s[:1].expand(B).clone()
    return s


def _tree32(x: torch.Tensor) -> torch.Tensor:
    """Lane 0's value after the xor butterfly 16, 8, 4, 2, 1 over the second-to-last axis (32 lanes), fp32."""
    n = 32
    while n > 1:
        n //= 2
        x = x[..., :n, :] + x[..., n:2 * n, :]
    return x[..., 0, :]


def vertex_stage(vposed, xf, gv, gp, w2, image_size: float, to_2d: bool, scale: float, mut: Mutation = NONE,
                 check: Optional[bool] = None):
    """flame_bwd_gmax_kernel + flame_bwd_vertex_kernel: (sigma [B], d_hi [B, npad], d_lo [B, npad] as fp32 values of the
    fp16 planes, partial [B, n_blocks, 30]).  vposed [B, npad] fp32 (ld npad), xf [B, 68], w2 [nv, 2] (w_rest, w_jaw).
    `check` (default: unmutated) asserts that every contractable expression is exact."""
    check = (mut == NONE) if check is None else check
    B, npad = vposed.shape
    nv = w2.shape[0]
    dev = vposed.device
    pc = 2 if to_2d else 3
    sig = sigma(gv, gp, xf, image_size, to_2d, scale, mut)
    half_img = torch.tensor(0.5 * image_size, dtype=torch.float32, device=dev)
    g, gp3, has_p = _grads(gv, gp, B, nv, pc, dev)
    gq = half_img * gp3
    if mut.half_img_twice:
        gq = half_img * gq
    p = vposed[:, :3 * nv].reshape(B, nv, 3)
    wr, wj = w2[:, 0][None, :], w2[:, 1][None, :]
    if mut.swap_w:
        wr, wj = wj, wr
    A0, A2 = xf[:, 0:12].reshape(B, 1, 3, 4), xf[:, 24:36].reshape(B, 1, 3, 4)
    if mut.swap_a:
        A0, A2 = A2, A0
    A0, A2 = A0.expand(B, nv, 3, 4).contiguous(), A2.expand(B, nv, 3, 4).contiguous()
    c = xf[:, None, 60:63].expand(B, nv, 3)
    o = []
    for r in range(3):
        a = fmaf(A0[..., r, 0], p[..., 0], fmaf(A0[..., r, 1], p[..., 1], fmaf(A0[..., r, 2], p[..., 2], A0[..., r, 3])))
        b = fmaf(A2[..., r, 0], p[..., 0], fmaf(A2[..., r, 1], p[..., 1], fmaf(A2[..., r, 2], p[..., 2], A2[..., r, 3])))
        o.append(fmaf(wj.expand(B, nv), b, fmaf(wr.expand(B, nv), a, c[..., r].contiguous())))
    terms = [gq[..., r].double() * o[r].double() for r in range(3)]
    acc27 = exact_sum(terms, "acc[27]") if check else sum(terms).float()
    sc = xf[:, 63][:, None, None].expand_as(g).contiguous()
    g = fmaf(sc, gq, g)
    acc = torch.zeros(B, nv, N_COT, device=dev)
    for r in range(3):
        for cc in range(3):
            acc[..., 3 * r + cc] = (wr * g[..., r]) * p[..., cc]
            acc[..., 12 + 3 * r + cc] = (wj * g[..., r]) * p[..., cc]
        acc[..., 9 + r] = wr * g[..., r]
        acc[..., 21 + r] = wj * g[..., r]
        acc[..., 24 + r] = g[..., r]
    acc[..., 27], acc[..., 28], acc[..., 29] = acc27, gq[..., 0], gq[..., 1]
    d = []
    for cc in range(3):
        t0 = [A0[..., r, cc].double() * g[..., r].double() for r in range(3)]
        t2 = [A2[..., r, cc].double() * g[..., r].double() for r in range(3)]
        if check:
            s0, s2 = exact_sum(t0, "dp (A0 part)"), exact_sum(t2, "dp (A2 part)")
            d.append(exact_sum([wr.double() * s0.double(), wj.double() * s2.double()], "dp"))
        else:
            d.append((wr.double() * sum(t0) + wj.double() * sum(t2)).float())
    lift = sig * torch.tensor(scale, dtype=torch.float32)
    x = torch.stack(d, -1).reshape(B, 3 * nv) * lift[:, None]
    hi = f16(x)
    lo = f16(x - hi)
    if mut.drop_d_lo:
        lo = torch.zeros_like(lo)
    d_hi = torch.zeros(B, npad, device=dev)
    d_lo = torch.zeros(B, npad, device=dev)
    d_hi[:, :3 * nv], d_lo[:, :3 * nv] = hi, lo
    nb = (nv + BLOCK - 1) // BLOCK
    pad = torch.zeros(B, nb * BLOCK, N_COT, device=dev)
    pad[:, :nv] = acc
    warps = _tree32(pad.view(B, nb, 8, 32, N_COT))             # [B, nb, 8, 30]
    part = torch.zeros(B, nb, N_COT, device=dev)
    for w in range(8):
        part = part + warps[:, :, w]
    return sig, d_hi, d_lo, part


# --------------------------------------------------------------------------------------------------------------- stage 2
DENSE_COLS = list(range(dm.TMPL)) + list(range(dm.TMPL + 2, K))   # every column but the two template columns


def dense_stage(d_hi, d_lo, pk: dm.Packed, mut: Mutation = NONE) -> torch.Tensor:
    """[B, 448] fp32 dcoef = fp32(acc0 + acc1) over the transposed basis planes (pk.hi / pk.lo are [3 nv, 448]).  The two
    template columns 436, 437 (which the finalize kernel never reads, and whose designed entries are too wide for an exact
    fp32 accumulation) come back NaN."""
    n3 = pk.hi.shape[0]
    a_hi, a_lo = d_hi[:, :n3], d_lo[:, :n3]
    if mut.drop_d_lo:
        a_lo = torch.zeros_like(a_lo)
    b_hi, b_lo = pk.hi.T[DENSE_COLS], pk.lo.T[DENSE_COLS]      # [446, 3 nv]
    check = mut == NONE
    acc0 = dm._exact_class([(a_hi, b_hi)], "acc0", check)
    t1 = ([] if mut.drop_lohi else [(a_lo, b_hi)]) + ([] if mut.drop_hilo else [(a_hi, b_lo)])
    acc1 = dm._exact_class(t1, "acc1", check) if t1 else torch.zeros_like(acc0)
    out = torch.full((d_hi.shape[0], K), float("nan"), device=d_hi.device)
    out[:, DENSE_COLS] = acc0 + acc1
    return out


# --------------------------------------------------------------------------------------------------------------- stage 3
def cotangents(partial: torch.Tensor, mut: Mutation = NONE) -> torch.Tensor:
    """[B, 30]: the finalize kernel's sum over the vertex blocks, blocks 0 ... n-1 in order, fp32."""
    part = partial[..., :N_COT]
    if mut.partial_next_block:
        part = torch.cat([part[:, 1:], torch.zeros_like(part[:, :1])], 1)
    s = torch.zeros(part.shape[0], N_COT, device=part.device)
    for b in range(part.shape[1]):
        s = s + part[:, b]
    return s


def unlift(sig: torch.Tensor, scale: float) -> torch.Tensor:
    return 1.0 / (sig * torch.tensor(scale, dtype=torch.float32))


def finalize_linear(params, dcoef, partial, sig, scale: float, flags: int = 0, mut: Mutation = NONE):
    """The entries of the finalize kernel's output that the model gives exactly, as (values [B, 413], mask [B, 413]):
    betas = dcoef * unlift where the joint term vanishes (no cotangents of F: partial == 0), translation (d tx, d ty, 0),
    scale (clamped), and the zeros of ZERO_ROT / ZERO_JAW."""
    B = params.shape[0]
    cot = cotangents(partial, mut)
    out = torch.zeros(B, N_PARAMS, device=params.device)
    mask = torch.zeros(B, N_PARAMS, dtype=torch.bool, device=params.device)
    no_j = (cot[:, :27] == 0).all(1)
    out[:, :N_BETAS] = dcoef[:, :N_BETAS] * unlift(sig, scale)[:, None]
    mask[:, :N_BETAS] = no_j[:, None]
    out[:, OFF_TRANS], out[:, OFF_TRANS + 1] = cot[:, 28], cot[:, 29]
    out[:, OFF_TRANS + 2] = cot[:, 28] if mut.tz_nonzero else 0.0
    clamp_ok = (params[:, OFF_SCALE] + 1.0) > torch.tensor(1e-8, dtype=torch.float32)
    out[:, OFF_SCALE] = torch.where(clamp_ok, cot[:, 27], torch.zeros_like(cot[:, 27]))
    mask[:, OFF_TRANS:] = True
    if flags & ZERO_JAW:
        mask[:, OFF_JAW:OFF_JAW + 3] = True
    if flags & ZERO_ROT:
        mask[:, OFF_ROT:OFF_ROT + 6] = True
    return out, mask


def joint_constants(static: Dict[str, np.ndarray]):
    """(jt [15], jdirsT [15, 400]) as dad3d_flame_create stores them (fp32 of the fp64 regression)."""
    jr = torch.from_numpy(np.asarray(static["J_regressor"], np.float64))
    vt = torch.from_numpy(np.asarray(static["v_template"], np.float64)).reshape(-1, 3)
    sd = torch.from_numpy(np.asarray(static["shapedirs"], np.float64))
    jt = (jr @ vt).float().reshape(15)
    jd = torch.einsum("jv,vcl->jcl", jr, sd).float().reshape(15, N_BETAS)
    return jt, jd


def transform_f64(jaw, rot6, J, flags: int, scale: float):
    """F(jaw[3], rot6[6], J[15]) -> out [B, 36] in fp64, as head_transforms_dual computes it: A0'[9] t0[3] A2'[9] t2[3]
    c[3] phi_jaw[9] (A' row-major with 1 / basis_scale folded in)."""
    B = jaw.shape[0]
    eye = torch.eye(3, dtype=jaw.dtype, device=jaw.device)
    jz = torch.zeros_like(jaw) if flags & ZERO_JAW else jaw
    R2 = dm._rodrigues(jz)
    Jm = J.reshape(B, 5, 3)
    Gt0 = Jm[:, 0]
    Gt1 = (Jm[:, 1] - Jm[:, 0]) + Gt0
    Gt2 = (Jm[:, 2] - Jm[:, 1]) + Gt1
    if flags & ZERO_ROT:
        R6 = eye.expand(B, 3, 3)
    else:
        vx, vy = rot6[:, :3], rot6[:, 3:]
        b1 = vx / torch.linalg.norm(vx, dim=-1, keepdim=True).clamp_min(1e-12)
        c3 = torch.linalg.cross(b1, vy, dim=-1)
        b3 = c3 / torch.linalg.norm(c3, dim=-1, keepdim=True).clamp_min(1e-12)
        b2 = -torch.linalg.cross(b1, b3, dim=-1)
        R6 = torch.stack([b1, b2, b3], -1)
    outs = []
    for GR, Gt, j in ((eye.expand(B, 3, 3), Gt0, 0), (R2, Gt2, 2)):
        t = Gt - (GR @ Jm[:, j, :, None])[..., 0]
        outs += [(R6 @ GR).reshape(B, 9) / scale, (R6 @ t[..., None])[..., 0]]
    outs += [R6[:, :, 2] * dm.MESH_OFFSET_Z, (R2 - eye).reshape(B, 9)]
    return torch.cat(outs, -1)


def transform_inputs(params, jt, jdirsT):
    """(jaw, rot6, J [B, 15]) in fp64; J = jt + jdirsT beta."""
    p = params.double()
    J = jt.double().to(p.device) + p[:, :N_BETAS] @ jdirsT.double().to(p.device).T
    return p[:, OFF_JAW:OFF_JAW + 3], p[:, OFF_ROT:OFF_ROT + 6], J


def transform_grads(params, cot, dc_phi, jt, jdirsT, scale: float, flags: int = 0):
    """fp64 gradients of <cot[:27], F[:27]> + <dc_phi, phi_jaw> w.r.t. (jaw, rot6, J), and the abs-contracted Jacobian
    sum_i |w_i| |dF_i / dx| (the magnitude an error bound scales with).  dc_phi = dcoef[jaw features] * unlift."""
    jaw, rot6, J = (t.clone().requires_grad_(True) for t in transform_inputs(params, jt, jdirsT))
    out = transform_f64(jaw, rot6, J, flags, scale)
    w =torch.cat([cot[:, :27].double(), dc_phi.double()], 1)
    mag = torch.zeros(out.shape[0], 24, dtype=torch.float64, device=out.device)
    for i in range(36):
        gi = torch.autograd.grad(out[:, i].sum(), (jaw, rot6, J), retain_graph=True, allow_unused=True)
        gi = torch.cat([g if g is not None else torch.zeros_like(x) for g, x in zip(gi, (jaw, rot6, J))], 1)
        mag = mag + w[:, i:i + 1].abs() * gi.abs()
    grads = torch.autograd.grad((out * w).sum(), (jaw, rot6, J), allow_unused=True)
    grads = torch.cat([g if g is not None else torch.zeros_like(x) for g, x in zip(grads, (jaw, rot6, J))], 1)
    return grads.detach(), mag.detach()


def jaw_feature_cols(mut: Mutation = NONE) -> slice:
    return slice(N_BETAS, N_BETAS + 9) if mut.jaw_cols_first else JAW_FEATS


def finalize_f64(params, dcoef, partial, sig, jt, jdirsT, scale: float, flags: int = 0, mut: Mutation = NONE):
    """fp64 reference of the whole finalize output [B, 413] from the kernel's inputs (dcoef * unlift is exact), and the
    magnitude [B, 413] its rounding bound scales with."""
    cot = cotangents(partial, mut).double()
    ul = unlift(sig, scale).double()[:, None]
    dc = dcoef.double() * ul
    grads, mag = transform_grads(params, cot, dc[:, jaw_feature_cols(mut)], jt, jdirsT, scale, flags)
    jd = jdirsT.double().to(params.device)
    B = params.shape[0]
    out = torch.zeros(B, N_PARAMS, dtype=torch.float64, device=params.device)
    m = torch.zeros_like(out)
    out[:, :N_BETAS] = dc[:, :N_BETAS] + grads[:, 9:] @ jd
    m[:, :N_BETAS] = dc[:, :N_BETAS].abs() + mag[:, 9:] @ jd.abs()
    out[:, OFF_JAW:OFF_JAW + 3] = 0.0 if flags & ZERO_JAW else grads[:, 0:3]
    m[:, OFF_JAW:OFF_JAW + 3] = mag[:, 0:3]
    out[:, OFF_ROT:OFF_ROT + 6] = 0.0 if flags & ZERO_ROT else grads[:, 3:9]
    m[:, OFF_ROT:OFF_ROT + 6] = mag[:, 3:9]
    lin, _ = finalize_linear(params, dcoef, partial, sig, scale, flags, mut)
    out[:, OFF_TRANS:] = lin[:, OFF_TRANS:].double()
    return out, m


def gram_schmidt_cond(params) -> torch.Tensor:
    """[B] 1 + |vy| / |b1 x vy|: the amplification of the 6-D Gram-Schmidt step (as decode_model.prep_records)."""
    p = params.double()
    vx, vy = p[:, OFF_ROT:OFF_ROT + 3], p[:, OFF_ROT + 3:OFF_ROT + 6]
    b1 = vx / torch.linalg.norm(vx, dim=-1, keepdim=True).clamp_min(1e-12)
    return 1.0 + torch.linalg.norm(vy, dim=-1) / torch.linalg.norm(torch.linalg.cross(b1, vy, dim=-1), dim=-1).clamp_min(1e-300)


FINALIZE_ULPS = 1024


def finalize_bound(params, mag) -> torch.Tensor:
    """Per-entry bound of |finalize - finalize_f64|: FINALIZE_ULPS u cond mag + 2^-126.  mag = sum_i |w_i| |dF_i / dx|
    (plus |dcoef unlift| and the joint directions for the betas), cond = gram_schmidt_cond.  The dual-number chain runs
    about a hundred fp32 operations deep per directional derivative (Rodrigues with its division by the angle, two 3x3
    products, Gram-Schmidt with two divisions by norms); FINALIZE_ULPS = 2^10 leaves a factor of a few over that count
    for the cancellation inside the chain that mag does not see."""
    u = 2.0 ** -24
    cond = gram_schmidt_cond(params)[:, None]
    return FINALIZE_ULPS * u * cond * mag + 2.0 ** -126


def designed_finalize_inputs(B: int, nv: int, generator: torch.Generator, device=None, zero_partial: bool = False,
                             zero_dcoef: bool = False):
    """(params [B, 413], dcoef [B, 448], partial [B, n_blocks, 32], sigma [B]) for the finalize stage.  Partials are
    integers times 2^-6 (|.| <= 64) in every block, so that their block sums are exact in any order; floats 30, 31 of every
    record are NaN (the kernel must not read them).  sigma = 2^n, |n| <= 20, per head.  Parameters: betas N(0, 0.3^2), jaw
    in [-0.3, 0.3], 6-D rotation N(0, 1), translation N(0, 0.1^2), scale in [-0.25, 0.25]; head 1 has scale -1.5 and
    head 2 scale -1 (the clamp max(s + 1, 1e-8) is active: d scale = 0)."""
    kw = dict(generator=generator, device=device)
    nb = (nv + BLOCK - 1) // BLOCK
    params = torch.zeros(B, N_PARAMS, device=device)
    params[:, :N_BETAS] = torch.randn(B, N_BETAS, **kw) * 0.3
    params[:, OFF_JAW:OFF_JAW + 3] = torch.rand(B, 3, **kw) * 0.6 - 0.3
    params[:, OFF_ROT:OFF_ROT + 6] = torch.randn(B, 6, **kw)
    params[:, OFF_TRANS:OFF_TRANS + 3] = torch.randn(B, 3, **kw) * 0.1
    params[:, OFF_SCALE] = torch.rand(B, **kw) * 0.5 - 0.25
    if B > 2:
        params[1, OFF_SCALE], params[2, OFF_SCALE] = -1.5, -1.0
    dcoef = torch.zeros(B, K, device=device) if zero_dcoef else torch.randn(B, K, **kw)
    partial = torch.randint(-64, 65, (B, nb, PARTIAL), **kw).float() * 2.0 ** -6
    if zero_partial:
        partial.zero_()
    partial[..., N_COT:] = float("nan")
    sig = torch.ldexp(torch.ones(B, device=device), torch.randint(-20, 21, (B,), **kw).float())
    return params, dcoef, partial, sig


# ------------------------------------------------------------------------------------------------------ designed operands
def designed_static(nv: int, seed: int = 0) -> Dict[str, np.ndarray]:
    """decode_model.designed_static with dyadic lbs weights k / 64, 1 <= k <= 7 (jaw weight zero at every third vertex), so
    that w_rest (the fp32 sum of four) and every product with it stay short."""
    st = dm.designed_static(nv, seed)
    g = np.random.default_rng(seed + 1)
    w = g.integers(1, 8, size=(nv, 5)).astype(np.float32) / 64.0
    w[::3, 2] = 0.0
    st["lbs_weights"] = w
    return st


def designed_vertex_inputs(B: int, nv: int, npad: int, scale: float, exps, generator: torch.Generator, device=None,
                           to_2d: bool = True, with_v: bool = True, with_p: bool = True):
    """Operands of the vertex stage on which every contraction is exact (see the module docstring):
      vposed  integers |p| <= 31 (columns past 3 nv: 0);
      xf      A0', A2' rotation parts alpha 2^-6 / basis_scale (|alpha| <= 7), translations tau 2^-12 (|tau| <= 15), offset
              c = gamma 2^-16 (|gamma| <= 15), sc = kappa / 16 (8 <= kappa <= 31), tx, ty in [-0.3, 0.3];
      gV, gP  i 2^E_h with |i| <= 7, E_h = exps[h] (None: the head's gradients are all zero)."""
    kw = dict(generator=generator, device=device)
    vposed = torch.zeros(B, npad, device=device)
    vposed[:, :3 * nv] = torch.randint(-31, 32, (B, 3 * nv), **kw).float()
    xf = torch.zeros(B, XF, device=device)
    A = torch.randint(-7, 8, (B, 5, 3, 4), **kw).float()
    A[..., :3] *= 2.0 ** -6 / scale
    A[..., 3] = torch.randint(-15, 16, (B, 5, 3), **kw).float() * 2.0 ** -12
    xf[:, :60] = A.reshape(B, 60)
    xf[:, 60:63] = torch.randint(-15, 16, (B, 3), **kw).float() * 2.0 ** -16
    xf[:, 63] = torch.randint(8, 32, (B,), **kw).float() / 16.0
    xf[:, 64:66] = torch.rand(B, 2, **kw) * 0.6 - 0.3
    pw = torch.tensor([0.0 if e is None else 2.0 ** e for e in exps], device=device)[:, None, None]
    gv = torch.randint(-7, 8, (B, nv, 3), **kw).float() * pw if with_v else None
    gp = torch.randint(-7, 8, (B, nv, 2 if to_2d else 3), **kw).float() * pw if with_p else None
    return vposed, xf, gv, gp


def designed_d_planes(B: int, nv: int, npad: int, generator: torch.Generator, device=None):
    """fp16 D planes for the dense stage, as fp32 values: hi = c 2^-4 (|c| <= 15) at one column in 32, lo = d 2^-16
    (|d| <= 5) at one column in 8 (independently), zero past 3 nv.  With the designed basis (|hi| <= 1023, lo on 2^-12)
    every accumulator of the shape / expression / pose-feature columns stays below 2^24 of its grid for the full mesh."""
    kw = dict(generator=generator, device=device)
    n3 = 3 * nv
    hi = torch.randint(-15, 16, (B, n3), **kw).float() * 2.0 ** -4
    lo = torch.randint(-5, 6, (B, n3), **kw).float() * 2.0 ** -16
    hi = torch.where(torch.randint(0, 32, (B, n3), **kw) == 0, hi, torch.zeros_like(hi))
    lo = torch.where(torch.randint(0, 8, (B, n3), **kw) == 0, lo, torch.zeros_like(lo))
    d_hi, d_lo = torch.zeros(B, npad, device=device), torch.zeros(B, npad, device=device)
    d_hi[:, :n3], d_lo[:, :n3] = hi, lo
    return d_hi, d_lo
