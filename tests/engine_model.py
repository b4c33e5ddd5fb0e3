"""Exact CPU model of one conv / linear step of the wgmma tile engine (csrc/tile_gemm.cuh + EpiConvT in
csrc/encoder_kernels.cuh), and designed operands on which the engine is exact.

What the engine promises, step by step:

1. Weight packing (dad3d_encoder_create): fp16 rows are scaled by 2^s (frexp of the row's max, s <= 15) and the epilogue
   multiplies by 2^-s; every fp32 value is split into P 16-bit pieces by round-to-nearest, the remainder carried in fp32.
   ``c3`` and ``td`` layers get identity columns behind their K axis (piece 0 = 2^s, or 1 for bf16).  The stem's 7x7/2
   filter is re-expressed as a 4x4/1 conv over the 2x2 space-to-depth image (exact: only a re-indexing).
2. Products and accumulator classes: 1 piece: (0,0) -> acc0.  2 pieces: (1,0), (0,1) -> acc1, (0,0) -> acc0.  3 pieces:
   (2,0), (0,2), (1,1), (1,0), (0,1) -> acc1, (0,0) -> acc0.  Residual-in-K blocks: residual pieces x identity piece 0,
   piece 0 into acc0, the others into acc1.  A projection-shortcut segment uses the full list.
3. Each class is summed exactly: the model asserts that every term lies on one grid and that sum |terms| < 2^24 x grid,
   which makes every partial sum an fp32 number whatever order the tensor core adds in.
4. The epilogue in fp32, in kernel order: fp32(acc0 + acc1) (n_acc = 2 only); fmaf(x, 2^-s, b) for fp16 or x + b for
   bf16; residual add or gate multiply with the operand's pieces summed smallest first; ReLU; RN split into pieces (fp16:
   cvt.rn.satfinite, so +-65504 saturates; bf16: RNE).  fp32 outputs (heat map, MLP) stop after ReLU.
5. Reading a piece tensor back sums its pieces smallest first (exact for canonical splits).

The mutation hooks (``Mutation``) exist so that the CPU tests can prove the designed data sees each kind of fault.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Tuple

import numpy as np
import scipy.sparse as sp

MODES = {"fp32": (3, False), "bf16x2": (2, False), "bf16": (1, False), "fp16x2": (2, True), "fp16": (1, True)}
F16_MAX = np.float32(65504.0)
BLOCK_K = 64


def products(P: int) -> List[Tuple[int, int, int]]:
    """(A piece, B piece, accumulator) of every tensor-core product, as dad3d_encoder_create lists them."""
    if P == 1:
        return [(0, 0, 0)]
    if P == 2:
        return [(1, 0, 1), (0, 1, 1), (0, 0, 0)]
    return [(2, 0, 1), (0, 2, 1), (1, 1, 1), (1, 0, 1), (0, 1, 1), (0, 0, 0)]


def n_acc(P: int) -> int:
    return 1 if P == 1 else 2


# ----------------------------------------------------------------------------------------------------------- rounding
def rn_bf16(x) -> np.ndarray:
    """fp32 -> nearest bf16 (ties to even), as an fp32 array."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def rz_bf16(x) -> np.ndarray:
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def rn_f16_sat(x) -> np.ndarray:
    """cvt.rn.satfinite.f16.f32 as an fp32 array."""
    return np.clip(np.asarray(x, np.float32), -F16_MAX, F16_MAX).astype(np.float16).astype(np.float32)


def rz_f16_sat(x) -> np.ndarray:
    x = np.clip(np.asarray(x, np.float32), -F16_MAX, F16_MAX)
    r = x.astype(np.float16).astype(np.float32)
    over = np.abs(r) > np.abs(x)                                   # rounded away from zero: step back one fp16 ulp
    r16 = r.astype(np.float16)
    r[over] = np.nextafter(r16[over], np.float16(0)).astype(np.float32)
    return r


def split(x, P: int, fp16: bool, trunc: bool = False) -> List[np.ndarray]:
    """The library's piece split: P rounds of (piece = round16(r); r -= piece) in fp32."""
    r = np.asarray(x, np.float32).copy()
    out = []
    for _ in range(P):
        if fp16:
            p = rz_f16_sat(r) if trunc else rn_f16_sat(r)
        else:
            p = rz_bf16(r) if trunc else rn_bf16(r)
        out.append(p)
        r = (r - p).astype(np.float32)
    return out


def sum_pieces(pieces: List[np.ndarray]) -> np.ndarray:
    """What read_activation returns: the pieces summed in fp32, smallest first."""
    s = np.zeros_like(pieces[0], dtype=np.float32)
    for p in reversed(pieces):
        s = (s + p).astype(np.float32)
    return s


def grid_of(x) -> float:
    """Largest power of two that divides every non-zero element (inf for an all-zero array)."""
    a = np.abs(np.asarray(x, np.float64))
    a = a[a != 0]
    if a.size == 0:
        return float("inf")
    m, e = np.frexp(a)
    mi = (m * 2.0 ** 53).astype(np.int64)
    low = mi & -mi
    return float(np.min(np.ldexp(low.astype(np.float64), (e - 53).astype(np.int64))))


# ----------------------------------------------------------------------------------------------------- weight packing
@dataclasses.dataclass
class Packed:
    pieces: List[np.ndarray]       # P x [cout, R, S, cin] fp32 (scaled by 2^s for fp16)
    scale: np.ndarray              # [cout] 2^-s
    up: np.ndarray                 # [cout] 2^s
    ident: Optional[np.ndarray]    # [cout] identity entry (piece 0) for residual-in-K layers, else None


def has_identity(name: str) -> bool:
    return len(name) > 4 and ((name.endswith("c3") and not name.endswith("u1c3")) or name.endswith("td"))


def stem_to_4x4(w7: np.ndarray) -> np.ndarray:
    """[64, 7, 7, 3] -> [64, 4, 4, 16]: tap (r, dx) over s2d channel (py*2 + px)*3 + c is the 7x7 tap (2r + py - 1,
    2dx + px - 1); channels 12..15 are zero."""
    w4 = np.zeros((w7.shape[0], 4, 4, 16), np.float32)
    for r in range(4):
        for dx in range(4):
            for py in range(2):
                for px in range(2):
                    ky, kx = 2 * r + py - 1, 2 * dx + px - 1
                    if 0 <= ky <= 6 and 0 <= kx <= 6:
                        w4[:, r, dx, (py * 2 + px) * 3:(py * 2 + px) * 3 + 3] = w7[:, ky, kx, :]
    return w4


def pack(name: str, w: np.ndarray, P: int, fp16: bool, trunc: bool = False) -> Packed:
    w = np.asarray(w, np.float32)
    if name == "stem":
        w = stem_to_4x4(w)
    cout = w.shape[0]
    up = np.ones(cout, np.float32)
    if fp16:
        amax = np.abs(w.reshape(cout, -1)).max(axis=1).astype(np.float32)
        _, e = np.frexp(amax)
        e = np.where(amax > 0, np.maximum(np.minimum(15, 15 - e), -100), 0)
        up = np.ldexp(np.float32(1), e).astype(np.float32)
    scale = (np.float32(1) / up).astype(np.float32)
    r = (w * up[:, None, None, None]).astype(np.float32)
    pieces = split(r, P, fp16, trunc)
    ident = None
    if has_identity(name) and w.shape[1] == 1 and w.shape[2] == 1:
        ident = rn_f16_sat(up) if fp16 else np.ones(cout, np.float32)
    return Packed(pieces, scale, up, ident)


# --------------------------------------------------------------------------------------------------------- the step
@dataclasses.dataclass
class Mutation:
    """Deliberate faults of the model (the CPU tests check that designed data sees each one)."""
    drop_product: Optional[int] = None       # index into products(P)
    trunc_acc_sum: bool = False              # fp32(acc0 + acc1) rounded toward zero
    trunc_split: bool = False                # output piece split by truncation
    bias_before_scale: bool = False          # (x + b) * 2^-s
    skip_last_kblock: bool = False           # the last 64-wide block of the packed K axis is never multiplied
    shift_tap: bool = False                  # tap 0 reads the input one pixel to the right
    no_identity: bool = False                # residual-in-K blocks dropped


@dataclasses.dataclass
class ConvSpec:
    """One conv step, as the plan describes it (Dad3dEncoder.describe_plan())."""
    name: str
    R: int
    S: int
    stride: int = 1
    pad_h: int = 0
    pad_w: int = 0
    Ho: int = 0
    Wo: int = 0
    relu: bool = False
    res_mode: int = 0          # 1: residual (in K for identity layers), 2: gate multiply, 4: second 1x1 source
    res_stride: int = 1
    parity: int = 0            # 1 + 2a + b
    up2: bool = False
    f32_out: bool = False
    stem: bool = False


def spec_from_step(st: dict) -> ConvSpec:
    """ConvSpec of a conv step of describe_plan()."""
    ti = st["in"]
    stem = bool(st["stem"])
    R, S = st["R"], st["S"]
    if stem:
        R, S = 4, 4
        pad_h, pad_w = 2, 0
        Ho, Wo = ti["H"], ti["W"] - 4
    elif st["parity"]:
        pad_h = pad_w = 0
        Ho, Wo = ti["H"] // 2, ti["W"] // 2
    else:
        pad_h = pad_w = st["pad"]
        Ho = (ti["H"] + 2 * st["pad"] - R) // st["stride"] + 1
        Wo = (ti["W"] + 2 * st["pad"] - S) // st["stride"] + 1
    return ConvSpec(name=st["layer"], R=R, S=S, stride=st["stride"], pad_h=pad_h, pad_w=pad_w, Ho=Ho, Wo=Wo,
                    relu=bool(st["relu"]), res_mode=st["res_mode"], res_stride=st["res_stride"], parity=st["parity"],
                    up2=bool(st["up2"]), f32_out="out" not in st, stem=stem)


def gather(x, n, h, w) -> np.ndarray:
    """x[n, h, w] -> fp32 numpy [len(n), C] for a numpy array or a (device) torch tensor [N, H, W, C]."""
    if isinstance(x, np.ndarray):
        return x[n, h, w].astype(np.float32)
    import torch
    idx = [torch.as_tensor(np.asarray(v), device=x.device) for v in (n, h, w)]
    return x[idx[0], idx[1], idx[2]].float().cpu().numpy()


def _im2col(x, pix: np.ndarray, spec: ConvSpec, mut: Mutation) -> np.ndarray:
    """Values of x [N, H, W, C] -> fp32 [len(pix), R*S*C] for output pixels pix [M, 3] (n, h, w); zero outside the
    image."""
    N, H, W, Cc = x.shape
    n, h, w = pix[:, 0], pix[:, 1], pix[:, 2]
    cols = []
    for r in range(spec.R):
        for s in range(spec.S):
            if spec.parity:
                a, b = (spec.parity - 1) >> 1, (spec.parity - 1) & 1
                ih, iw = 2 * h + a, 2 * w + b
            else:
                ih = h * spec.stride + r - spec.pad_h
                iw = w * spec.stride + s - spec.pad_w
            if mut.shift_tap and r == 0 and s == 0:
                iw = iw + 1
            ok = (ih >= 0) & (ih < H) & (iw >= 0) & (iw < W)
            v = np.zeros((len(pix), Cc), np.float32)
            if ok.any():
                v[ok] = gather(x, n[ok], ih[ok], iw[ok])
            cols.append(v)
    return np.concatenate(cols, axis=1)


def conv_step(spec: ConvSpec, packed: Packed, bias: np.ndarray, x, pix: np.ndarray, P: int, fp16: bool, res=None,
              src2=None, mut: Mutation = Mutation()) -> np.ndarray:
    """Output values (as read back) of one conv step at output pixels pix [M, 3] (n, h, w of the layer's output grid),
    all cout_pad channels -> fp32 [M, cout_pad].

    x: the input tensor's values [N, H, W, C_in_stored] (numpy, or a torch tensor on the device: only the pixels the
    sampled outputs read are fetched); res: the residual / gate tensor (at the output grid, or the half-resolution grid
    for parity steps); src2: the projection shortcut's input.  Every operand is split into pieces with the library's
    split, so the values must be designed canonical (assert_canonical)."""
    cout = packed.pieces[0].shape[0]
    cout_pad = bias.shape[0]
    Ci = x.shape[3]
    wk = []                                                       # P x [K, cout] sparse, K laid out (tap, channel)
    for q in packed.pieces:
        R, S, cin = q.shape[1:]
        # (a projection shortcut's weights are K-concatenated: [W | W2] over [main ; second source] channels)
        full = np.zeros((cout, R, S, Ci + (src2.shape[3] if src2 is not None else 0)), np.float64)
        full[..., :cin] = q
        full = full.reshape(cout, -1)
        if mut.skip_last_kblock and packed.ident is None:
            full[:, -BLOCK_K:] = 0
        wk.append(sp.csr_matrix(full.T))
    a = _im2col(x, pix, spec, mut)
    if src2 is not None:
        rs = spec.res_stride
        a = np.concatenate([a, gather(src2, pix[:, 0], pix[:, 1] * rs, pix[:, 2] * rs)], axis=1)
    A = [q.astype(np.float64) for q in split(a, P, fp16)]
    M = len(pix)
    acc = [np.zeros((M, cout), np.float64), np.zeros((M, cout), np.float64)]
    mag = [np.zeros((M, cout), np.float64), np.zeros((M, cout), np.float64)]
    grids = [float("inf"), float("inf")]
    for i, (pa, pb, ac) in enumerate(products(P)):
        if mut.drop_product == i:
            continue
        acc[ac] += (wk[pb].T @ A[pa].T).T
        mag[ac] += (abs(wk[pb]).T @ np.abs(A[pa]).T).T
        grids[ac] = min(grids[ac], grid_of(A[pa]) * grid_of(wk[pb].data))
    res_pieces = split(gather(res, pix[:, 0], pix[:, 1], pix[:, 2]), P, fp16) if res is not None else None
    if packed.ident is not None and spec.res_mode == 1 and not mut.no_identity:
        # residual pieces x identity piece 0, smallest first; piece 0 -> acc0, the others -> acc1 (n_acc = 2)
        if res_pieces is None:
            raise ValueError(f"{spec.name}: residual-in-K layer without a residual")
        for p in reversed(range(P)):
            rv = res_pieces[p][:, :cout].astype(np.float64)
            ident = packed.ident.astype(np.float64)
            if mut.skip_last_kblock:                             # the identity block is the last k-block here
                ident = ident.copy()
                ident[max(0, cout_pad - BLOCK_K):] = 0
            term = rv * ident[None, :]
            ac = 0 if p == 0 or n_acc(P) == 1 else 1
            acc[ac] += term
            mag[ac] += np.abs(term)
            grids[ac] = min(grids[ac], grid_of(rv) * grid_of(ident))
    # the exactness premise: every class on one grid, sum |terms| < 2^24 grid (a mutated model makes no such claim)
    exact = mut == Mutation()
    for c in range(n_acc(P) if exact else 0):
        if np.isfinite(grids[c]):
            assert grids[c] >= 2.0 ** -126, f"{spec.name}: accumulator class {c} grid {grids[c]} below fp32 normals"
            worst = float(mag[c].max() / grids[c])
            assert worst < 2.0 ** 24, f"{spec.name}: accumulator class {c} not exact (sum |terms| = {worst:.3g} grid)"
    a0 = acc[0].astype(np.float32)
    a1 = acc[1].astype(np.float32)
    assert not exact or (np.array_equal(a0.astype(np.float64), acc[0]) and np.array_equal(a1.astype(np.float64), acc[1]))
    pad = np.zeros((M, cout_pad - cout), np.float32)
    a0 = np.concatenate([a0, pad], axis=1)
    a1 = np.concatenate([a1, pad], axis=1)
    # ---- epilogue, fp32, kernel order
    if n_acc(P) == 2:
        x = a0 + a1
        if mut.trunc_acc_sum:
            s64 = a0.astype(np.float64) + a1.astype(np.float64)
            away = np.abs(x.astype(np.float64)) > np.abs(s64)
            x[away] = np.nextafter(x[away], np.float32(0))
    else:
        x = a0
    scale = np.concatenate([packed.scale, np.ones(cout_pad - cout, np.float32)])
    b = bias.astype(np.float32)[None, :]
    if fp16:
        assert not exact or np.all((x == 0) | (np.abs(x * scale) >= np.float32(2.0 ** -126))), "scaled acc subnormal"
        x = (x + b) * scale if mut.bias_before_scale else x * scale + b     # x * 2^-s is exact: fmaf == one rounding
    else:
        x = x + b
    if spec.res_mode in (1, 2) and packed.ident is None and not spec.f32_out:
        r = sum_pieces(res_pieces)
        x = x + r if spec.res_mode == 1 else x * r
    if spec.relu:
        x = np.maximum(x, np.float32(0))
    x = x.astype(np.float32)
    if spec.f32_out:
        return x
    return sum_pieces(split(x, P, fp16, trunc=mut.trunc_split))


def stored_pixels(spec: ConvSpec, pix: np.ndarray) -> List[np.ndarray]:
    """Where the output of computed pixel pix is stored in the output tensor: up2 -> four pixels, parity -> one pixel of
    the full-resolution grid, otherwise the pixel itself."""
    n, h, w = pix[:, 0], pix[:, 1], pix[:, 2]
    if spec.up2:
        return [np.stack([n, 2 * h + a, 2 * w + b], 1) for a in (0, 1) for b in (0, 1)]
    if spec.parity:
        a, b = (spec.parity - 1) >> 1, (spec.parity - 1) & 1
        return [np.stack([n, 2 * h + a, 2 * w + b], 1)]
    return [pix]


def sample_pixels(N: int, Ho: int, Wo: int, tw: int, th: int, tn: int, rows: Optional[List[int]] = None,
                  limit: int = 4096, n_random: int = 384, seed: int = 0) -> np.ndarray:
    """Output pixels to check: all of them when there are at most ``limit``; otherwise every pixel of the last
    (partial) tile along each dimension, the image borders of the first and last image, and a seeded random sample.
    ``rows`` restricts to the computed rows (sparse heat map)."""
    hs = np.arange(Ho) if rows is None else np.asarray(sorted(set(rows)))
    if N * len(hs) * Wo <= limit:
        g = np.stack(np.meshgrid(np.arange(N), hs, np.arange(Wo), indexing="ij"), -1).reshape(-1, 3)
        return g
    sel = set()
    ws = np.arange(Wo)
    last_w = range(((Wo - 1) // tw) * tw, Wo)
    last_h = [h for h in hs if h >= ((Ho - 1) // th) * th]
    last_n = range(((N - 1) // tn) * tn, N)
    for n in {0, N - 1}:
        for h in hs:
            for w in (0, Wo - 1):
                sel.add((n, h, w))
        for h in {hs[0], hs[-1]}:
            for w in ws:
                sel.add((n, h, w))
    for n in {0, N - 1}:
        for h in hs:
            for w in last_w:
                sel.add((n, h, w))
        for h in last_h:
            for w in ws:
                sel.add((n, h, w))
    for n in last_n:
        for h in (hs[0], hs[len(hs) // 2], hs[-1]):
            for w in (0, Wo // 2, Wo - 1):
                sel.add((n, h, w))
    rng = np.random.default_rng(seed)
    for _ in range(n_random):
        sel.add((int(rng.integers(N)), int(hs[rng.integers(len(hs))]), int(rng.integers(Wo))))
    return np.asarray(sorted(sel), np.int64)


# ------------------------------------------------------------------------------------------------- designed operands
# Pieces of a designed value: piece p = +-m_p * 2^(k - 9p) (bf16) or 2^(k - 12p) (fp16) with m_p in [9, 15]: each
# piece is a 4-bit number below half an ulp of the one before, so the RN split reproduces them (canonical), the value is an
# fp32 number (<= 22 bits), and every piece is non-zero.
PIECE_STEP = {False: 9, True: 12}


def designed_mantissas(rng, shape, P: int) -> List[np.ndarray]:
    """Signed 4-bit mantissas +-(9..15) of each piece (9..15: the value stays inside the binade of piece 0)."""
    return [(rng.integers(9, 16, size=shape, dtype=np.int8) * np.where(rng.random(shape) < 0.5, -1, 1).astype(np.int8))
            for _ in range(P)]


def designed_values(rng, shape, P: int, fp16: bool, k, mant: Optional[List[np.ndarray]] = None
                    ) -> Tuple[np.ndarray, List[np.ndarray]]:
    """-> (fp32 values, their P designed pieces).  k: exponent of piece 0 (scalar, or broadcastable to shape); mant:
    mantissas from designed_mantissas (drawn here when absent)."""
    if mant is None:
        mant = designed_mantissas(rng, shape, P)
    k = np.asarray(k)
    pieces = []
    for p in range(P):
        pieces.append(np.ldexp(mant[p].astype(np.float32), (k - PIECE_STEP[fp16] * p).astype(np.int32)))
    x = pieces[-1].astype(np.float64) if P else np.zeros(shape)
    for pc in reversed(pieces[:-1]):
        x += pc
    x32 = x.astype(np.float32)
    assert np.array_equal(x32.astype(np.float64), x)
    return x32, pieces


def assert_canonical(x: np.ndarray, pieces: List[np.ndarray], P: int, fp16: bool) -> None:
    got = split(x, P, fp16)
    for p in range(P):
        assert np.array_equal(got[p], pieces[p]), f"piece {p} of the designed values is not the RN split"


# exponent of piece 0 of activations / weights per mode: weights are scaled to [2^14, 2^15) for fp16, so the fp16 rows get a
# per-row exponent 14 - s with s in S_RANGE
K_ACT = 0
K_W_BF16 = -8
S_RANGE = (8, 13)


def design_weights(rng, name: str, cout: int, R: int, S: int, cin: int, P: int, fp16: bool, nnz: int = 6):
    """Sparse designed weights [cout, R, S, cin]: row o touches nnz (tap, 64-channel block) k-blocks, chosen so that any
    64 consecutive rows cover every k-block of the layer; mixed signs; every piece of every non-zero present.
    -> (fp32 weights, per-row exponent of piece 0 in the real domain)."""
    w = np.zeros((cout, R, S, cin), np.float32)
    cb = (cin + 63) // 64
    nkb = R * S * cb
    if fp16:
        s = rng.integers(S_RANGE[0], S_RANGE[1], size=cout)
        kw = 11 - s                                               # scaled piece 0 in [2^14, 2^15)
    else:
        kw = np.full(cout, K_W_BF16)
    for o in range(cout):
        for j in range(nnz):
            kb = (o * nnz + j) % nkb
            tap, c = divmod(kb, cb)
            ch = c * 64 + int(rng.integers(min(64, cin - c * 64)))
            v, _ = designed_values(rng, (), P, fp16, int(kw[o]))
            w[o, tap // S, tap % S, ch] = v
    return w, kw


def design_stem(rng, P: int, fp16: bool, nnz: int = 6):
    """Designed 7x7x3 -> 64 stem weights: every row touches taps of all four 4x4 row taps (r = (ky + 1) // 2)."""
    w = np.zeros((64, 7, 7, 3), np.float32)
    if fp16:
        kw = 11 - rng.integers(S_RANGE[0], S_RANGE[1], size=64)
    else:
        kw = np.full(64, K_W_BF16)
    for o in range(64):
        kys = [(o + j) % 7 for j in range(nnz)]
        for ky in kys:
            kx, c = int(rng.integers(7)), int(rng.integers(3))
            v, _ = designed_values(rng, (), P, fp16, int(kw[o]))
            w[o, ky, kx, c] = v
    return w, kw


def design_bias(rng, cout: int, fp16: bool, kw: np.ndarray, saturate: bool = False) -> np.ndarray:
    """Mixed-sign biases about the size of a designed output (so that ReLU clips some outputs and keeps others); with
    saturate, every eighth channel gets +-1e5, past the fp16 range."""
    m = rng.integers(1, 16, size=cout) * np.where(rng.random(cout) < 0.5, -1, 1)
    e = (kw + 1) if fp16 else np.full(cout, K_W_BF16 + 3)
    b = np.ldexp(m.astype(np.float64), e.astype(np.int64)).astype(np.float32)
    if saturate:
        b[::8] = np.where(rng.random(b[::8].shape) < 0.5, -1e5, 1e5)
    return b


def residual_exponent(fp16: bool, kw: np.ndarray) -> np.ndarray:
    """Exponent of piece 0 of a designed residual channel: the size of the conv output it is added to (for fp16 the
    residual also rides the identity column 2^s, so it follows the row's scale)."""
    return (kw + 2) if fp16 else np.full(kw.shape, K_ACT + K_W_BF16 + 4)


def design_tensor(rng, shape, P: int, fp16: bool, k=K_ACT, valid_c: Optional[int] = None, mant=None):
    """Designed activation [N, H, W, C] (channels >= valid_c zero) -> (fp32 values, pieces)."""
    x, pieces = designed_values(rng, shape, P, fp16, k, mant)
    if valid_c is not None and valid_c < shape[-1]:
        x[..., valid_c:] = 0
        for pc in pieces:
            pc[..., valid_c:] = 0
    assert_canonical(x, pieces, P, fp16)
    return x, pieces


def design_network(rng, shapes: List[Tuple[str, Tuple[int, int, int, int]]], mode: str, saturate: bool = False):
    """Designed folded records for every layer: -> (layers [(name, w, b)], {name: per-row exponent of piece 0})."""
    P, fp16 = MODES[mode]
    layers, kws = [], {}
    for name, (cout, R, S, cin) in shapes:
        if name == "stem":
            w, kw = design_stem(rng, P, fp16)
        else:
            w, kw = design_weights(rng, name, cout, R, S, cin, P, fp16)
        b = design_bias(rng, cout, fp16, kw, saturate=saturate and name not in ("heat", "mlp2"))
        layers.append((name, w, b))
        kws[name] = kw
    return layers, kws
