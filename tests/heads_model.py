"""Exact numpy model of csrc/heads.cu: the regression heads' forward and weight gradients, every fp32 rounding in the
kernels' order (fma by round-to-odd, as tests/metrics_model.fma32), and Philox4x32-10 for the dropout mask.

tanhf is not restated: it lowers to MUFU.EX2 / MUFU.RCP for larger |x|.  The forward returns the logits o; the caller supplies
y = tanh(o) (the kernel's saved y, checked within 2 ulp of fp64 tanh and exactly where tanh is +-1), and everything downstream
of y is exact.
"""
import numpy as np

from tests.metrics_model import fma32

f32, f64 = np.float32, np.float64
FEAT, HID, HID_ALL, OUT, SHAPE, PARAMS, LMS = 2048, 512, 1536, 549, 403, 413, 136
HEAD_ROWS = (403, 10, 136)
FC1_SPLITS, FC2_SPLITS = 8, 4
MASK_WORDS, OUT_WORDS = 48, 18
_M = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Random123 philox4x32 with 10 rounds; ctr: 4 uint32 arrays, key: 2 uint32 arrays -> 4 uint32 arrays."""
    c = [np.asarray(x, np.uint64) & _M for x in ctr]
    k0, k1 = (np.asarray(x, np.uint64) & _M for x in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & _M, (k1 + 0xBB67AE85) & _M
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M]
    return [x.astype(np.uint32) for x in c]


def keep_prob(p):
    return f32(1.0 - p)


def dropout_scale(train, p):
    """torch's dropout scale: fp32(1 / (1 - p)) computed in fp64 (pinned in tests/test_heads_model_cpu.py)."""
    return f32(1.0 / (1.0 - p)) if train else f32(1.0)


def keep_mask(B, seed, counter, p):
    """[B, 1536] bool: Philox4x32-10 at key (seed lo, hi), counter (counter lo, hi, row * 1536 + column, 0), word 0 x;
    kept iff fp32(x >> 8) * 2^-24 < fp32(1 - p)."""
    i = np.arange(B * HID_ALL, dtype=np.uint64)
    z = np.zeros_like(i)
    x = philox4x32_10((z + (counter & _M), z + (counter >> 32), i, z), (z + (seed & _M), z + (seed >> 32)))[0]
    u = (x >> 8).astype(f32) * f32(2.0 ** -24)
    return (u < keep_prob(p)).reshape(B, HID_ALL)


def pack_bits(m):
    """[B, 32 w] bool -> [B, w] uint32, bit j of word w = column 32 w + j (the kernels' ballots)."""
    B, n = m.shape
    w = -(-n // 32)
    mm = np.zeros((B, w * 32), bool)
    mm[:, :n] = m
    return (mm.reshape(B, w, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)


def unpack_bits(words, n):
    words = np.asarray(words, np.uint32)
    return ((words[..., None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(words.shape[0], -1)[:, :n]


def _fma_acc(p, c):
    """fp32(p + c) rounded once, for an exact fp64 product p and fp64 c holding an fp32 value (fma32's round-to-odd)."""
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    bits = s.view(np.int64)
    adj = (e != 0) & ((bits & 1) == 0)
    bits += np.where(adj, np.where((e > 0) == (s > 0), 1, -1), 0)
    return s.astype(f32).astype(f64)


def gemm(A, Bk, kchunk):
    """heads_gemm_kernel: A [M, K], Bk [K, N] -> [S, M, N] fp32, split s the fma chain over k in [s kchunk, (s + 1) kchunk)
    in increasing k from +0."""
    A = np.asarray(A, f32).astype(f64)
    Bk = np.asarray(Bk, f32).astype(f64)
    M, K = A.shape
    S = -(-K // kchunk)
    out = np.zeros((S, M, Bk.shape[1]), f32)
    for s in range(S):
        acc = np.zeros((M, Bk.shape[1]), f64)
        for k in range(s * kchunk, min(K, (s + 1) * kchunk)):
            acc = _fma_acc(A[:, k, None] * Bk[None, k, :], acc)
        out[s] = acc
    return out


def sum_splits(parts, bias):
    s = parts[0].copy()
    for p in parts[1:]:
        s = s + p
    return s + np.asarray(bias, f32)


def column_total(x):
    """heads_dout_kernel / heads_dhidden_kernel: per row lane w (rows w, w + 8, ...) a sum in row order from +0, then the
    8 lane sums in order."""
    x = np.asarray(x, f32)
    lanes = []
    for w in range(8):
        acc = np.zeros(x.shape[1], f32)
        for b in range(w, x.shape[0], 8):
            acc = acc + x[b]
        lanes.append(acc)
    s = lanes[0]
    for a in lanes[1:]:
        s = s + a
    return s


def _blocks():
    r0 = 0
    for hd, n in enumerate(HEAD_ROWS):
        yield hd, r0, n
        r0 += n


def forward(f, w1, b1, w2, b2, train, p=0.3, seed=0, counter=0):
    """-> dict h, d, mask (words [B,48]), o [B,549] (the pre-epilogue logits), obits [B,18], pose [B,10], landmarks [B,136]."""
    f = np.asarray(f, f32)
    B = f.shape[0]
    h = np.fmax(sum_splits(gemm(f, np.asarray(w1, f32).T, FEAT // FC1_SPLITS), b1), f32(0))
    keep = keep_mask(B, seed, counter, p) if train else np.ones((B, HID_ALL), bool)
    d = np.where(keep, h * dropout_scale(train, p), f32(0)).astype(f32)
    parts = np.zeros((FC2_SPLITS, B, OUT), f32)
    for hd, r0, n in _blocks():
        parts[:, :, r0:r0 + n] = gemm(d[:, hd * HID:(hd + 1) * HID], np.asarray(w2, f32)[r0:r0 + n].T, HID // FC2_SPLITS)
    o = sum_splits(parts, b2)
    return dict(h=h, d=d, mask=pack_bits(keep), o=o, obits=pack_bits(o > 0), pose=o[:, SHAPE:PARAMS],
                landmarks=np.fmax(o[:, PARAMS:], f32(0)))


def params(y, o, limit=3.0):
    """[B,413] = [fp32(y * limit) | o]"""
    return np.concatenate([np.asarray(y, f32) * f32(limit), np.asarray(o, f32)[:, SHAPE:PARAMS]], 1)


def dout(dparams, dlms, y, obits, limit=3.0):
    dparams, dlms, y = (np.asarray(x, f32) for x in (dparams, dlms, y))
    g_shape = (dparams[:, :SHAPE] * f32(limit)) * fma32(-y, y, np.ones_like(y))      # torch's tanh_backward
    g_lms = np.where(unpack_bits(obits, OUT)[:, PARAMS:], dlms.reshape(-1, LMS), f32(0))
    return np.concatenate([g_shape, dparams[:, SHAPE:PARAMS], g_lms], 1).astype(f32)


def backward(dparams, dlms, f, w2, h, d, mask, y, obits, train, p=0.3, limit=3.0):
    """-> dw1 [1536,2048], db1 [1536], dw2 [549,512], db2 [549]"""
    f, w2, h, d = (np.asarray(x, f32) for x in (f, w2, h, d))
    B = f.shape[0]
    do = dout(dparams, dlms, y, obits, limit)
    db2 = column_total(do)
    dw2 = np.zeros((OUT, HID), f32)
    dd = np.zeros((B, HID_ALL), f32)
    for hd, r0, n in _blocks():
        dw2[r0:r0 + n] = gemm(do[:, r0:r0 + n].T, d[:, hd * HID:(hd + 1) * HID], B)[0]
        dd[:, hd * HID:(hd + 1) * HID] = gemm(do[:, r0:r0 + n], w2[r0:r0 + n], n)[0]
    kept = unpack_bits(mask, HID_ALL)
    dh = np.where(kept & (h > 0), dd * dropout_scale(train, p), f32(0)).astype(f32)
    db1 = column_total(dh)
    dw1 = gemm(dh.T, f, B)[0]
    return dict(dw1=dw1, db1=db1, dw2=dw2, db2=db2)
