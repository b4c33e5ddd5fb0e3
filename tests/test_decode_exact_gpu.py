"""-m gpu: every decode path checked exactly.  Each test runs one stage of the decoder alone (dad3d_flame_prep /
dad3d_flame_decode_from) on designed operands whose result is fully determined, and compares every output bit for bit with
the exact model in tests/decode_model.py, evaluated on the device in chunks of heads.  Outputs sit inside guarded buffers:
the guard bands in front of and behind them must come back bit-unchanged and no output float may keep its sentinel.

On the real asset and real parameters the default and hi/lo paths are held to an error bound derived from the arithmetic
(test_real_asset_within_derived_bound)."""
import math

import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from oracle.flame_oracle import FLAME_CONSTS, sample_params
from tests import decode_model as dm

pytestmark = pytest.mark.gpu

FLAGS = {"dedicated": 0, "lbs": _lib.DAD3D_BLEND_HILO, "cluster": _lib.DAD3D_BLEND_HILO | _lib.DAD3D_DECODE_CLUSTER,
         "blend": _lib.DAD3D_DECODE_UNFUSED, "simt": _lib.DAD3D_BLEND_SIMT}
MODEL_PATH = {"dedicated": "dedicated", "lbs": "lbs", "cluster": "lbs", "blend": "blend", "simt": "simt"}
GUARD = 64
SENT_OUT = 0x7FC0BEEF         # NaN payloads as int32
SENT_GUARD = 0x7FC0DEAD
CHUNK = 2048                             # heads per model chunk (fp64 intermediates stay within a few GB)

_decoders = {}


def designed(nv, device):
    if nv not in _decoders:
        from dad_3dheads_b200.flame import FlameDecoder
        st = dm.designed_static(nv, seed=nv)
        _decoders[nv] = (FlameDecoder(st, FLAME_CONSTS, device), dm.pack(st).to(device))
    return _decoders[nv]


@pytest.fixture(scope="module")
def real(flame_static, cuda_device):
    from dad_3dheads_b200.flame import FlameDecoder
    return FlameDecoder(flame_static, FLAME_CONSTS, cuda_device), dm.pack(flame_static).to(cuda_device)


class Guarded:
    """An output [B, nv, nc] at `off` floats (0..7) past a GUARD-float band inside a larger buffer."""

    def __init__(self, B, nv, nc, off, device):
        self.n, self.off, self.shape = B * nv * nc, off, (B, nv, nc)
        self.buf = torch.empty(2 * GUARD + 8 + self.n, dtype=torch.float32, device=device)
        bits = self.buf.view(torch.int32)
        bits.fill_(SENT_GUARD)
        bits[GUARD + off:GUARD + off + self.n] = SENT_OUT
        self.out = self.buf[GUARD + off:GUARD + off + self.n].view(self.shape)
        assert (self.out.data_ptr() // 4) % 8 == off

    def check_guards(self, what):
        bits = self.buf.view(torch.int32)
        front, back = bits[:GUARD + self.off], bits[GUARD + self.off + self.n:]
        assert (front == SENT_GUARD).all() and (back == SENT_GUARD).all(), f"{what}: store outside the output"
        left = (self.out.view(torch.int32) == SENT_OUT).nonzero()
        assert left.numel() == 0, f"{what}: output never written at (head, vertex, coordinate) {left[0].tolist()}"


def _first_mismatch(got, want, h0):
    bad = (got.view(torch.int32) != want.view(torch.int32)).nonzero()
    if bad.numel() == 0:
        return None
    h, v, c = bad[0].tolist()
    return (f"{bad.shape[0]} floats differ; first at head {h0 + h}, vertex {v}, coordinate {c}: "
            f"got {got[h, v, c].item()!r}, want {want[h, v, c].item()!r}")


def designed_inputs(B, pk, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    hi, lo = dm.designed_rows(B, g, device)
    return hi, lo, dm.designed_xf(B, g, pk.scale, device)


def rows_for(path, x):
    """fp16 coefficient rows as decode_from expects them: permuted for the dedicated kernel, else padded to 256."""
    x = x.half()
    if path == "dedicated":
        return dm.permute_rows(x)
    return torch.cat([x, torch.zeros(dm.rows_padded(x.shape[0]) - x.shape[0], x.shape[1], dtype=x.dtype, device=x.device)])


def compare_to_model(path, hi, lo, xf, pk, outs, image_size, to_2d, what):
    B = xf.shape[0]
    for h0 in range(0, B, CHUNK):
        sl = slice(h0, min(B, h0 + CHUNK))
        v, p = dm.decode(MODEL_PATH[path], hi[sl], lo[sl], xf[sl], pk, image_size=image_size, to_2d=to_2d)
        for name, got, want in (("vertices", outs[0], v), ("projected", outs[1], p)):
            if got is not None:
                msg = _first_mismatch(got.out[sl], want, h0)
                assert msg is None, f"{what} {name}: {msg}"


def run_designed(dec, pk, path, B, *, to_2d=True, image_size=256.0, want=(True, True), offs=(0, 0), seed=0):
    dev = dec.device
    hi, lo, xf = designed_inputs(B, pk, seed, dev)
    nv = dec.n_vertices
    gv = Guarded(B, nv, 3, offs[0], dev) if want[0] else None
    gp = Guarded(B, nv, 2 if to_2d else 3, offs[1], dev) if want[1] else None
    dec.decode_from(rows_for(path, hi), rows_for(path, lo), xf, flags=FLAGS[path], vertices=gv.out if gv else None,
                    projected=gp.out if gp else None, image_size=image_size, to_2d=to_2d)
    torch.cuda.synchronize()
    what = f"{path} nv={nv} B={B} to_2d={to_2d} image={image_size} offs={offs}"
    for gd in (gv, gp):
        if gd is not None:
            gd.check_guards(what)
    compare_to_model(path, hi, lo, xf, pk, (gv, gp), image_size, to_2d, what)


# ------------------------------------------------------------------------------------------------------- dedicated kernel
SMALL_NV = [1, 2, 3, 4, 5, 6, 7, 8, 63, 64, 65, 96, 97]


def test_vertex_counts_cover_every_phase_and_tile_end():
    """The vertex counts below give every value of 3 nv mod 24, a last tile whose half 1 is empty, and n_tiles == 1."""
    nvs = SMALL_NV + [5023]
    assert {3 * nv % 24 for nv in nvs} == set(range(0, 24, 3))
    assert any(0 < 3 * nv % 192 <= 96 and nv > 64 for nv in nvs) and any(3 * nv <= 192 for nv in nvs)


@pytest.mark.parametrize("nv", SMALL_NV)
def test_dedicated_small_meshes_bit_exact(cuda_device, nv):
    dec, pk = designed(nv, cuda_device)
    for i, B in enumerate((1, 9, 257)):
        run_designed(dec, pk, "dedicated", B, to_2d=bool(i % 2), image_size=(256.0, 224.0)[i % 2],
                     offs=((nv + i) % 8, (nv + 3 * i + 5) % 8), seed=nv * 10 + i)


DEDICATED_B = [1, 7, 8, 9, 33, 255, 256, 257, 1000, 2560, 16897]


@pytest.mark.parametrize("B", DEDICATED_B)
def test_dedicated_full_mesh_bit_exact(cuda_device, B):
    dec, pk = designed(5023, cuda_device)
    d = dec.describe(B, 0)
    (ps,) = d["passes"]
    assert ps["path"] == "dedicated" and ps["rows"] == B
    units = ps["m_units"] * ps["splits"]
    if B == 16897:          # one CTA takes two units with different row tiles
        assert ps["splits"] == 1 and units > ps["grid"] and units % ps["grid"] != 0, ps
    elif B in (1000, 2560):  # split sweeps, more units than CTAs
        assert ps["splits"] > 1 and units > ps["grid"] and units % ps["grid"] != 0, ps
    elif B <= 257:
        assert ps["splits"] > 1, ps
    i = DEDICATED_B.index(B)
    want = {33: (True, False), 255: (False, True)}.get(B, (True, True))
    run_designed(dec, pk, "dedicated", B, to_2d=bool(i % 2), image_size=(256.0, 224.0)[(i // 2) % 2], want=want,
                 offs=(i % 8, (7 - i) % 8), seed=B)


# ---------------------------------------------------------------------------------------------------------- other paths
@pytest.mark.parametrize("path,nv,B", [("lbs", 97, 9), ("lbs", 5023, 1), ("lbs", 5023, 257), ("lbs", 5023, 2560),
                                       ("cluster", 5023, 16897), ("blend", 97, 33), ("blend", 5023, 7),
                                       ("blend", 5023, 4096), ("simt", 97, 33), ("simt", 5023, 7)])
def test_other_paths_bit_exact(cuda_device, path, nv, B):
    dec, pk = designed(nv, cuda_device)
    (ps,) = dec.describe(B, FLAGS[path])["passes"]
    assert ps["path"] == MODEL_PATH[path] and ps["clustered"] == (path == "cluster"), ps
    for i, to_2d in enumerate((True, False)):
        run_designed(dec, pk, path, B, to_2d=to_2d, image_size=(256.0, 224.0)[i], offs=((B + i) % 8, (B + 3 + 2 * i) % 8),
                     seed=B + 7 * i)


def test_decode_from_rejects_more_than_one_pass(cuda_device):
    dec, pk = designed(1, cuda_device)
    for path in ("dedicated", "blend", "simt"):
        chunk = dec.describe(1, FLAGS[path])["fused_chunk"] if path == "dedicated" else 4096
        assert dec.describe(chunk + 1, FLAGS[path])["passes"][1]["rows"] == 1
        B = chunk + 1
        hi = torch.zeros(dm.rows_padded(B), 448, dtype=torch.float16, device=cuda_device)
        xf = torch.zeros(B, 68, device=cuda_device)
        v = torch.zeros(B, 1, 3, device=cuda_device)
        with pytest.raises(_lib.Dad3dError, match="one pass"):
            dec.decode_from(hi, hi, xf, flags=FLAGS[path], vertices=v)


@pytest.mark.parametrize("path", ["dedicated", "lbs", "blend", "simt"])
def test_full_decode_matches_its_stages_with_guarded_stores(cuda_device, path):
    """dad3d_flame_decode over several passes equals prep + decode_from per pass bit for bit, stays inside its outputs,
    writes every float, and launches 2 kernels per pass on the fused paths and 3 on the others."""
    dec, _ = designed(97, cuda_device)
    flags = FLAGS[path]
    d = dec.describe(1, flags)
    chunk = d["fused_chunk"] if path in ("dedicated", "lbs") else 4096
    B = chunk + 300 if path != "simt" else 4096 + 9
    p = sample_params(B, seed=31)
    p[:, :400] *= 0.5
    p = p.to(cuda_device)
    passes = dec.describe(B, flags)["passes"]
    assert len(passes) == 2 and passes[0]["rows"] == chunk
    for i, to_2d in enumerate((True, False)):
        gv, gp = Guarded(B, 97, 3, 3 + i, cuda_device), Guarded(B, 97, 2 if to_2d else 3, 6 - i, cuda_device)
        before = _lib.launch_count()
        dec.decode_into(p, flags=flags, vertices=gv.out, projected=gp.out, image_size=224.0, to_2d=to_2d)
        torch.cuda.synchronize()
        assert _lib.launch_count() - before == 2 * (2 if path in ("dedicated", "lbs") else 3)
        gv.check_guards(path)
        gp.check_guards(path)
        for b0 in range(0, B, chunk):
            q = p[b0:b0 + chunk]
            hi, lo, xf = dec.prep(q, flags=flags, permute=path == "dedicated")
            v = torch.empty(q.shape[0], 97, 3, device=cuda_device)
            pj = torch.empty(q.shape[0], 97, 2 if to_2d else 3, device=cuda_device)
            dec.decode_from(hi, lo, xf, flags=flags, vertices=v, projected=pj, image_size=224.0, to_2d=to_2d)
            assert torch.equal(v.view(torch.int32), gv.out[b0:b0 + chunk].view(torch.int32)), (path, b0)
            assert torch.equal(pj.view(torch.int32), gp.out[b0:b0 + chunk].view(torch.int32)), (path, b0)


# ------------------------------------------------------------------------------------------------------------ prep kernel
def test_prep_rows_bit_exact(real, cuda_device):
    dec, pk = real
    d = dec.describe(1, 0)
    assert d["basis_scale"] == pk.scale and d["jaw_only"] and d["nv"] == 5023
    B = 300
    p = sample_params(B, seed=41).to(cuda_device)
    hi, lo, xf = dec.prep(p)
    want_hi, want_lo = dm.prep_rows(p[:, :400], torch.zeros(B, 36, device=cuda_device))
    cols = torch.cat([torch.arange(0, 400), torch.arange(436, 448)]).to(cuda_device)
    for got, want in ((hi, want_hi), (lo, want_lo)):
        assert torch.equal(got[:B][:, cols].float().view(torch.int32), want[:, cols].view(torch.int32))
    hp, lp, xfp = dec.prep(p, permute=True)
    phys = dm.dec_phys_row(torch.arange(B, device=cuda_device))
    assert hp.shape[0] == dm.rows_padded(B) and torch.equal(hp[phys], hi[:B]) and torch.equal(lp[phys], lo[:B])
    assert torch.equal(xfp, xf)


def _signed_axes(g, B):
    """6-D rotation inputs whose two 3-vectors are distinct signed unit axes, and the signed permutation they give."""
    r6 = np.zeros((B, 6), np.float32)
    R6 = np.zeros((B, 3, 3), np.float32)
    for b in range(B):
        i, j = g.choice(3, 2, replace=False)
        si, sj = g.choice([-1.0, 1.0], 2)
        b1 = np.eye(3)[i] * si
        vy = np.eye(3)[j] * sj
        b3 = np.cross(b1, vy)
        b2 = -np.cross(b1, b3)
        r6[b, :3], r6[b, 3:] = b1, vy
        R6[b] = np.stack([b1, b2, b3], 1)                 # columns b1, b2, b3
    return r6, R6


def test_prep_designed_poses_are_exact(cuda_device):
    """Zero jaw and signed-axis 6-D vectors: every joint transform is R6 / basis_scale with zero translation, exactly."""
    dec, pk = designed(97, cuda_device)
    B = 64
    g = np.random.default_rng(5)
    p = torch.zeros(B, 413)
    r6, R6 = _signed_axes(g, B)
    p[:, 403:409] = torch.from_numpy(r6)
    p[:, 409:411] = torch.rand(B, 2, generator=torch.Generator().manual_seed(1)) - 0.5
    p[:, 412] = torch.rand(B, generator=torch.Generator().manual_seed(2)) - 0.5
    _, _, xf = dec.prep(p.to(cuda_device))
    xf = xf.cpu().view(B, 68)
    AR = torch.from_numpy(R6) * np.float32(1.0 / pk.scale)
    for j in range(5):
        A = xf[:, 12 * j:12 * j + 12].view(B, 3, 4)
        assert torch.equal(A[..., :3], AR), j
        assert (A[..., 3] == 0).all(), j
    assert torch.equal(xf[:, 60:63], torch.from_numpy(R6[:, :, 2]) * np.float32(0.05))
    assert torch.equal(xf[:, 63], torch.clamp(p[:, 412] + 1.0, min=1e-8)) and torch.equal(xf[:, 64:66], p[:, 409:411])
    assert (xf[:, 66:] == 0).all()


def test_prep_group_size_does_not_change_results(real, cuda_device):
    """Big batches run 32 heads per warp, small ones one: same arithmetic in the same order, bit-identical."""
    dec, _ = real
    n_big = 32 * 8 * dec.describe(1, 0)["num_sms"]
    p = sample_params(n_big + 5, seed=43).to(cuda_device)
    hi, lo, xf = dec.prep(p)
    half = (n_big + 5) // 2
    for a, b in ((0, half), (half, n_big + 5)):
        h2, l2, x2 = dec.prep(p[a:b])
        assert torch.equal(h2[:b - a], hi[a:b]) and torch.equal(l2[:b - a], lo[a:b]) and torch.equal(x2, xf[a:b])


def test_prep_records_within_ulp_bound(real, flame_static, cuda_device):
    """Real asset, sample_params: the jaw-dependent part of the prep kernel against the fp64 restatement
    dm.prep_records (joint constants rounded to fp32 as the library stores them).  With u = 2^-24 and cond = 1 + |vy| /
    |b1 x vy| (the 6-D Gram-Schmidt amplification), per element:
      pose features (rows 400..435, hi + lo)   |f - f64| <= 32 u + 2^-22 |f64| + 2^-25   (fp16 hi/lo split of an fp32 value)
      rotation parts of the five transforms     <= 32 u cond / basis_scale
      translation parts                         <= 32 u cond max|J|   (J = the head's joints)
      offset c = R6 (0, 0, 0.05)                <= 32 u cond 0.05
      scale, tx, ty                             exact
    and the features of the unposed joints 1, 3, 4 are exactly zero."""
    dec, pk = real
    B = 512
    p = sample_params(B, seed=61)
    hi, lo, xf = dec.prep(p.to(cuda_device))
    f64, r64, cond, J = dm.prep_records(p.to(cuda_device), flame_static, pk.scale)
    u = 2.0 ** -24
    feats = hi[:B, 400:436].double() + lo[:B, 400:436].double()
    jaw = slice(9, 18)
    assert (hi[:B, 400:436][:, list(range(9)) + list(range(18, 36))] == 0).all()
    assert (lo[:B, 400:436][:, list(range(9)) + list(range(18, 36))] == 0).all()
    err = (feats - f64).abs()
    bound = 32 * u + 2.0 ** -22 * f64.abs() + 2.0 ** -25
    assert (err <= bound).all(), f"pose features: worst excess {(err - bound).max().item():.3g} at {(err - bound).argmax().item()}"
    assert (f64[:, jaw].abs() > 1e-3).any()               # the jaw really is posed
    x = xf.double()
    rot = [12 * i + 4 * r + k for i in range(5) for r in range(3) for k in range(3)]
    tr = [12 * i + 4 * r + 3 for i in range(5) for r in range(3)]
    mj = J.abs().amax((1, 2))
    for name, cols, scale in (("rotation", rot, torch.full_like(mj, 1.0 / pk.scale)), ("translation", tr, mj),
                              ("offset", list(range(60, 63)), torch.full_like(mj, 0.05))):
        e = (x[:, cols] - r64[:, cols]).abs() / (u * cond[:, None] * scale[:, None])
        assert e.max().item() <= 32, f"{name}: {e.max().item():.3g} ulp-units at head {e.amax(1).argmax().item()}"
    assert torch.equal(xf[:, 63:66], r64[:, 63:66].float()) and (xf[:, 66:] == 0).all()


# -------------------------------------------------------------------------------------------- real asset, derived bound
@pytest.mark.parametrize("path", ["dedicated", "lbs"])
def test_real_asset_within_derived_bound(real, cuda_device, path):
    """Real asset, real parameters, the device's own prep rows.  Reference: the fp64 epilogue over an fp64 product of the
    same fp16 operands (the path's own product list).  Per element
        |v - v64| <= (|wr| |R_row|_1 + |wj| |J_row|_1) (gamma_448 S + u max|p|) + 6 u M
    with u = 2^-24, gamma_n = n 2^-23 / (1 - n 2^-23) (truncating accumulation), S = max over the vertex's three columns of
    sum_k |a_k b_k|, and M = |wr| (sum |R_rc p_c| + |t_r|) + |wj| (same for J) + |c_r| (at most five fmaf roundings);
    the projection adds its three roundings: (fmaf(v, sc, t) + 1) * hs."""
    dec, pk = real
    B = 96
    p = sample_params(B, seed=51).to(cuda_device)
    hi, lo, xf = dec.prep(p, flags=FLAGS[path], permute=path == "dedicated")
    v = torch.empty(B, 5023, 3, device=cuda_device)
    pj = torch.empty(B, 5023, 3, device=cuda_device)
    dec.decode_from(hi, lo, xf, flags=FLAGS[path], vertices=v, projected=pj, to_2d=False)
    if path == "dedicated":
        idx = dm.dec_phys_row(torch.arange(B, device=cuda_device))
        hi, lo = hi[idx], lo[idx]
    else:
        hi, lo = hi[:B], lo[:B]
    a_hi, a_lo, b_hi, b_lo = hi.double(), lo.double(), pk.hi.double(), pk.lo.double()
    terms = [(a_hi, b_hi)] + ([(a_lo, b_hi), (a_hi, b_lo)] if path == "lbs" else [])
    acc = sum(a @ b.T for a, b in terms).view(B, 5023, 3)
    S = sum(a.abs() @ b.abs().T for a, b in terms).view(B, 5023, 3).amax(-1)
    u = 2.0 ** -24
    gamma = 448 * 2.0 ** -23 / (1 - 448 * 2.0 ** -23)
    x = xf.double()
    R, J, c = x[:, 0:12].view(B, 1, 3, 4), x[:, 24:36].view(B, 1, 3, 4), x[:, None, 60:63]
    wr, wj = pk.w2[:, 0].double()[None, :, None], pk.w2[:, 1].double()[None, :, None]
    r = (R[..., :3] * acc[..., None, :]).sum(-1) + R[..., 3]
    j = (J[..., :3] * acc[..., None, :]).sum(-1) + J[..., 3]
    v64 = wr * r + wj * j + c
    pmax = acc.abs().amax(-1, keepdim=True)
    lip = wr.abs() * R[..., :3].abs().sum(-1) + wj.abs() * J[..., :3].abs().sum(-1)
    M = (wr.abs() * ((R[..., :3] * acc[..., None, :]).abs().sum(-1) + R[..., 3].abs())
         + wj.abs() * ((J[..., :3] * acc[..., None, :]).abs().sum(-1) + J[..., 3].abs()) + c.abs())
    bound_v = lip * (gamma * S[..., None] + u * pmax) + 6 * u * M
    err_v = (v.double() - v64).abs()
    assert (err_v <= bound_v).all(), (err_v - bound_v).max().item()
    sc = x[:, None, 63:64]
    t = torch.cat([x[:, 64:66], torch.zeros(B, 1, device=cuda_device, dtype=torch.float64)], 1)[:, None, :]
    hs = 128.0
    q64 = (v64 * sc + t + 1.0) * hs
    bound_q = hs * sc * bound_v + 3 * u * hs * ((v64 * sc).abs() + t.abs() + 1.0) * (1 + 1e-6)
    err_q = (pj.double() - q64).abs()
    assert (err_q <= bound_q).all(), (err_q - bound_q).max().item()
    assert err_v.max().item() > 0                     # the bound is tested on a real rounding error, not on zeros
    assert math.isfinite(bound_v.max().item())
