"""-m gpu: the decoder backward checked stage by stage.  Each test runs one stage of dad3d_flame_backward alone
(dad3d_flame_backward_blend / _vertex / _dense / _finalize) on caller buffers and compares it with the model in
tests/backward_model.py:
- vertex and dense stages: bit for bit, on designed operands on which every output is fully determined;
- finalize: the linear parts bit for bit, the directional derivatives of the transform function within an ulp bound of
  fp64 autograd;
- composition and multi-pass: the hooks reproduce dad3d_flame_backward bit for bit, pass by pass;
- real asset: the dense gradient per head and per entry within a bound derived from the arithmetic
  (test_real_asset_dense_within_derived_bound), including a head whose incoming gradient is tiny.

What only the designed tests can see: with K = 15104 terms, gamma_K (~1.8e-3) exceeds the cost of a dropped lo plane of D
or of the basis, or of a dropped lo*hi / hi*lo product (~2^-11 relative), so those errors pass the real-asset bound; they
are caught by the bit-exact vertex and dense tests (tests/test_backward_model_cpu.py shows each one changes their output)."""
import math

import numpy as np
import pytest
import torch

from dad_3dheads_b200 import _lib
from oracle.flame_oracle import FLAME_CONSTS, sample_params
from tests import backward_model as bm
from tests import decode_model as dm
from tests.test_decode_exact_gpu import Guarded

pytestmark = pytest.mark.gpu

NAN16 = 0x7E01               # fp16 NaN payload: D planes never written
_decoders = {}


def designed(nv, device):
    if nv not in _decoders:
        from dad_3dheads_b200.flame import FlameDecoder
        st = bm.designed_static(nv, seed=nv)
        _decoders[nv] = (FlameDecoder(st, FLAME_CONSTS, device), dm.pack(st).to(device), st)
    return _decoders[nv]


@pytest.fixture(scope="module")
def real(flame_static, cuda_device):
    from dad_3dheads_b200.flame import FlameDecoder
    return FlameDecoder(flame_static, FLAME_CONSTS, cuda_device), dm.pack(flame_static).to(cuda_device)


def npad_of(nv):
    return (3 * nv + 127) // 128 * 128


def nblocks(nv):
    return (nv + 255) // 256


def _bits(x):
    return x.contiguous().view(torch.int32 if x.dtype == torch.float32 else torch.int16)


def mismatch(got, want, what):
    bad = (_bits(got) != _bits(want)).nonzero()
    if bad.numel() == 0:
        return None
    return (f"{what}: {bad.shape[0]} values differ; first at {bad[0].tolist()}: "
            f"got {got[tuple(bad[0])].item()!r}, want {want[tuple(bad[0])].item()!r}")


def assert_bits(got, want, what):
    msg = mismatch(got, want, what)
    assert msg is None, msg


def run_vertex(dec, vposed, xf, gv, gp, image_size, to_2d):
    B, nv, dev = xf.shape[0], dec.n_vertices, xf.device
    sigma = torch.full((B,), float("nan"), device=dev)
    d_hi = torch.full((B, npad_of(nv)), NAN16, dtype=torch.int16, device=dev).view(torch.float16)
    d_lo = d_hi.clone()
    partial = torch.full((B, nblocks(nv), 32), float("nan"), device=dev)
    dec.backward_vertex(vposed, xf, gv, gp, sigma=sigma, d_hi=d_hi, d_lo=d_lo, partial=partial, image_size=image_size,
                        to_2d=to_2d)
    return sigma, d_hi, d_lo, partial


# ---------------------------------------------------------------------------------------------------------- vertex stage
VERTEX_EXPS = [-100, -60, -20, -3, 0, 7, 20, 40, None, -120]       # None: all-zero gradients; -120: sigma at its cap
VERTEX_CASES = [(True, 256.0, True, True), (False, 224.0, True, True), (True, 512.0, True, False),
                (False, 256.0, False, True), (True, 224.0, False, True), (False, 512.0, True, False)]


@pytest.mark.parametrize("nv", [97, 256, 300, 512, 5023])
def test_vertex_stage_bit_exact(cuda_device, nv):
    """sigma, both D planes (padding columns included; the sign of a zero is not compared) and the partial records against
    the model, for heads whose max |g|
    spans 2^-120 ... 2^40, an all-zero head, gV only / gP only / both, to_2d True and False, image 224, 256 and 512; the
    last 256-vertex block partly full (97, 300, 5023) and exactly full (256, 512)."""
    dec, pk, _ = designed(nv, cuda_device)
    assert dec.describe(1)["basis_scale"] == pk.scale == 1024.0
    errors = []
    for i, (to_2d, image, with_v, with_p) in enumerate(VERTEX_CASES):
        g = torch.Generator(device=cuda_device).manual_seed(nv * 10 + i)
        vposed, xf, gv, gp = bm.designed_vertex_inputs(len(VERTEX_EXPS), nv, npad_of(nv), pk.scale, VERTEX_EXPS, g,
                                                       cuda_device, to_2d=to_2d, with_v=with_v, with_p=with_p)
        sigma, d_hi, d_lo, partial = run_vertex(dec, vposed, xf, gv, gp, image, to_2d)
        torch.cuda.synchronize()
        s, hi, lo, part = bm.vertex_stage(vposed, xf, gv, gp, pk.w2, image, to_2d, pk.scale)
        what = f"nv={nv} to_2d={to_2d} image={image} gV={with_v} gP={with_p}"
        # an exactly zero dp keeps the sign nvcc's contraction of the plain `a*b + c` gives it: zeros of D compare unsigned
        errors += [mismatch(sigma, s, what + " sigma"), mismatch(d_hi.float() + 0.0, hi + 0.0, what + " D hi"),
                   mismatch(d_lo.float() + 0.0, lo + 0.0, what + " D lo"), mismatch(partial[..., :30], part, what + " partial")]
        if not torch.isnan(partial[..., 30:]).all():
            errors.append(what + ": floats 30, 31 of a partial record were written")
    errors = [e for e in errors if e]
    assert not errors, "\n".join(errors)


# ----------------------------------------------------------------------------------------------------------- dense stage
DENSE_CASES = [(5023, B) for B in (1, 127, 128, 129, 255, 256, 257, 4096)] + [(97, 1), (97, 129), (300, 257), (300, 1)]


@pytest.mark.parametrize("nv,B", DENSE_CASES)
def test_dense_stage_bit_exact(cuda_device, nv, B):
    """dcoef = hi hi + (lo hi + hi lo) over K = npad (6, 8 and 236 k-blocks of 64) against the model, across the row-tile
    edges of the GEMM, into a guarded buffer: the guard bands stay unchanged and every float is written."""
    dec, pk, _ = designed(nv, cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(B + nv)
    d_hi, d_lo = bm.designed_d_planes(B, nv, npad_of(nv), g, cuda_device)
    out = Guarded(B, 448, 1, 4 * (B % 2), cuda_device)      # float4 stores: 16-byte aligned
    dec.backward_dense(d_hi.half(), d_lo.half(), out.out.view(B, 448))
    torch.cuda.synchronize()
    out.check_guards(f"dense nv={nv} B={B}")
    got = out.out.view(B, 448)
    for h0 in range(0, B, 1024):
        want = bm.dense_stage(d_hi[h0:h0 + 1024], d_lo[h0:h0 + 1024], pk)
        assert_bits(got[h0:h0 + 1024][:, bm.DENSE_COLS], want[:, bm.DENSE_COLS], f"dense nv={nv} B={B} heads {h0}..")
    assert (got[:, 438:] == 0).all()


# -------------------------------------------------------------------------------------------------------- finalize stage
def run_finalize(dec, params, dcoef, partial, sig, flags=0):
    B = params.shape[0]
    out = Guarded(B, 413, 1, 3, params.device)
    dec.backward_finalize(params, dcoef, partial, sig, out.out.view(B, 413), flags=flags)
    torch.cuda.synchronize()
    out.check_guards("finalize")
    return out.out.view(B, 413).clone()


def test_finalize_dense_part_exact(cuda_device):
    """No transform cotangents (partials 0): grad[beta] == dcoef * unlift exactly (the joint term vanishes because the jaw
    pose features do not depend on J), translation (0, 0, 0), scale 0; every entry written."""
    dec, pk, _ = designed(97, cuda_device)
    B = 64
    params, dcoef, partial, sig = bm.designed_finalize_inputs(B, 97, torch.Generator(device=cuda_device).manual_seed(1),
                                                              cuda_device, zero_partial=True)
    got = run_finalize(dec, params, dcoef, partial, sig)
    want, mask = bm.finalize_linear(params, dcoef, partial, sig, pk.scale)
    assert mask[:, :400].all()
    assert torch.equal(got[mask], want[mask])
    assert (got[:, :400] != 0).all()


@pytest.mark.parametrize("nv", [97, 300])
def test_finalize_within_bound_of_fp64_autograd(cuda_device, nv):
    """Designed partials in every vertex block and random dcoef: translation and scale (with the clamp heads 1, 2) exact;
    jaw, rotation and betas within bm.finalize_bound of the fp64 autograd gradient of the same transform function."""
    dec, pk, st = designed(nv, cuda_device)
    jt, jd = bm.joint_constants(st)
    B = 64
    for zero_dcoef in (True, False):
        params, dcoef, partial, sig = bm.designed_finalize_inputs(
            B, nv, torch.Generator(device=cuda_device).manual_seed(nv + zero_dcoef), cuda_device, zero_dcoef=zero_dcoef)
        got = run_finalize(dec, params, dcoef, partial, sig)
        lin, mask = bm.finalize_linear(params, dcoef, partial, sig, pk.scale)
        lm = mask.clone()
        lm[:, :400] = False
        assert torch.equal(got[lm], lin[lm])
        assert (got[1:3, 412] == 0).all() and (lin[1:3, 412] == 0).all() and (lin[3:, 412] != 0).any()
        ref, mag = bm.finalize_f64(params, dcoef, partial, sig, jt.to(cuda_device), jd.to(cuda_device), pk.scale)
        bound = bm.finalize_bound(params, mag)
        err = (got.double() - ref).abs()
        assert (err <= bound).all(), f"worst excess at {(err - bound).argmax().item()}: {(err / bound).max().item():.3g}"
        assert err.max().item() > 0 and (ref[:, 400:409].abs() > 0).all()


def test_finalize_zero_flags(cuda_device):
    """ZERO_ROT / ZERO_JAW give exact zeros in their slots and leave every other entry equal to the unflagged run, on heads
    whose jaw is 0 and whose 6-D rotation is the identity (there the flags do not change the transform function)."""
    dec, pk, _ = designed(97, cuda_device)
    B = 32
    params, dcoef, partial, sig = bm.designed_finalize_inputs(B, 97, torch.Generator(device=cuda_device).manual_seed(5),
                                                              cuda_device)
    params[:, 400:403] = 0.0
    params[:, 403:409] = torch.tensor([1.0, 0, 0, 0, 1.0, 0], device=cuda_device)
    base = run_finalize(dec, params, dcoef, partial, sig)
    assert (base[:, 400:409] != 0).any()
    for flags, zero in ((bm.ZERO_ROT, slice(403, 409)), (bm.ZERO_JAW, slice(400, 403)),
                        (bm.ZERO_ROT | bm.ZERO_JAW, slice(400, 409))):
        got = run_finalize(dec, params, dcoef, partial, sig, flags)
        assert (got[:, zero] == 0).all(), flags
        keep = torch.ones(413, dtype=torch.bool)
        keep[zero] = False
        assert torch.equal(got[:, keep], base[:, keep]), flags


# ---------------------------------------------------------------------------------------------- composition, multi-pass
def _grads(B, nv, to_2d, seed, device, spread=30):
    g = torch.Generator().manual_seed(seed)
    mag = torch.ldexp(torch.ones(B), torch.randint(-spread, spread + 1, (B,), generator=g).float())[:, None, None]
    gv = torch.randn(B, nv, 3, generator=g) * mag
    gp = torch.randn(B, nv, 2 if to_2d else 3, generator=g) * mag * 0.01
    return gv.to(device), gp.to(device)


def test_hooks_compose_to_the_full_backward(real, cuda_device):
    """prep + blend + vertex + dense + finalize on caller buffers reproduce dad3d_flame_backward bit for bit; the full call
    writes every entry of a sentinel-filled grad_params and nothing outside it."""
    dec, pk = real
    B, nv = 300, 5023
    p = sample_params(B, seed=91).to(cuda_device)
    gv, gp = _grads(B, nv, False, 92, cuda_device)
    out = Guarded(B, 413, 1, 5, cuda_device)
    nbytes = int(dec.lib.dad3d_flame_backward_workspace_bytes(dec._h, B))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda_device)
    _lib.check(dec.lib.dad3d_flame_backward(dec._h, p.data_ptr(), B, 0, gv.data_ptr(), gp.data_ptr(), 224.0, 0,
                                            out.out.data_ptr(), ws.data_ptr(), ws.numel(),
                                            torch.cuda.current_stream().cuda_stream), "dad3d_flame_backward")
    torch.cuda.synchronize()
    out.check_guards("dad3d_flame_backward")
    hi, lo, xf = dec.prep(p)
    vposed = torch.empty(B, npad_of(nv), device=cuda_device)
    dec.backward_blend(hi, lo, B, vposed)
    sigma, d_hi, d_lo, partial = run_vertex(dec, vposed, xf, gv, gp, 224.0, False)
    dcoef = torch.empty(B, 448, device=cuda_device)
    dec.backward_dense(d_hi, d_lo, dcoef)
    got = run_finalize(dec, p, dcoef, partial, sigma)
    assert_bits(got, out.out.view(B, 413), "hooks vs dad3d_flame_backward")
    assert len(set(sigma.tolist())) > 20                    # the heads really have their own sigma


def test_multi_pass_equals_each_pass_alone(real, cuda_device):
    """B = 4096 + 37: two passes, heads of magnitudes 2^-30 ... 2^30 in both; every row equals its pass run alone."""
    dec, _ = real
    B = 4096 + 37
    p = sample_params(B, seed=93).to(cuda_device)
    gv, gp = _grads(B, 5023, True, 94, cuda_device)
    full = dec.backward(p, gv, gp, to_2d=True)
    for a, b in ((0, 4096), (4096, B)):
        part = dec.backward(p[a:b], gv[a:b], gp[a:b], to_2d=True)
        assert_bits(full[a:b], part, f"pass {a}..{b}")
    assert torch.isfinite(full).all()


# ------------------------------------------------------------------------------------------- real asset, derived bound
def _real_basis(static, scale, device):
    sd = torch.from_numpy(np.asarray(static["shapedirs"], np.float64)).reshape(-1, 400)
    pd = torch.from_numpy(np.asarray(static["posedirs"], np.float64)).T
    return (torch.cat([sd, pd], 1) * scale).to(device)                    # [3 V, 436] fp64, the scaled fp32 basis


def test_real_asset_dense_within_derived_bound(real, flame_static, cuda_device):
    """Real asset and parameters, the device's own prep rows, blend and vertex stage; per head and per entry the dense
    gradient dcoef * unlift against the fp64 sum_k dp64_k Bs_k, with dp64 computed in fp64 from the same fp32 inputs and
    Bs the scaled fp32 basis.  In lifted units (x = dp64 L, L = sigma basis_scale):
        |dcoef - L ref| <= L sum_k |Bs_k| (8 u P_k + 2^-145)                dp in fp32 (P_k = its terms' magnitude)
                         + (3 2^-22 + 1.01 gamma_{2K+2}) sum_k |x_k| |Bs_k|  fp16 splits of D and Bs, dropped lo*lo,
                                                                             the three accumulator classes
                         + 2^-24 (sum_k |Bs_k| + sum_k |x_k|) + u |L ref|    fp16 subnormal lo pieces, final rounding
    with u = 2^-24, gamma_n = n 2^-23 / (1 - n 2^-23), K = 3 V.  Head 0's incoming gradient is tiny: its max |g| is below
    2^(k - 118), k = log2 basis_scale from describe() -- without the exponent cap of sigma its gradient was NaN."""
    dec, pk = real
    k = bm.log2_scale(dec.describe(1)["basis_scale"])
    B, nv = 48, 5023
    p = sample_params(B, seed=95).to(cuda_device)
    gv, gp = _grads(B, nv, True, 96, cuda_device, spread=20)
    gv[0] = torch.randn(nv, 3, generator=torch.Generator().manual_seed(7)).to(cuda_device) * 2.0 ** (k - 124)
    gp[0] = 0.0
    assert gv[0].abs().max().item() < 2.0 ** (k - 118)
    hi, lo, xf = dec.prep(p)
    vposed = torch.empty(B, npad_of(nv), device=cuda_device)
    dec.backward_blend(hi, lo, B, vposed)
    sigma, d_hi, d_lo, partial = run_vertex(dec, vposed, xf, gv, gp, 256.0, True)
    dcoef = torch.empty(B, 448, device=cuda_device)
    dec.backward_dense(d_hi, d_lo, dcoef)
    torch.cuda.synchronize()
    assert sigma[0].item() == 2.0 ** bm.sigma_emax(pk.scale)
    assert torch.isfinite(dcoef).all() and torch.isfinite(d_hi.float()).all() and torch.isfinite(d_lo.float()).all()
    u = 2.0 ** -24
    Bs = _real_basis(flame_static, pk.scale, cuda_device)
    x64 = xf.double()
    half_img = 128.0
    g64 = gv.double() + x64[:, 63, None, None] * half_img * torch.cat([gp.double(), torch.zeros_like(gp[..., :1]).double()], -1)
    gabs = gv.double().abs() + x64[:, 63, None, None] * half_img * torch.cat([gp.double().abs(),
                                                                               torch.zeros_like(gp[..., :1]).double()], -1)
    A0, A2 = x64[:, 0:12].view(B, 1, 3, 4)[..., :3], x64[:, 24:36].view(B, 1, 3, 4)[..., :3]
    wr, wj = pk.w2[:, 0].double()[None, :, None], pk.w2[:, 1].double()[None, :, None]
    dp64 = wr * (A0.transpose(-1, -2) @ g64[..., None])[..., 0] + wj * (A2.transpose(-1, -2) @ g64[..., None])[..., 0]
    P = (wr.abs() * (A0.abs().transpose(-1, -2) @ gabs[..., None])[..., 0]
         + wj.abs() * (A2.abs().transpose(-1, -2) @ gabs[..., None])[..., 0])
    L = (sigma.double() * pk.scale)[:, None]
    xk = dp64.reshape(B, -1) * L
    ref = xk @ Bs
    Babs = Bs.abs()
    n = 2 * 3 * nv + 2
    gamma = n * 2.0 ** -23 / (1 - n * 2.0 ** -23)
    bound = (L * ((8 * u * P.reshape(B, -1) + 2.0 ** -145) @ Babs) + (3 * 2.0 ** -22 + 1.01 * gamma) * (xk.abs() @ Babs)
             + 2.0 ** -24 * (Babs.sum(0)[None, :] + xk.abs().sum(1, keepdim=True)) + u * ref.abs())
    err = (dcoef[:, :436].double() - ref).abs()
    ratio = (err / bound).max().item()
    print(f"real-asset dense: max err / bound = {ratio:.3g}; tiny head max |dcoef - ref| / |ref| = "
          f"{(err[0] / ref[0].abs().clamp_min(1e-300)).max().item():.3g}")
    assert (err <= bound).all(), f"worst excess at {(err - bound).argmax().item()}: err / bound = {ratio:.3g}"
    assert err.max().item() > 0 and math.isfinite(bound.max().item())
    assert (ref[0] != 0).any()


def test_tiny_gradient_head_is_finite_and_leaves_its_neighbour_unchanged(real, cuda_device):
    """dad3d_flame_backward with a head whose max |g| is below 2^(k - 118) next to a normal head: the tiny head's
    gradient is finite and the neighbour's equals its gradient computed alone, bit for bit."""
    dec, _ = real
    k = bm.log2_scale(dec.describe(1)["basis_scale"])
    p = sample_params(2, seed=97).to(cuda_device)
    gv, gp = _grads(2, 5023, True, 98, cuda_device, spread=0)
    gv[0] *= 2.0 ** (k - 124)
    gp[0] = 0.0
    out = dec.backward(p, gv, gp)
    alone = dec.backward(p[1:], gv[1:], gp[1:])
    assert torch.isfinite(out[0]).all() and (out[0, :400] != 0).any()
    assert_bits(out[1:], alone, "neighbour of the tiny head")
