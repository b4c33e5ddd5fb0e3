"""-m gpu: the CUDA FLAME decoder (through the C ABI) against the CPU oracle on identical seeded inputs.

Tolerances (BASELINE.json north_star: 1e-4 relative, vertex L2 < 1e-4):
  default (dedicated decode kernel, ONE fp16 tensor-core product, TF32-class operands, template exact to 22 bits):
      norm-wise relL2 < 5e-5 (measured 1.5e-5), element-wise |err| <= 1e-4 |ref| + 1e-5 m, per-vertex L2 < 1e-4 m
  hilo=True (fp16 hi/lo 3-product blend through the tile engine; what the reference-facing per-image methods use):
      norm-wise relL2 < 2e-6, max abs error < 4e-6 * max|ref|  (the oracle's own fp32-vs-fp64 noise level)
"""
import numpy as np
import pytest
import torch

from oracle.flame_oracle import FLAME_CONSTS, FlameOracle, sample_params, synthetic_static
from tests import eval_model

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _maxrel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.fixture(scope="module")
def head_mesh(cuda_device):
    from dad_3dheads_b200 import HeadMesh
    return HeadMesh()


@pytest.fixture(scope="module")
def oracle64(flame_static):
    return FlameOracle(flame_static, dtype=torch.float64)


def test_simt_blend_matches_oracle(head_mesh, oracle64, cuda_device):
    """CUDA-core verification path: isolates prep / LBS / projection kernels from the tensor-core GEMM."""
    p = sample_params(5, seed=1)
    dec = head_mesh.flame.decoder(cuda_device)
    v3, pj = dec.decode(p.to(cuda_device), want_vertices=True, want_projected=True, simt=True)
    assert _rel(v3, oracle64.vertices_3d(p)) < 2e-6
    assert _rel(pj, oracle64.reprojected_vertices(p)) < 2e-6


@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 64, 127, 128, 129, 255, 257, 261, 512])   # incl. the edges of the 256-head row permutation blocks
@pytest.mark.parametrize("hilo", [False, True])
def test_decode_matches_oracle(head_mesh, oracle64, cuda_device, B, hilo):
    p = sample_params(B, seed=100 + B)
    v3, pj = head_mesh.decode(p.to(cuda_device), hilo=hilo)
    v_ref = oracle64.vertices_3d(p)
    p_ref = oracle64.reprojected_vertices(p)
    assert v3.shape == (B, 5023, 3) and pj.shape == (B, 5023, 2)
    tol, mtol = (2e-6, 4e-6) if hilo else (5e-5, 2e-4)
    assert _rel(v3, v_ref) < tol and _maxrel(v3, v_ref) < mtol, (_rel(v3, v_ref), _maxrel(v3, v_ref))
    assert _rel(pj, p_ref) < tol and _maxrel(pj, p_ref) < mtol
    assert (v3.double().cpu() - v_ref).norm(dim=-1).max().item() < 1e-4          # north_star: vertex L2 < 1e-4


@pytest.mark.parametrize("B", [1, 77, 300])
def test_decode_3d_projection_and_single_outputs(head_mesh, oracle64, cuda_device, B):
    """to_2d=False (3-component projection) and the one-output variants of the default kernel."""
    dec = head_mesh.flame.decoder(cuda_device)
    p = sample_params(B, seed=200 + B)
    d = p.to(cuda_device)
    v3, pj3 = dec.decode(d, want_vertices=True, want_projected=True, to_2d=False)
    assert _rel(pj3, oracle64.reprojected_vertices(p, to_2d=False)) < 5e-5
    only_v = dec.decode(d, want_vertices=True, want_projected=False)
    only_p = dec.decode(d, want_vertices=False, want_projected=True, to_2d=False)
    assert only_v[1] is None and only_p[0] is None
    assert torch.equal(only_v[0], v3) and torch.equal(only_p[1], pj3)
    _, pj2 = dec.decode(d, want_vertices=False, want_projected=True, to_2d=True)
    assert torch.equal(pj2, pj3[..., :2])


def test_decode_matches_fp32_oracle_within_contract(head_mesh, flame_static, cuda_device):
    """The contract itself: within 1e-4 relative of the reference-arithmetic (fp32) path, element-wise where it is defined."""
    p = sample_params(16, seed=5)
    o32 = FlameOracle(flame_static)
    v_ref = o32.vertices_3d(p)
    v3, _ = head_mesh.decode(p.to(cuda_device), hilo=True)
    err = (v3.cpu() - v_ref).abs()
    assert (err <= 1e-4 * v_ref.abs() + 1e-6).all()        # rtol 1e-4, atol 1 micrometre for coordinates near 0
    assert _rel(v3, v_ref) < 1e-5
    v3, _ = head_mesh.decode(p.to(cuda_device))            # default one-product kernel: atol 10 micrometres
    err = (v3.cpu() - v_ref).abs()
    assert (err <= 1e-4 * v_ref.abs() + 1e-5).all(), (err - 1e-4 * v_ref.abs()).max()
    assert _rel(v3, v_ref) < 5e-5


def test_fast_mode_within_stated_tolerance(head_mesh, oracle64, cuda_device):
    p = sample_params(32, seed=6)
    v3, pj = head_mesh.decode(p.to(cuda_device))
    assert _rel(v3, oracle64.vertices_3d(p)) < 1e-4
    assert _rel(pj, oracle64.reprojected_vertices(p)) < 1e-4


def test_reference_api_cpu_tensors_and_side_effects(head_mesh, flame_static):
    """vertices_3d / reprojected_vertices with CPU tensors like predictor.py:136-137, incl. the tz in-place zeroing."""
    o = FlameOracle(flame_static)
    p = sample_params(2, seed=8)
    p_ref = p.clone()
    v = head_mesh.vertices_3d(p)
    assert v.device.type == "cpu" and _rel(v, o.vertices_3d(p_ref)) < 1e-5
    vz = head_mesh.vertices_3d(p, zero_rotation=True)
    assert _rel(vz, o.vertices_3d(p_ref, zero_rotation=True)) < 1e-5
    q3 = head_mesh.reprojected_vertices(p.clone(), to_2d=False)
    assert q3.shape == (2, 5023, 3) and _rel(q3, o.reprojected_vertices(p_ref.clone(), to_2d=False)) < 1e-5
    q = head_mesh.reprojected_vertices(p, to_2d=True)
    assert (p[:, 411] == 0).all(), "translation z must be zeroed through the view (head_mesh.py:41)"
    assert _rel(q, o.reprojected_vertices(p_ref, to_2d=True)) < 1e-5


def test_zero_jaw_flag(head_mesh, flame_static, cuda_device):
    from dad_3dheads_b200 import FlameParams
    o = FlameOracle(flame_static, dtype=torch.float64)
    p = sample_params(3, seed=9)
    fp = FlameParams.from_3dmm(p.to(cuda_device), FLAME_CONSTS)
    v = head_mesh.flame.forward(fp, zero_rot=False, zero_jaw=True)
    from oracle.flame_oracle import split_3dmm
    want = o.flame_forward(split_3dmm(p.double(), FLAME_CONSTS), zero_rot=False, zero_jaw=True)
    assert _rel(v, want) < 2e-6


def test_degenerate_inputs(head_mesh, oracle64, cuda_device):
    """zero vector (template), huge negative scale (clamp 1e-8), zero rotation 6-vector (F.normalize eps path)."""
    p = torch.zeros(3, 413)
    p[:, 403:409] = torch.tensor([1.0, 0, 0, 0, 1.0, 0])
    p[1, 412] = -5.0
    p[2, 403:409] = 0.0
    v3, pj = head_mesh.decode(p.to(cuda_device))
    v_ref, p_ref = oracle64.vertices_3d(p), oracle64.reprojected_vertices(p)
    assert torch.isfinite(v3).all() and torch.isfinite(pj).all()
    assert (v3.cpu().double() - v_ref).abs().max() < 1e-6
    assert (pj.cpu().double() - p_ref).abs().max() < 1e-3       # pixels
    assert v3[2].abs().max() == 0                               # zero 6-vector -> zero matrix, like the reference


def test_general_layout_neck_eyeballs_synthetic(cuda_device):
    from dad_3dheads_b200 import HeadMesh
    st = synthetic_static(seed=4, n_vertices=301)
    consts = dict(FLAME_CONSTS, shape=120, expression=40, neck=3, eyeballs=6)
    hm = HeadMesh(flame_config=consts, static=st)
    o = FlameOracle(st, consts=consts, dtype=torch.float64)
    p = sample_params(37, seed=9, consts=consts)
    v3, pj = hm.decode(p.to(cuda_device), to_2d=False)
    assert _rel(v3, o.vertices_3d(p)) < 2e-6
    assert _rel(pj, o.reprojected_vertices(p, to_2d=False)) < 2e-6


def test_chunk_boundary_and_batch_independence(head_mesh, cuda_device):
    """B larger than one internal pass of either path; a head's result must not depend on its batch (bit-exact).
    The fused path switches to the row-tile-persistent schedule once there are >= #SM row tiles (B >= 148*128)."""
    dec = head_mesh.flame.decoder(cuda_device)
    B = 4096 + 300
    p = sample_params(B, seed=12).to(cuda_device)
    sel = torch.tensor([0, 127, 128, 4095, 4096, 4097, B - 1], device=cuda_device)
    for unfused in (False, True):
        v3, pj = dec.decode(p, want_vertices=True, want_projected=True, unfused=unfused)
        v_sel, pj_sel = dec.decode(p[sel], want_vertices=True, want_projected=True, unfused=unfused)
        assert torch.equal(v3[sel], v_sel) and torch.equal(pj[sel], pj_sel)
    del v3, pj
    props = torch.cuda.get_device_properties(cuda_device)
    fused_chunk = props.multi_processor_count * 128 * 4
    B = fused_chunk + 333                                   # crosses the fused pass boundary, persistent schedule
    p = sample_params(B, seed=13).to(cuda_device)
    v3, pj = dec.decode(p, want_vertices=True, want_projected=True)
    sel = torch.tensor([0, 1, 127, 128, 18943, 18944, fused_chunk - 1, fused_chunk, fused_chunk + 1, B - 1],
                       device=cuda_device)
    v_sel, pj_sel = dec.decode(p[sel], want_vertices=True, want_projected=True)
    assert torch.equal(v3[sel], v_sel) and torch.equal(pj[sel], pj_sel)
    assert torch.isfinite(v3).all()
    # opt-in variant: big passes as 2x2 thread-block clusters with TMA multicast of both operands -- same arithmetic
    n = props.multi_processor_count * 128 + 77
    va, pa = dec.decode(p[:n], want_vertices=True, want_projected=True, hilo=True)
    vb, pb = dec.decode(p[:n], want_vertices=True, want_projected=True, cluster=True)
    assert torch.equal(va, vb) and torch.equal(pa, pb)
    del va, pa, vb, pb
    # DAD3D_DECODE_PAIR (CTA pairs; no effect on sm_90) and the DAD3D_DECODE_PAIR=0 environment leave the results unchanged
    import os
    n = props.multi_processor_count * 128 * 2 + 77
    old_env = os.environ.get("DAD3D_DECODE_PAIR")
    os.environ["DAD3D_DECODE_PAIR"] = "0"
    try:
        va, pa = dec.decode(p[:n], want_vertices=True, want_projected=True)
    finally:
        if old_env is None:
            del os.environ["DAD3D_DECODE_PAIR"]
        else:
            os.environ["DAD3D_DECODE_PAIR"] = old_env
    vb, pb = dec.decode(p[:n], want_vertices=True, want_projected=True, pair=True)
    assert torch.equal(va, vb) and torch.equal(pa, pb)


def test_fused_equals_unfused(head_mesh, oracle64, cuda_device):
    """The fused epilogue (default) and the two-kernel A/B path run the same arithmetic."""
    dec = head_mesh.flame.decoder(cuda_device)
    p = sample_params(300, seed=21)
    for to_2d in (True, False):
        a = dec.decode(p.to(cuda_device), want_vertices=True, want_projected=True, to_2d=to_2d, hilo=True)
        b = dec.decode(p.to(cuda_device), want_vertices=True, want_projected=True, to_2d=to_2d, unfused=True)
        assert (a[0] - b[0]).abs().max().item() < 1e-7 and (a[1] - b[1]).abs().max().item() < 1e-4
        assert _rel(b[0], oracle64.vertices_3d(p)) < 2e-6
        assert _rel(a[1], oracle64.reprojected_vertices(p, to_2d=to_2d)) < 2e-6
    only_v = dec.decode(p.to(cuda_device), want_vertices=True, want_projected=False, hilo=True)
    only_p = dec.decode(p.to(cuda_device), want_vertices=False, want_projected=True, hilo=True)
    assert only_v[1] is None and only_p[0] is None
    assert torch.equal(only_v[0], a[0]) and torch.equal(only_p[1], dec.decode(p.to(cuda_device), want_projected=True, hilo=True)[1])


def test_blend_linearity_property(head_mesh, cuda_device):
    """With jaw = 0 and no rotation the decoder is affine in beta: v(a+b) - v(a) - v(b) + v(0) = 0  (full-size check)."""
    g = torch.Generator().manual_seed(3)
    a = torch.zeros(256, 413)
    b = torch.zeros(256, 413)
    a[:, :400] = torch.randn(256, 400, generator=g)
    b[:, :400] = torch.randn(256, 400, generator=g)
    z = torch.zeros(256, 413)
    dec = head_mesh.flame.decoder(cuda_device)
    f = lambda x: dec.decode(x.to(cuda_device), zero_rot=True, hilo=True)[0].double()
    r = f(a + b) - f(a) - f(b) + f(z)
    assert r.abs().max().item() < 5e-7
    f = lambda x: dec.decode(x.to(cuda_device), zero_rot=True)[0].double()       # default kernel: betas are rounded to fp16
    r = f(a + b) - f(a) - f(b) + f(z)
    assert r.abs().max().item() < 3e-5


def test_landmark_gathers(head_mesh, flame_static, cuda_device):
    p = sample_params(6, seed=14)
    _, pj = head_mesh.decode(p.to(cuda_device))
    dec = head_mesh.flame.decoder(cuda_device)
    for key in ("keypoints_191", "keypoints_445", "keypoints_565"):
        idx = torch.from_numpy(flame_static[key].astype(np.int64))
        got = dec.gather(pj, idx)
        assert torch.equal(got.cpu(), pj.cpu()[:, idx])
    faces = torch.from_numpy(flame_static["faces"].astype(np.int64))
    fi = torch.from_numpy(flame_static["static_lmk_face_idx"].astype(np.int64))
    tri = faces[fi]
    bary = torch.from_numpy(flame_static["static_lmk_b_coords"])
    got = dec.gather_bary(pj, tri, bary)
    want = eval_model.gather_bary(pj.cpu(), tri, bary.float())
    assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32))
    assert dec.gather(pj, torch.zeros(0, dtype=torch.int64)).shape == (6, 0, 2)


def test_empty_batch(head_mesh, cuda_device):
    v3, pj = head_mesh.decode(torch.zeros(0, 413, device=cuda_device))
    assert v3.shape == (0, 5023, 3) and pj.shape == (0, 5023, 2)


@pytest.mark.parametrize("B", [1, 6])
def test_reference_fixture(head_mesh, cuda_device, B):
    """tests/golden/reference_flame.npz: outputs of the UNMODIFIED reference HeadMesh (head_mesh.py:28-46) over its own
    flame.pkl (tools/make_reference_golden.py), fp64 run as the yard-stick; north_star tolerance 1e-4, measured ~2e-7."""
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_flame.npz"))
    p = torch.from_numpy(z[f"params_b{B}"])
    for hilo, tol, l2tol in ((True, 2e-6, 1e-6), (False, 5e-5, 1e-4)):     # strict hi/lo blend; default one-product kernel
        v3, pj = head_mesh.decode(p.to(cuda_device), to_2d=False, hilo=hilo)
        assert _rel(v3, torch.from_numpy(z[f"vertices3d_f64_b{B}"])) < tol
        assert _rel(pj, torch.from_numpy(z[f"projected3_f64_b{B}"])) < tol
        l2 = (v3.double().cpu() - torch.from_numpy(z[f"vertices3d_f64_b{B}"])).norm(dim=-1).max().item()
        assert l2 < l2tol, l2                                   # per-vertex L2 in metres (north_star target < 1e-4)
    vz = head_mesh.vertices_3d(p.to(cuda_device), zero_rotation=True)
    assert _rel(vz, torch.from_numpy(z[f"vertices3d_zero_rot_f32_b{B}"])) < 2e-6
    q = p.clone()
    pr = head_mesh.reprojected_vertices(q, to_2d=False)         # CPU tensor in -> CPU out, tz zeroed through the view
    assert _rel(pr, torch.from_numpy(z[f"projected3_f64_b{B}"])) < 2e-6
    assert np.array_equal(q.numpy(), z[f"params_after_reproject_f32_b{B}"])
