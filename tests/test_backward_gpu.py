"""-m gpu: the decoder backward (dad3d_flame_backward through the C ABI) against torch.autograd through the fp64 oracle
(oracle/flame_oracle.py, itself pinned to the reference's FLAMELayer / HeadMesh): gradients of a random linear functional of
(vertices_3d, reprojected_vertices) w.r.t. all 413 parameters.  Tolerance: relL2 < 1e-4 per parameter group (measured ~1e-6;
the forward blend inside is the 3-product hi/lo GEMM, the dense backward part a 3-product wgmma GEMM)."""
import pytest
import torch

from oracle.flame_oracle import FLAME_CONSTS, FlameOracle, sample_params

pytestmark = pytest.mark.gpu
GROUPS = {"shape": (0, 300), "expression": (300, 400), "jaw": (400, 403), "rotation": (403, 409), "translation": (409, 412),
          "scale": (412, 413)}


def _oracle_grad(p, gv, gp, to_2d, zero_rot=False):
    o = FlameOracle(dtype=torch.float64)
    q = p.double().clone().requires_grad_(True)
    from oracle.flame_oracle import split_3dmm
    loss = 0.0
    if gv is not None:
        loss = loss + (o.flame_forward(split_3dmm(q, FLAME_CONSTS), zero_rot=zero_rot) * gv.double()).sum()
    if gp is not None:
        fp = split_3dmm(q, FLAME_CONSTS)
        v = o.flame_forward(fp, zero_rot=zero_rot)
        scale = torch.clamp(fp["scale"][:, None] + 1.0, min=1e-8)
        t = torch.cat([fp["translation"][:, :2], torch.zeros_like(fp["translation"][:, 2:])], dim=1)     # z zeroed (head_mesh.py:41)
        proj = (v * scale + t[:, None] + 1.0) / 2.0 * 256.0
        loss = loss + ((proj[..., :2] if to_2d else proj) * gp.double()).sum()
    loss.backward()
    return q.grad


@pytest.mark.parametrize("B,to_2d,which", [(1, True, "both"), (3, True, "both"), (5, False, "both"), (130, True, "v"), (64, True, "p")])
def test_backward_matches_autograd(cuda_device, B, to_2d, which):
    from dad_3dheads_b200 import HeadMesh
    hm = HeadMesh()
    dec = hm.flame.decoder(cuda_device)
    p = sample_params(B, seed=300 + B)
    g = torch.Generator().manual_seed(B)
    gv = torch.randn(B, 5023, 3, generator=g) if which in ("both", "v") else None
    gp = torch.randn(B, 5023, 2 if to_2d else 3, generator=g) * 0.01 if which in ("both", "p") else None
    want = _oracle_grad(p, gv, gp, to_2d)
    got = dec.backward(p.to(cuda_device), gv.to(cuda_device) if gv is not None else None,
                       gp.to(cuda_device) if gp is not None else None, to_2d=to_2d).cpu().double()
    for name, (a, b) in GROUPS.items():
        w, q = want[:, a:b], got[:, a:b]
        if name == "translation":
            assert (q[:, 2] == 0).all()
        denom = w.norm().item()
        if denom == 0:
            assert q.norm().item() == 0, name
        else:
            assert ((q - w).norm() / denom).item() < 1e-4, (name, ((q - w).norm() / denom).item())


def test_autograd_function_and_zero_rotation(cuda_device):
    """HeadMesh.decode_with_grad under torch autograd: a Vertices3DLoss / ReprojectionLoss-like objective backpropagates to the
    parameter tensor; zero_rotation zeroes the 6-DoF gradient."""
    from dad_3dheads_b200 import HeadMesh
    hm = HeadMesh()
    p0 = sample_params(4, seed=77)
    tgt_v = torch.randn(4, 5023, 3, generator=torch.Generator().manual_seed(1)) * 0.1
    p = p0.to(cuda_device).requires_grad_(True)
    v3, pj = hm.decode_with_grad(p, to_2d=True)
    loss = (v3 - tgt_v.to(cuda_device)).abs().mean() + 1e-3 * pj.pow(2).mean()
    loss.backward()
    o = FlameOracle(dtype=torch.float64)
    q = p0.double().requires_grad_(True)
    from oracle.flame_oracle import split_3dmm
    fp = split_3dmm(q, FLAME_CONSTS)
    v = o.flame_forward(fp)
    scale = torch.clamp(fp["scale"][:, None] + 1.0, min=1e-8)
    t = torch.cat([fp["translation"][:, :2], torch.zeros_like(fp["translation"][:, 2:])], dim=1)
    proj = ((v * scale + t[:, None] + 1.0) / 2.0 * 256.0)[..., :2]
    ((v - tgt_v.double()).abs().mean() + 1e-3 * proj.pow(2).mean()).backward()
    assert ((p.grad.cpu().double() - q.grad).norm() / q.grad.norm()).item() < 1e-3       # |.| kinks: sign flips at ~0 residuals
    p2 = p0.to(cuda_device).requires_grad_(True)
    v3, _ = hm.decode_with_grad(p2, zero_rotation=True)
    v3.sum().backward()
    assert (p2.grad[:, 403:409] == 0).all() and p2.grad[:, :400].abs().sum() > 0
