"""-m gpu: the reference's OWN demo.py / demo_utils.py, unmodified, over the H100 path (north_star: "keeping
predictor.FaceMeshPredictor's API so demo.py ... run unchanged").

``sys.path`` = [compat/ (predictor, model_training, utils, Sim3DR -> libdad3d.so), oracle/ref_shims (stand-ins for the
third-party packages demo.py imports that the image lacks: fire, pytorch_toolbelt), the reference tree (demo.py, demo_utils.py
and its static index files; /root/reference here, its byte-compiled twin oracle/_ref on the GPU box)].  The checkpoint is a
synthetic-weight ``dad_3dheads.trcd`` written with torch.jit exactly like the reference's exporter
(train/flame_lightning_model.py:384-401), placed at ~/.dad_checkpoints/ of a temporary HOME -- so predictor.py:72's
``torch.jit.load(...)`` + the state-dict key mapping are exercised end to end.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ref_harness as R

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not R.available(), reason="reference tree (oracle/_ref) not built")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def demo_home(tmp_path_factory, cuda_device):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    home = tmp_path_factory.mktemp("home")
    os.makedirs(home / ".dad_checkpoints")
    # written in a subprocess: the harness puts the reference's `predictor` / `model_training` on sys.path, which must not
    # leak into this process (compat/ provides the same names)
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from oracle import ref_harness as R\n"
            "from dad_3dheads_b200.encoder_weights import synthetic_state_dict\n"
            "R.trace_checkpoint(synthetic_state_dict(0), %r)\n" % (ROOT, str(home / ".dad_checkpoints" / "dad_3dheads.trcd")))
    out = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    return home


def _run_demo(home, outdir, kind):
    ref_root = R.root()
    demo = os.path.join(ref_root, "demo.py") if os.path.isfile(os.path.join(ref_root, "demo.py")) else os.path.join(ref_root, "demo.pyc")
    code = ("import sys, runpy\n"
            "sys.path[:0] = [%r, %r, %r, %r]\n"
            "sys.argv = ['demo.py', 'images/demo_heads/1.jpeg', %r, %r]\n"
            "runpy.run_path(%r, run_name='__main__')\n"
            % (os.path.join(ROOT, "compat"), ROOT, os.path.join(ROOT, "oracle", "ref_shims"), ref_root, str(outdir), kind, demo))
    env = dict(os.environ, HOME=str(home))
    out = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=600, cwd=ref_root,
                         env=env)
    assert out.returncode == 0, (kind, out.stderr[-3000:])


def test_demo_flame_params_and_landmark_outputs(demo_home, tmp_path):
    """BASELINE configs[0]: ``python demo.py images/demo_heads/1.jpeg <out> flame_params`` (+ the three landmark renderings)."""
    import cv2
    for kind in ("flame_params", "68_landmarks", "191_landmarks", "445_landmarks"):
        _run_demo(demo_home, tmp_path, kind)
    got = json.load(open(tmp_path / "1_flame_params.json"))
    assert set(got) == {"shape", "expression", "rotation", "translation", "scale", "jaw", "eyeballs", "neck"}
    assert [len(got[k]) for k in ("shape", "expression", "rotation", "translation", "scale", "jaw")] == [300, 100, 6, 3, 1, 3]
    # same numbers as the reference predictor on the same image / weights (tests/golden/reference_predictor.npz)
    z = np.load(os.path.join(ROOT, "tests", "golden", "reference_predictor.npz"))
    p = z["params_3dmm"][0]
    flat = np.concatenate([got["shape"], got["expression"], got["jaw"], got["rotation"], got["translation"], got["scale"]])
    assert np.linalg.norm(flat - p) / np.linalg.norm(p) < 5e-5
    assert got["translation"][2] == 0.0                                   # zeroed in place by reprojected_vertices
    img0 = cv2.imread(os.path.join(R.root(), "images", "demo_heads", "1.jpeg"))
    for kind in ("68_landmarks", "191_landmarks", "445_landmarks"):
        img = cv2.imread(str(tmp_path / f"1_{kind}.png"))
        assert img is not None and img.shape == img0.shape
        assert (img != img0).any()                                        # landmarks were drawn


def test_demo_pncc_runs_the_reference_estimator_on_the_gpu_rasteriser(demo_home, tmp_path):
    """``python demo.py ... pncc``: the reference's own inference/pncc_estimator.py (HeadMesh.reprojected_vertices(to_2d=False)
    -> Sim3DR.rasterize) over compat/ -- the decode and the rasteriser both run in libdad3d.so.  Expected image: the reference's
    C++ rasteriser (oracle/_ref/libsim3dr_ref.so) on the vertices of the reference predictor's parameters for the same image;
    the two parameter sets differ by ~1e-5 relative, so a few silhouette pixels may flip (bit-exactness of the rasteriser on
    identical input is tests/test_rasterizer_gpu.py)."""
    import cv2
    import torch
    from dad_3dheads_b200.flame import load_flame_static
    from oracle.flame_oracle import FlameOracle
    _run_demo(demo_home, tmp_path, "pncc")
    got = cv2.cvtColor(cv2.imread(str(tmp_path / "1_pncc.png")), cv2.COLOR_BGR2RGB)
    img0 = cv2.imread(os.path.join(R.root(), "images", "demo_heads", "1.jpeg"))
    assert got.shape == img0.shape
    sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shims"))
    try:
        import importlib
        ref_sim = importlib.import_module("Sim3DR")
        assert "ref_shims" in ref_sim.__file__
    finally:
        sys.path.pop(0)
        sys.modules.pop("Sim3DR", None)
    z = np.load(os.path.join(ROOT, "tests", "golden", "reference_predictor.npz"))
    st = load_flame_static()
    # predictor.py:136-150 scales the parameters' projection back to the input image: rebuild the same vertices from the params
    p = torch.from_numpy(z["params_3dmm"]).double().clone()
    v = FlameOracle(st, image_size=256).reprojected_vertices(p, to_2d=False)[0].numpy().astype(np.float32)
    v[:, 2] *= -1
    faces = np.load(os.path.join(R.root(), "model_training", "model", "static", "flame_indices", "faces_wo_ears_remapped.npy"))
    sub = st["v_template"][np.unique(faces)]
    lo, hi = sub.min(0, keepdims=True, initial=0), sub.max(0, keepdims=True, initial=0)
    colors = ((st["v_template"] - lo) / (hi - lo)).astype(np.float32)
    want = ref_sim.rasterize(v, np.ascontiguousarray(faces), colors, bg=np.zeros_like(got))
    covered = (want.sum(-1) > 0).mean()
    assert covered > 0.005
    assert (got != want).any(-1).mean() < 0.03 * covered, ((got != want).any(-1).mean(), covered)
