"""-m "not gpu": rasterizer.load_render_static (assets/render_static.json) gives the reference's own PNCC inputs bit for bit: the faces its PNCC estimator
renders and the colours it computes (inference/pncc_estimator.py:46-60,66-68), run through the reference harness."""
import numpy as np
import pytest

from dad_3dheads_b200.rasterizer import load_render_static
from oracle import ref_harness

pytestmark = pytest.mark.skipif(not ref_harness.available(), reason="reference harness unavailable")


@pytest.fixture(scope="module")
def estimator():
    ref_harness.activate()
    from inference.pncc_estimator import PNCCEstimator
    return PNCCEstimator()


def test_faces_equal_reference(estimator):
    faces = load_render_static()["faces_wo_ears"]
    want = np.asarray(estimator.faces_wo_back_remapped)
    assert faces.dtype == np.int32 and faces.shape == (6270, 3)
    assert np.array_equal(faces, want)


def test_colors_equal_reference(estimator):
    colors = load_render_static()["ncc_colors"]
    want = np.asarray(estimator.colors).astype(np.float32)
    assert colors.dtype == np.float32 and colors.shape == want.shape == (5023, 3)
    assert np.array_equal(colors.view(np.uint32), want.view(np.uint32))


def test_colors_need_the_fp64_template(estimator):
    """Recomputed from the packed fp32 template, the colours differ in the last bits: the fp64 pickle is the source."""
    from inference.pncc_estimator import compute_ncc_color_codes
    from dad_3dheads_b200.flame import load_flame_static
    st = load_render_static()
    faces, colors = st["faces_wo_ears"], st["ncc_colors"]
    template32 = load_flame_static()["v_template"].astype(np.float64)
    from_fp32 = compute_ncc_color_codes(template32, np.unique(faces)).astype(np.float32)
    assert not np.array_equal(from_fp32, colors)
    assert np.abs(from_fp32 - colors).max() < 1e-6
