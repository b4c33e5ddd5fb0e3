"""``import Sim3DR`` (reference: Sim3DR/__init__.py, Sim3DR/Sim3DR.py, Sim3DR/lighting.py) -> the GPU rasteriser and lit
renderer of dad_3dheads_b200 (bit-exact with the reference's Cython/C++ module; the lighting as described in
``Sim3DR.lighting``); lets the reference's ``inference/pncc_estimator.py`` run unchanged."""
from dad_3dheads_b200.rasterizer import get_normal, rasterize  # noqa: F401
from .lighting import RenderPipeline  # noqa: F401
