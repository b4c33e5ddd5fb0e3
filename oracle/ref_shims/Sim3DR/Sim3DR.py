"""TEST INFRASTRUCTURE.  ``Sim3DR.Sim3DR`` (Sim3DR/Sim3DR.py), the module the reference's Sim3DR/lighting.py imports
``get_normal`` and ``rasterize`` from: the same two functions as this shim package, over the reference's own C++."""
from . import get_normal, rasterize  # noqa: F401
