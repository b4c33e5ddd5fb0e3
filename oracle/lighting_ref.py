"""The reference's UNMODIFIED ``Sim3DR/lighting.py`` (RenderPipeline) as a live oracle (TEST INFRASTRUCTURE).

``build()`` byte-compiles /root/reference/Sim3DR/lighting.py into ``oracle/_ref/Sim3DR/lighting.pyc``, as
oracle/build_ref.py does for the rest of the reference (nothing is copied; the .pyc travels with the built tree).
``load()`` imports it under a private package name whose ``Sim3DR`` submodule is oracle/ref_shims/Sim3DR (the
reference's own C++ rasteriser and normals through ctypes), so it never collides with ``compat/Sim3DR``.
A test sees the light the reference computes by replacing the loaded module's ``rasterize``, which receives it as colours."""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import py_compile
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DAD3D_REFERENCE", "/root/reference")
PYC = os.path.join(_HERE, "_ref", "Sim3DR", "lighting.pyc")
SHIM = os.path.join(_HERE, "ref_shims", "Sim3DR")
_PKG = "_dad3d_ref_sim3dr"


def build(ref: str = REF) -> bool:
    src = os.path.join(ref, "Sim3DR", "lighting.py")
    if not os.path.isfile(src):
        return False
    os.makedirs(os.path.dirname(PYC), exist_ok=True)
    py_compile.compile(src, cfile=PYC, dfile=os.path.join("<reference>", "Sim3DR", "lighting.py"), doraise=True,
                       invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
    return True


def available() -> bool:
    return os.path.isfile(PYC) and os.path.isfile(os.path.join(_HERE, "_ref", "libsim3dr_ref.so"))


def load():
    """-> the reference's ``Sim3DR.lighting`` module (RenderPipeline, norm_vertices, _norm) over the shim package."""
    name = _PKG + ".lighting"
    if name in sys.modules:
        return sys.modules[name]
    if not available():
        raise RuntimeError("oracle/_ref/Sim3DR/lighting.pyc or libsim3dr_ref.so is not built (__graft_entry__.build())")
    spec = importlib.util.spec_from_file_location(_PKG, os.path.join(SHIM, "__init__.py"), submodule_search_locations=[SHIM])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules[_PKG] = pkg
    spec.loader.exec_module(pkg)
    loader = importlib.machinery.SourcelessFileLoader(name, PYC)
    spec = importlib.util.spec_from_file_location(name, PYC, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    loader.exec_module(mod)
    return mod
