"""ctypes binding of libdad3d.so (include/dad3d.h).  Fails loudly: no library / no GPU => exception, never a fallback."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DAD3D_LIB_PATH") or os.path.join(_HERE, "libdad3d.so")   # override: A/B runs of two builds

DAD3D_ZERO_ROT = 1
DAD3D_ZERO_JAW = 2
DAD3D_BLEND_FAST = 4
DAD3D_BLEND_SIMT = 8
DAD3D_DECODE_UNFUSED = 16
DAD3D_DECODE_CLUSTER = 32
DAD3D_BLEND_HILO = 64
DAD3D_DECODE_PAIR = 128


class Dad3dError(RuntimeError):
    pass


class FlameLayout(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("shape", "expression", "jaw", "rotation", "eyeballs", "neck", "translation",
                                         "scale")]


class Lighting(C.Structure):
    """dad3d_lighting: RenderPipeline's parameters (Sim3DR/lighting.py:24-32), passed by value."""
    _fields_ = [("intensity_ambient", C.c_float), ("intensity_directional", C.c_float), ("intensity_specular", C.c_float),
                ("specular_exp", C.c_int32), ("color_ambient", C.c_float * 3), ("color_directional", C.c_float * 3),
                ("light_pos", C.c_float * 3), ("view_pos", C.c_float * 3)]


_lib = None

# every symbol include/dad3d.h declares: (restype, argtypes)
_f32p = C.c_void_p
SIGNATURES = {
    "dad3d_last_error": (C.c_char_p, []),
    "dad3d_version": (C.c_int, []),
    "dad3d_launch_count": (C.c_ulonglong, []),
    "dad3d_flame_create": (C.c_int, [C.POINTER(C.c_void_p), _f32p, _f32p, _f32p, _f32p, C.c_void_p, _f32p, C.c_int32,
                                      C.c_int32, C.c_int32, C.POINTER(FlameLayout), C.c_int32]),
    "dad3d_flame_destroy": (None, [C.c_void_p]),
    "dad3d_flame_num_params": (C.c_int32, [C.c_void_p]),
    "dad3d_flame_num_vertices": (C.c_int32, [C.c_void_p]),
    "dad3d_flame_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32]),
    "dad3d_flame_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_float,
                                      C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dad3d_flame_prep": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int32, C.c_void_p]),
    "dad3d_flame_decode_from": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                           C.c_void_p, C.c_float, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dad3d_flame_describe": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_char_p, C.c_size_t]),
    "dad3d_flame_backward_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32]),
    "dad3d_flame_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_float,
                                        C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dad3d_flame_backward_blend": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "dad3d_flame_backward_vertex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_float,
                                               C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_flame_backward_dense": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "dad3d_flame_backward_finalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_gather_landmarks": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                          C.c_void_p, C.c_void_p]),
    "dad3d_gather_landmarks_bary": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                               C.c_int32, C.c_void_p, C.c_void_p]),
    "dad3d_encoder_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_int32]),
    "dad3d_encoder_destroy": (None, [C.c_void_p]),
    "dad3d_encoder_num_layers": (C.c_int, [C.c_void_p]),
    "dad3d_encoder_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32]),
    "dad3d_encoder_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    "dad3d_preprocess": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_preprocess_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_roi_setup": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "dad3d_preprocess_rois": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_readjust_rois": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_rasterize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "dad3d_rasterize_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "dad3d_rasterize_frames": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dad3d_vertex_normals": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "dad3d_light_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                    Lighting, C.c_void_p, C.c_void_p]),
    "dad3d_render_lit": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_int32, Lighting, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]),
    "dad3d_pose_geometry": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "dad3d_overlay_points": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p]),
    "dad3d_overlay_pose": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p]),
    "dad3d_overlay_mesh": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "dad3d_comm_unique_id": (C.c_int, [C.c_void_p]),
    "dad3d_comm_init": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "dad3d_comm_destroy": (None, [C.c_void_p]),
    "dad3d_bcast_constants": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32, C.c_void_p]),
    "dad3d_allgather_outputs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dad3d_eval_chamfer": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "dad3d_eval_zn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "dad3d_eval_align": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "dad3d_encoder_set_profile": (C.c_int, [C.c_void_p, C.c_int32]),
    "dad3d_encoder_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_longlong),
                                              C.POINTER(C.c_double)]),
    "dad3d_encoder_profile_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_double),
                                               C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int32)]),
    "dad3d_encoder_set_debug": (C.c_int, [C.c_void_p, C.c_int32]),
    "dad3d_encoder_read_activation": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t,
                                                 C.POINTER(C.c_int32), C.c_void_p]),
    "dad3d_encoder_describe_plan": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "dad3d_encoder_write_activation": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dad3d_encoder_run_steps": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
}


def load():
    """Load libdad3d.so (built in-tree by __graft_entry__.build() / csrc/Makefile)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise Dad3dError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                         f"(there is no CPU fallback for this path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().dad3d_last_error()
        raise Dad3dError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def launch_count() -> int:
    return int(load().dad3d_launch_count())
