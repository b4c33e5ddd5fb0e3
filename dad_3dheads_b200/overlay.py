"""The demo's landmark, pose and wireframe overlays drawn into whole frames on the GPU (csrc/overlay.cu), and head pose
angles.

``demo.py``'s ``68_landmarks``, ``191_landmarks``, ``445_landmarks``, ``pose``, ``head_mesh`` and ``face_mesh`` outputs are
cv2 drawings made by ``demo_utils.py`` (``draw_landmarks``, ``draw_3d_landmarks``, ``draw_mesh``, ``draw_pose``, lines
22-94), one image at a time on the host.
These functions draw the same pixels, byte for byte, for every box of a batch of frames, from device tensors and without a
host synchronisation, so they run inside a captured CUDA graph.  ``rpy`` is ``calculate_rpy``
(model_training/model/flame.py:254-259) for every head instead of head 0.  The drawing rules (cv2 4.13.0) are restated in
``tests/overlay_model.py`` and ``tests/wireframe_model.py``; DESIGN §4.8 lists them and what draws nothing.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib

OVERLAY_KINDS = ("68_landmarks", "191_landmarks", "445_landmarks", "pose", "head_mesh", "face_mesh")
POINT_COLOR = (255, 0, 0)                  # demo_utils.POINT_COLOR
EDGE_COLOR = (39, 48, 218)                 # demo_utils.EDGE_COLOR
POSE_RECORD_INTS = 32                      # DAD3D_POSE_RECORD_INTS, include/dad3d.h
MESH_WS_INTS = 5                           # DAD3D_MESH_WS_INTS
# the vertex subset whose edges draw_mesh draws: head_edges.npy is over the face with ears, not flame_indices_head
MESH_VERTICES = {"head_mesh": "flame_indices_face_w_ears", "face_mesh": "flame_indices_face"}
_POINT_COLOR = np.array(POINT_COLOR, dtype=np.uint8)
_EDGE_COLOR = np.array(EDGE_COLOR, dtype=np.uint8)


def mesh_edges(faces: np.ndarray, vertices: np.ndarray) -> np.ndarray:
    """[E,2] int32: the sorted unique (i < j) edges of the triangles ``faces`` with both ends in ``vertices``.  For the
    FLAME faces and a subset of MESH_VERTICES this is, row for row, the reference's ``{subset}_edges.npy``."""
    f = np.asarray(faces, dtype=np.int64)
    e = np.unique(np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1), axis=0)
    return np.ascontiguousarray(e[np.isin(e, np.asarray(vertices)).all(axis=1)], dtype=np.int32)


def point_radius(height: int, width: int) -> int:
    """draw_points' disk radius for an image of this size (demo_utils.py:26)."""
    return max(1, int(min(height, width) * 0.005))


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def pose_geometry(params: Tensor, rotation_index: int, rois: Optional[Tensor] = None) -> Tuple[Tensor, Optional[Tensor]]:
    """params [R,P] fp32 (device) -> ("rpy" [R,3] float64 degrees: roll, pitch, yaw of calculate_rpy, per head;
    the [R,32] int32 pose records of draw_pose in each box's crop view, when ``rois`` ([R,72] uint8 dad3d_roi records)
    is given, else None)."""
    assert params.dtype == torch.float32 and params.ndim == 2 and params.is_contiguous()
    R, P = (int(d) for d in params.shape)
    dev = params.device
    rpy = torch.empty(R, 3, dtype=torch.float64, device=dev)
    pose = torch.empty(R, POSE_RECORD_INTS, dtype=torch.int32, device=dev) if rois is not None else None
    lib = _lib.load()
    with torch.cuda.device(dev):
        _lib.check(lib.dad3d_pose_geometry(params.data_ptr(), R, P, int(rotation_index),
                                           rois.data_ptr() if rois is not None else None, rpy.data_ptr(),
                                           pose.data_ptr() if pose is not None else None, None, _stream(dev)),
                   "dad3d_pose_geometry")
    return rpy, pose


def rotation_matrices(params: Tensor, rotation_index: int) -> Tensor:
    """params [R,P] fp32 (device) -> [R,3,3] fp32: rot_mat_from_6dof (model/utils.py:92-101) of every head, as
    :func:`pose_geometry` computes it (bit-exact with torch on the CPU)."""
    assert params.dtype == torch.float32 and params.ndim == 2 and params.is_contiguous()
    R, P = (int(d) for d in params.shape)
    rot = torch.empty(R, 3, 3, dtype=torch.float32, device=params.device)
    lib = _lib.load()
    with torch.cuda.device(params.device):
        _lib.check(lib.dad3d_pose_geometry(params.data_ptr(), R, P, int(rotation_index), None, None, None, rot.data_ptr(),
                                           _stream(params.device)), "dad3d_pose_geometry")
    return rot


def draw_points(frames: Tensor, points: Tensor, rois: Tensor, index: Optional[Tensor] = None) -> None:
    """In place on frames [F,H,W,3] uint8 (device): draw_points of every valid box's points onto its frame.
    points [R,N,C] int64 (used as they are) or fp32 (truncated, as ``astype(int)``); ``index`` [L] int64 picks the points
    of each head (None: all N)."""
    assert frames.dtype == torch.uint8 and frames.ndim == 4 and frames.is_contiguous()
    assert points.dtype in (torch.int64, torch.float32) and points.ndim == 3 and points.is_contiguous()
    F, H, W = (int(d) for d in frames.shape[:3])
    R, N, C = (int(d) for d in points.shape)
    L = int(index.shape[0]) if index is not None else N
    lib = _lib.load()
    with torch.cuda.device(frames.device):
        _lib.check(lib.dad3d_overlay_points(points.data_ptr(), 1 if points.dtype == torch.float32 else 0, R, N, C,
                                            index.data_ptr() if index is not None else None, L, rois.data_ptr(),
                                            point_radius(H, W), _POINT_COLOR.ctypes.data, frames.data_ptr(), F, H, W,
                                            _stream(frames.device)), "dad3d_overlay_points")


def draw_pose(frames: Tensor, pose: Tensor) -> None:
    """In place on frames [F,H,W,3] uint8 (device): draw_pose's three arrows of every record of :func:`pose_geometry`,
    each box's into its crop view; where arrows overlap, the later box, then the later arrow, wins."""
    assert frames.dtype == torch.uint8 and frames.ndim == 4 and frames.is_contiguous()
    F, H, W = (int(d) for d in frames.shape[:3])
    key = torch.empty(F, H, W, dtype=torch.int32, device=frames.device)
    lib = _lib.load()
    with torch.cuda.device(frames.device):
        _lib.check(lib.dad3d_overlay_pose(pose.data_ptr(), int(pose.shape[0]), key.data_ptr(), frames.data_ptr(), F, H, W,
                                          _stream(frames.device)), "dad3d_overlay_pose")


def draw_mesh(frames: Tensor, vertices: Tensor, rois: Tensor, edges: Tensor) -> None:
    """In place on frames [F,H,W,3] uint8 (device): draw_mesh of every valid box's head onto its frame -- cv2.line(...,
    1, LINE_AA) of every edge of ``edges`` [E,2] int32 in order, the blends of a pixel in box order.  ``vertices``
    [R,N,2|3] fp32 (x, y truncated, as ``astype(int)``).  A box whose edges reach a point that is not finite or does not
    fit int32 draws nothing."""
    assert frames.dtype == torch.uint8 and frames.ndim == 4 and frames.is_contiguous()
    assert vertices.dtype == torch.float32 and vertices.ndim == 3 and vertices.is_contiguous()
    assert edges.dtype == torch.int32 and edges.ndim == 2 and edges.shape[1] == 2 and edges.is_contiguous()
    F, H, W = (int(d) for d in frames.shape[:3])
    R, N, C = (int(d) for d in vertices.shape)
    ws = torch.empty(R, MESH_WS_INTS, dtype=torch.int32, device=frames.device)
    lib = _lib.load()
    with torch.cuda.device(frames.device):
        _lib.check(lib.dad3d_overlay_mesh(vertices.data_ptr(), R, N, C, edges.data_ptr(), int(edges.shape[0]),
                                          rois.data_ptr(), _EDGE_COLOR.ctypes.data, ws.data_ptr(), frames.data_ptr(), F, H,
                                          W, _stream(frames.device)), "dad3d_overlay_mesh")
