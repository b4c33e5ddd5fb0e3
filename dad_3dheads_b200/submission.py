"""Producer of DAD-3DHeads benchmark submissions (SURVEY §8f "next" row 1) from the GPU path's outputs.

The evaluator (dad_3dheads_benchmark/benchmark.py:153-196) reads a JSON ``{item_id: {"68_landmarks_2d": [68][2],
"N_landmarks_3d": [N][3], "7_landmarks_3d": [7][3], "rotation_matrix": [3][3]}}`` (dad_3dheads_benchmark/README.md:78-90).
Here those four fields are produced for a whole batch on the device:
  * 68 landmarks = 17 dynamic-contour (zero-pose row of flame_dynamic_embedding) + 51 static barycentric embeddings
    evaluated on the mesh (model_training/data/utils.py:120-206 ``get_68_landmarks``) -- ``dad3d_gather_landmarks_bary``,
  * "68_landmarks_2d": the same embedding evaluated on the PROJECTED vertices (image pixels),
  * "7_landmarks_3d": rows [36, 39, 42, 45, 33, 48, 54] of the 3-D 68 set (dad_3dheads_benchmark/utils.py:143-150),
  * "rotation_matrix": rot_mat_from_6dof(params[403:409]) (model_training/model/utils.py:92-101), computed on the host in
    torch from the 6 numbers per head (trivial work; everything heavy stays on the GPU).
"""
from __future__ import annotations

import json
from typing import Dict, Iterable, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from .flame import load_flame_static

SEVEN_OF_68 = (36, 39, 42, 45, 33, 48, 54)


def landmark68_tables(static: Optional[Dict[str, np.ndarray]] = None) -> Tuple[Tensor, Tensor]:
    """(triangle vertex indices [68,3] int64, barycentric coordinates [68,3] fp32): dynamic (row 0) then static."""
    st = static if static is not None else load_flame_static()
    faces = torch.from_numpy(np.asarray(st["faces"], dtype=np.int64))
    dyn_f = torch.from_numpy(np.asarray(st["dynamic_lmk_face_idx"], dtype=np.int64))[0]      # zero pose -> row 0
    dyn_b = torch.from_numpy(np.asarray(st["dynamic_lmk_b_coords"], dtype=np.float32))[0]
    sta_f = torch.from_numpy(np.asarray(st["static_lmk_face_idx"], dtype=np.int64))
    sta_b = torch.from_numpy(np.asarray(st["static_lmk_b_coords"], dtype=np.float32))
    tri = faces[torch.cat([dyn_f, sta_f])]
    bary = torch.cat([dyn_b, sta_b])
    return tri, bary


def rot_mat_from_6dof(v: Tensor) -> Tensor:
    """Columns b1, b2, b3 by Gram-Schmidt (model/utils.py:92-101; cross products over the last axis)."""
    v = v.reshape(-1, 6).float()
    b1 = torch.nn.functional.normalize(v[:, :3], dim=-1)
    b3 = torch.nn.functional.normalize(torch.linalg.cross(b1, v[:, 3:], dim=-1), dim=-1)
    b2 = -torch.linalg.cross(b1, b3, dim=-1)
    return torch.stack((b1, b2, b3), dim=-1)


class SubmissionWriter:
    def __init__(self, predictor, static: Optional[Dict[str, np.ndarray]] = None):
        self.pred = predictor
        tri, bary = landmark68_tables(static)
        self.tri = tri.to(predictor.device)
        self.bary = bary.to(predictor.device)
        c = predictor.flame_constants
        self.rot_off = c["shape"] + c["expression"] + c["jaw"]

    def fields_from_outputs(self, out: Dict[str, Tensor]) -> Dict[str, Tensor]:
        """out = FaceMeshPredictor.predict_batch(...) (device tensors) -> the four benchmark fields as device tensors."""
        dec = self.pred.head_mesh.flame.decoder(self.pred.device)
        lm3d = dec.gather_bary(out["3d_vertices"], self.tri, self.bary)                       # [B,68,3]
        lm2d = dec.gather_bary(out["projected_vertices"][..., :2].contiguous(), self.tri, self.bary)   # [B,68,2]
        seven = lm3d[:, list(SEVEN_OF_68)]
        rot = rot_mat_from_6dof(out["3dmm_params"][:, self.rot_off:self.rot_off + 6])
        return {"68_landmarks_2d": lm2d, "N_landmarks_3d": out["3d_vertices"], "7_landmarks_3d": seven,
                "rotation_matrix": rot}

    def letterbox_geometry(self, shapes) -> Tensor:
        """[(h, w), ...] of the ORIGINAL images -> [B,3] (pad_left, pad_top, scale) of the letter-box the predictor applies
        (predictor.py:117-123: scale = 256/max(h,w), py3round-ed size, centred padding)."""
        from .predictor import calculate_paddings, py3round
        S = self.pred._img_size
        rows = []
        for h, w in shapes:
            scale = S / float(max(h, w))
            nh, nw = (py3round(h * scale), py3round(w * scale))
            pads = calculate_paddings(nh, nw)
            rows.append([float(pads[2]), float(pads[0]), scale])
        return torch.tensor(rows, dtype=torch.float32, device=self.pred.device)

    def predict(self, images, item_ids: Iterable[str], input_shapes=None, boxes=None, frame_index=None,
                extend=0.0) -> Dict[str, Dict[str, list]]:
        """images: raw RGB frames (list of HxWx3 uint8 arrays/tensors of any sizes, or one [B,H,W,3] uint8 tensor) -- the
        benchmark's inputs -- or an already letter-boxed [B,3,256,256] fp32 batch together with ``input_shapes`` =
        [(h, w), ...] of the originals.  "68_landmarks_2d" is returned in ORIGINAL-image pixels, which is what the evaluator
        compares with its ground truth (dad_3dheads_benchmark/benchmark.py:86-99): the letter-box is undone exactly as
        ``readjust_3dmm_to_the_input_image`` + ``reprojected_vertices`` do in the reference (predictor.py:154-176,
        head_mesh.py:33-46): xy_orig = (xy_256 - [pad_left, pad_top]) / scale.

        With ``boxes`` ([R,4] integer [x, y, w, h], one per item, as the benchmark's metadata gives them), ``images`` is one
        [F,H,W,3] uint8 tensor of whole frames and item r is the head in box r on frame ``frame_index[r]`` (default: frame r).
        The heads are cropped and read back into frame pixels by ``predict_batch(..., boxes=)``, so "68_landmarks_2d" is the
        barycentric 68 on the frame-space projected vertices: already in the evaluator's full-image frame."""
        if boxes is not None:
            R = int(torch.as_tensor(boxes).shape[0])
            if frame_index is None:
                if not (isinstance(images, Tensor) and images.ndim == 4 and int(images.shape[0]) == R):
                    raise ValueError("boxes without frame_index need one frame per box")
                frame_index = torch.arange(R, dtype=torch.int32)
            out = self.pred.predict_batch(images, landmark_subset=None, to_2d=True, boxes=boxes, frame_index=frame_index,
                                          extend=extend)
            return self._items(self.fields_from_outputs(out), item_ids)
        if input_shapes is None:
            if isinstance(images, (list, tuple)):
                input_shapes = [tuple(int(d) for d in torch.as_tensor(im).shape[:2]) for im in images]
            elif isinstance(images, Tensor) and images.dtype == torch.uint8:
                input_shapes = [(int(images.shape[1]), int(images.shape[2]))] * int(images.shape[0])
        out = self.pred.predict_batch(images, landmark_subset=None, to_2d=True)
        fields = self.fields_from_outputs(out)
        if input_shapes is not None:
            geo = self.letterbox_geometry(input_shapes)                            # [B,3]
            fields["68_landmarks_2d"] = (fields["68_landmarks_2d"] - geo[:, None, :2]) / geo[:, None, 2:3]
        return self._items(fields, item_ids)

    @staticmethod
    def _items(fields: Dict[str, Tensor], item_ids: Iterable[str]) -> Dict[str, Dict[str, list]]:
        f = {k: v.detach().cpu() for k, v in fields.items()}
        res = {}
        for i, item in enumerate(item_ids):
            res[str(item)] = {k: f[k][i].tolist() for k in f}
        return res

    @staticmethod
    def save(submission: Dict[str, Dict[str, list]], path: str) -> None:
        with open(path, "w") as fd:
            json.dump(submission, fd)
