"""GPU evaluator for the DAD-3DHeads benchmark (SURVEY §8f row 1): the four metrics of
``dad_3dheads_benchmark/benchmark.py::DADEvaluator`` -- pose error, NME of the reprojected 68 landmarks, Z5 ordinal-depth
accuracy and the chamfer distance -- computed for ALL annotated heads in a few batched launches instead of per-sample python
loops (calc_zn: O(K^2) cdist + K x 5 python iterations per head, benchmark.py:110-138; align_pred_to_gt: a python loop over
5023 vertices, utils.py:178-197; kaolin chamfer per head, utils.py:139).  Same inputs (ground-truth json + submission json),
same output structure (``overall_result, attribute_result``) as the reference's ``DADEvaluator.__call__``.

Heavy parts run in libdad3d.so (csrc/evaluator.cu: dad3d_eval_chamfer / dad3d_eval_zn / dad3d_eval_align, plus the landmark
gathers of csrc/flame.cu); the 7-point procrustes fit and the 3x3 pose algebra are a few hundred flops per head and stay in
torch on the device.  No CPU fallback.
"""
from __future__ import annotations

import json
from collections import defaultdict
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .flame import load_flame_static
from .submission import SEVEN_OF_68, landmark68_tables


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class DADEvaluatorGPU:
    def __init__(self, ground_truth_path: Optional[str] = None, submission_path: Optional[str] = None, cuda_id: int = 0,
                 static: Optional[Dict[str, np.ndarray]] = None):
        if not torch.cuda.is_available():
            raise _lib.Dad3dError("DADEvaluatorGPU needs a CUDA (sm_90a) device: there is no CPU path")
        self.lib = _lib.load()
        self.device = torch.device("cuda", cuda_id)
        self.target_file_path = ground_truth_path
        self.prediction_file_path = submission_path
        st = static if static is not None else load_flame_static()
        tri, bary = landmark68_tables(st)
        self.tri = tri.to(self.device, torch.int32).contiguous()
        self.bary = bary.to(self.device).contiguous()
        self.head_indices = torch.from_numpy(np.asarray(st["head_indices"], dtype=np.int32)).to(self.device)   # utils.py:310
        self.face_indices = torch.from_numpy(np.asarray(st["flame_indices_face"], dtype=np.int32)).to(self.device)
        self.seven = torch.tensor(SEVEN_OF_68, device=self.device)

    # ------------------------------------------------------------------ thin wrappers over the C ABI
    def _gather(self, src: Tensor, idx: Tensor) -> Tensor:
        src = src.contiguous()
        B, V, nc = src.shape
        out = torch.empty(B, idx.numel(), nc, dtype=torch.float32, device=self.device)
        _lib.check(self.lib.dad3d_gather_landmarks(src.data_ptr(), B, V, nc, idx.data_ptr(), idx.numel(), out.data_ptr(),
                                                   _stream(self.device)), "dad3d_gather_landmarks")
        return out

    def _lm68(self, verts: Tensor) -> Tensor:
        verts = verts.contiguous()
        B, V, nc = verts.shape
        out = torch.empty(B, 68, nc, dtype=torch.float32, device=self.device)
        _lib.check(self.lib.dad3d_gather_landmarks_bary(verts.data_ptr(), B, V, nc, self.tri.data_ptr(), self.bary.data_ptr(),
                                                        68, out.data_ptr(), _stream(self.device)), "dad3d_gather_landmarks_bary")
        return out

    def _align(self, verts: Tensor, scale: Tensor, rot: Tensor, trans: Tensor) -> Tensor:
        B, V, _ = verts.shape
        # keep every contiguous copy alive until the launch has been enqueued: a temporary released between two
        # ``.contiguous()`` calls hands its block straight to the next one (same stream), which would overwrite it
        verts, scale, rot, trans = verts.contiguous(), scale.contiguous(), rot.contiguous(), trans.contiguous()
        out = torch.empty_like(verts)
        _lib.check(self.lib.dad3d_eval_align(verts.data_ptr(), V, B, scale.data_ptr(), rot.data_ptr(), trans.data_ptr(),
                                             out.data_ptr(), _stream(self.device)), "dad3d_eval_align")
        return out

    def chamfer_one_sided(self, a: Tensor, b: Tensor) -> Tensor:
        B = a.shape[0]
        a, b = a.contiguous(), b.contiguous()
        out = torch.empty(B, dtype=torch.float32, device=self.device)
        _lib.check(self.lib.dad3d_eval_chamfer(a.data_ptr(), a.shape[1], b.data_ptr(), b.shape[1], B, out.data_ptr(),
                                               _stream(self.device)), "dad3d_eval_chamfer")
        return out

    def calc_zn(self, pred: Tensor, gt: Tensor, top_k: int = 5) -> Tensor:
        """[B,K,3] x2 -> [B] (benchmark.py:110-138, its index selection included)."""
        B, K, _ = gt.shape
        pred, gt = pred.contiguous(), gt.contiguous()
        out = torch.empty(B, dtype=torch.float32, device=self.device)
        _lib.check(self.lib.dad3d_eval_zn(pred.data_ptr(), gt.data_ptr(), K, B, top_k, out.data_ptr(), _stream(self.device)),
                   "dad3d_eval_zn")
        return out

    # ------------------------------------------------------------------ the four metrics, batched
    def metrics(self, annotations: List[Dict[str, Any]], predictions: List[Dict[str, Any]]) -> Dict[str, np.ndarray]:
        dev = self.device
        f32 = lambda key, src: torch.tensor(np.asarray([s[key] for s in src], dtype=np.float32), device=dev)
        with torch.cuda.device(dev):
            verts = f32("vertices", annotations)                                  # [B,5023,3] model space
            mv = f32("model_view_matrix", annotations)                            # [B,4,4]
            pm = f32("projection_matrix", annotations)
            B = verts.shape[0]
            bbox = f32("bbox", annotations)
            height = f32("image_height", annotations)
            pred_v = f32("N_landmarks_3d", predictions).reshape(B, -1, 3).contiguous()
            pred_7 = f32("7_landmarks_3d", predictions).reshape(B, 7, 3)
            pred_2d = f32("68_landmarks_2d", predictions).reshape(B, 68, 2)
            R_pred = f32("rotation_matrix", predictions).reshape(B, 3, 3)
            ones = torch.ones(B, device=dev)
            # world coordinates (benchmark.py:43-45): v @ mv[:3,:3]^T + mv[:3,3]
            world = self._align(verts, ones, mv[:, :3, :3].transpose(1, 2), mv[:, :3, 3])
            # ---- pose error (:80-85)
            rot_180 = torch.diag(torch.tensor([1.0, -1.0, -1.0], device=dev))
            R_gt = rot_180 @ mv[:, :3, :3]
            pose = torch.linalg.matrix_norm(torch.eye(3, device=dev) - R_pred @ R_gt.transpose(1, 2), "fro")
            # ---- NME of the reprojected 68 landmarks (:29-37, :87-99)
            lm = self._lm68(verts)
            lmh = torch.cat([lm, torch.ones(B, 68, 1, device=dev)], -1)
            q = (pm @ (mv @ lmh.transpose(1, 2))).transpose(1, 2)
            q2 = q[..., :2] / q[..., 3:4]
            gt2d = torch.stack((q2[..., 0], height[:, None] - q2[..., 1]), -1)
            nme = (torch.linalg.vector_norm(gt2d - pred_2d, dim=-1) / torch.sqrt(bbox[:, 2] * bbox[:, 3])[:, None]).mean(1) * 100.0
            # ---- chamfer (:101-108, utils.py:122-197)
            l68w = self._lm68(world)
            g7 = l68w[:, self.seven]
            scale = 20.0 / torch.linalg.vector_norm(g7[:, 1] - g7[:, 2], dim=-1)      # scale_gt_to_standard
            gt_s = world * scale[:, None, None]
            g7 = g7 * scale[:, None, None]                                            # landmarks are linear in the vertices
            T, b, c = self._procrustes(g7.double(), pred_7.double())
            aligned = self._align(pred_v, b.float(), T.float(), c.float())
            gface = self._gather(gt_s.contiguous(), self.face_indices)
            chamfer = self.chamfer_one_sided(gface, aligned)
            # ---- Z5 (:140-151)
            gt_head = self._gather(world, self.head_indices) * -1.0
            pred_head = self._gather(pred_v, self.head_indices)
            z5 = self.calc_zn(pred_head, gt_head, 5)
            torch.cuda.synchronize(dev)
        return {"pose_error": pose.cpu().numpy(), "nme": nme.cpu().numpy(), "z5": z5.cpu().numpy(),
                "chamfer": chamfer.cpu().numpy()}

    @staticmethod
    def _procrustes(X: Tensor, Y: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
        """Batched utils.py:200-298 (scaling, best reflection): rotation T, scale b, translation c with Y b T + c ~ X."""
        muX, muY = X.mean(1, keepdim=True), Y.mean(1, keepdim=True)
        X0, Y0 = X - muX, Y - muY
        normX = torch.sqrt((X0 ** 2).sum((1, 2)))
        normY = torch.sqrt((Y0 ** 2).sum((1, 2)))
        X0, Y0 = X0 / normX[:, None, None], Y0 / normY[:, None, None]
        U, s, Vt = torch.linalg.svd(X0.transpose(1, 2) @ Y0, full_matrices=False)
        T = Vt.transpose(1, 2) @ U.transpose(1, 2)
        b = s.sum(1) * normX / normY
        c = muX[:, 0] - b[:, None] * (muY[:, 0][:, None, :] @ T)[:, 0]
        return T, b, c

    # ------------------------------------------------------------------ the reference's entry point (:153-196)
    def __call__(self, batch: int = 256):
        with open(self.prediction_file_path) as f:
            submission = json.load(f)
        with open(self.target_file_path) as f:
            ground_truth = json.load(f)
        names = {"pose_error": "pose_error", "nme": "nme_reprojection", "z5": "z5_accuracy", "chamfer": "chamfer"}
        metrics = {n: {"overall": [], "attributes": defaultdict(lambda: defaultdict(list))} for n in names}
        todo = [a for a in ground_truth if a["id"] in submission]
        for a in ground_truth:
            if a["id"] not in submission:
                print(f'No prediction with ID: {a["id"]}.')
        for i in range(0, len(todo), batch):
            chunk = todo[i:i + batch]
            res = self.metrics(chunk, [submission[a["id"]] for a in chunk])
            for j, a in enumerate(chunk):
                for n in names:
                    v = float(res[n][j])
                    metrics[n]["overall"].append(v)
                    if a.get("attributes") is not None:
                        for attr_name, attr_value in a["attributes"].items():
                            metrics[n]["attributes"][attr_name][attr_value].append(v)
        overall = {out: np.mean(metrics[n]["overall"]) for n, out in names.items()}
        attribute_result = {}
        for n, out in names.items():
            attribute_result[out] = {}
            for attr_name, attr_values in metrics[n]["attributes"].items():
                attribute_result[out][attr_name] = {k: np.mean(v) for k, v in attr_values.items()}
        return overall, attribute_result
