"""Host-side mirror of the reference's inference API (predictor.py:68-211) over libdad3d.so.

``FaceMeshPredictor`` keeps the reference's constructor, ``dad_3dnet()``, ``__call__`` (HxWx3 uint8 RGB -> dict with
"points", "projected_vertices", "3d_vertices", "3dmm_params"), the overridable ``preprocess / process / postprocess``
stages and their helper names, so ``demo.py`` / ``demo_utils.py`` code written against the reference keeps working.
What changes is where the arithmetic runs: ``self.model`` is the CUDA encoder (csrc/encoder.cu) instead of a TorchScript
module, and ``self.head_mesh`` decodes on the GPU (csrc/flame.cu), once instead of twice per image.
``predict_batch`` is the batched, device-resident entry point the reference does not have (SURVEY §8b); with ``render`` it
also draws the PNCC, depth and triangle-index maps of every head (rasterizer.PnccRenderer) and its lit render
(rasterizer.LitRenderer, the reference's Sim3DR RenderPipeline) inside the same step, and with ``boxes`` plus
``frame_render`` the same maps of every whole frame, all its heads in one z-buffer.
"""
from __future__ import annotations

import logging
import os
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch
import yaml
from torch import Tensor

from . import _lib
from .encoder import OUTPUT_2D_LANDMARKS, OUTPUT_3DMM_PARAMS, OUTPUT_LANDMARKS_HEATMAP, Dad3dEncoder
from .flame import load_flame_static
from .head_mesh import HeadMesh
from .rasterizer import LitRenderer, PnccRenderer

logger = logging.getLogger(__name__)
ROI_RECORD_BYTES = 72                                # sizeof(dad3d_roi), include/dad3d.h
MAX_ROIS = 65535                                     # ROIs per call: dad3d_preprocess_rois runs them along grid z
_FILENAME = "dad_3dheads.trcd"
_MEAN = (0.485, 0.456, 0.406)
_STD = (0.229, 0.224, 0.225)
RENDER_KEYS = ("pncc", "depth", "tri_index", "lit")
FRAME_RENDER_KEYS = ("pncc", "depth", "tri_index", "head_index", "lit")    # predict_batch(boxes=, frame_render=) -> "frame_<key>"

DEFAULT_CONFIG = {                                   # == the reference's dad_3dnet.yaml
    "model_path": ".dad_checkpoints/dad_3dheads.trcd",
    "stride": 4,
    "img_size": 256,
    "constants": {"shape": 300, "expression": 100, "jaw": 3, "rotation": 6, "eyeballs": 0, "neck": 0,
                  "translation": 3, "scale": 1},
}


def load_yaml(path: str) -> Dict[str, Any]:
    with open(path) as fd:
        return yaml.load(fd, yaml.FullLoader)


def model_exists() -> bool:
    return os.path.isfile(os.path.join(os.path.expanduser("~"), ".dad_checkpoints", _FILENAME))


def py3round(number: float) -> int:
    """albumentations.augmentations.geometric.py3round == Python-3 (banker's) rounding to int (predictor.py:12,121)."""
    return int(round(number))


def calculate_paddings(orig_h: int, orig_w: int) -> List[int]:
    """model_training/model/utils.py:71-77 -> [pad_top, pad_bottom, pad_left, pad_right] to a centred square."""
    side = max(orig_h, orig_w)
    top = int((side - orig_h) / 2)
    left = int((side - orig_w) / 2)
    return [top, side - orig_h - top, left, side - orig_w - left]


def extend_sides(extend) -> Tuple[float, float, float, float]:
    """``extend_bbox``'s offset (model_training/data/utils.py:73-100) -- one fraction, (width, height) or
    (left, right, top, bottom) -- as the four fractions (left, right, top, bottom)."""
    if isinstance(extend, (tuple, list)):
        if len(extend) == 4:
            return tuple(float(v) for v in extend)
        if len(extend) == 2:
            return (float(extend[0]),) * 2 + (float(extend[1]),) * 2
        raise ValueError(f"extend: a float, a 2-tuple or a 4-tuple, got {len(extend)} values")
    return (float(extend),) * 4


def letterbox_normalise(x: np.ndarray, img_size: int) -> np.ndarray:
    """predictor.py:195-203 (albumentations 1.0.0 LongestMaxSize -> PadIfNeeded(constant 0, centred) -> Normalize),
    restated with cv2/numpy: HxWx3 uint8 RGB -> img_size x img_size x 3 float32."""
    import cv2
    h, w = x.shape[:2]
    scale = img_size / float(max(w, h))
    if scale != 1.0:
        nh, nw = py3round(h * scale), py3round(w * scale)
        x = cv2.resize(x, dsize=(nw, nh), interpolation=cv2.INTER_LINEAR)
    h, w = x.shape[:2]
    top = int((img_size - h) / 2.0) if h < img_size else 0
    bottom = (img_size - h - top) if h < img_size else 0
    left = int((img_size - w) / 2.0) if w < img_size else 0
    right = (img_size - w - left) if w < img_size else 0
    if top or bottom or left or right:
        x = cv2.copyMakeBorder(x, top, bottom, left, right, cv2.BORDER_CONSTANT, value=0)
    mean = np.array(_MEAN, dtype=np.float32) * 255.0
    denom = np.reciprocal(np.array(_STD, dtype=np.float32) * 255.0, dtype=np.float32)
    out = x.astype(np.float32)
    out -= mean
    out *= denom
    return out


class FaceMeshPredictor:
    def __init__(self, config: Dict[str, Any], cuda_id: int = 0, state_dict: Optional[Dict[str, Tensor]] = None,
                 precision: str = "fp32"):
        if not torch.cuda.is_available():
            raise _lib.Dad3dError("FaceMeshPredictor needs a CUDA (sm_90a) device: there is no CPU path")
        self.cuda_id = cuda_id
        self.device = torch.device("cuda", cuda_id)
        self.flame_constants = config["constants"]
        if state_dict is None:
            path = os.path.join(os.path.expanduser("~"), config["model_path"])
            if not os.path.isfile(path):
                raise FileNotFoundError(
                    f"{path} not found. The reference downloads its TorchScript checkpoint on first use "
                    f"(predictor.py:205-211); offline, pass state_dict= (e.g. encoder_weights.synthetic_state_dict).")
            state_dict = torch.jit.load(path, map_location="cpu").state_dict()
        self.model = Dad3dEncoder(state_dict, self.device, precision=precision).eval()
        self.head_mesh = HeadMesh(self.flame_constants, cuda_id=cuda_id)
        self._img_size = config["img_size"]
        self._stride = config.get("stride", 2)
        self._static = None
        self._lm_index: Dict[str, Tensor] = {}
        self._graphs: Dict[Any, Any] = {}
        self._renderer: Optional[PnccRenderer] = None
        self._lit_renderer: Optional[LitRenderer] = None

    # ------------------------------------------------------------------ reference single-image API
    def __call__(self, x: Any) -> Any:
        cache: Dict[str, Any] = {}
        x = self.preprocess(x, cache)
        res = self.process(x, cache)
        return self.postprocess(res, cache)

    @staticmethod
    def _array_to_batch(x: np.ndarray) -> Tensor:
        return torch.from_numpy(np.expand_dims(np.transpose(x, (2, 0, 1)), 0))

    def _transform(self, x: np.ndarray) -> np.ndarray:
        return letterbox_normalise(x, self._img_size)

    def preprocess(self, x: np.ndarray, cache: Dict[str, Any], *kw: Any) -> Tensor:
        cache["input_shape"] = x.shape[:2]
        x = self._array_to_batch(self._transform(x))
        return x.to(self.device)

    def process(self, x: Tensor, *kw: Any) -> Dict[str, Tensor]:
        with torch.no_grad():
            return self.model(x)

    def _parse_output(self, x: Dict[str, Tensor]):
        pred_3dmm = x[OUTPUT_3DMM_PARAMS].detach().cpu()
        if OUTPUT_2D_LANDMARKS in x.keys():
            pred_landmarks = x[OUTPUT_2D_LANDMARKS].detach().cpu().numpy() * 256.0
        elif OUTPUT_LANDMARKS_HEATMAP in x.keys():
            hm = torch.sigmoid(x[OUTPUT_LANDMARKS_HEATMAP]).detach()
            B, C_, H, W = hm.shape                                    # model/utils.py:38-52 (divides by H for both axes)
            idx = hm.view(B, C_, -1).argmax(-1).view(-1, 1)
            kp = torch.cat((torch.div(idx, H, rounding_mode="trunc"), idx % H), dim=1).reshape(B, C_, 2)
            pred_landmarks = float(self._stride) * kp.flip(-1)[0].cpu().numpy()
        else:
            return pred_3dmm
        return pred_landmarks, pred_3dmm

    def _get_paddings(self, cache: Dict[str, Any]) -> Tuple[List[int], float]:
        h, w = cache["input_shape"]
        scale = self._img_size / float(max(h, w))
        new_h, new_w = tuple(py3round(dim * scale) for dim in (h, w))
        return calculate_paddings(new_h, new_w), scale

    def readjust_landmarks_to_the_input_image(self, landmarks: np.ndarray, paddings: List[int], scale: float):
        landmarks = landmarks - np.array([[paddings[2], paddings[0]]])
        return (landmarks / scale).astype(int)

    @staticmethod
    def find_3dmm_idx(key: str, consts: Dict[str, int]) -> int:
        idx = 0
        for k, v in consts.items():
            if k == key:
                break
            idx += v
        return idx

    def readjust_3dmm_to_the_input_image(self, pred_3dmm: Tensor, paddings: List[int], scale: float) -> Tensor:
        """predictor.py:154-176 -- in place on the 413-vector, so projections land in input-image pixels."""
        si = self.find_3dmm_idx("scale", self.flame_constants)
        ti = self.find_3dmm_idx("translation", self.flame_constants)
        ns, nt = self.flame_constants["scale"], self.flame_constants["translation"]
        new_scale = (pred_3dmm[:, si:si + ns] + 1.0) / scale - 1.0
        pad = torch.tensor([[paddings[2], paddings[0], 0]], dtype=pred_3dmm.dtype, device=pred_3dmm.device)
        new_t = (pred_3dmm[:, ti:ti + nt] + 1.0 - pad * 2 / self._img_size) / scale - 1.0
        pred_3dmm[:, si:si + ns] = new_scale
        pred_3dmm[:, ti:ti + nt] = new_t
        return pred_3dmm

    def _get_predictions(self, x, cache: Dict[str, Any]) -> Dict[str, Any]:
        paddings, scale = self._get_paddings(cache)
        if type(x) is tuple:
            landmarks, pred_3dmm = x
            landmarks = landmarks.clip(min=0, max=self._img_size)
            landmarks = self.readjust_landmarks_to_the_input_image(landmarks, paddings, scale)
            pred_3dmm = self.readjust_3dmm_to_the_input_image(pred_3dmm, paddings, scale)
            # the reference decodes twice (predictor.py:136-137); one GPU pass yields both outputs
            v3, proj = self.head_mesh.decode(pred_3dmm, to_2d=True, hilo=True)     # per-image path: strict blend
            ti = self.find_3dmm_idx("translation", self.flame_constants)
            pred_3dmm[:, ti + 2] = 0.0                       # side effect of reprojected_vertices (head_mesh.py:41)
            return {"points": landmarks, "projected_vertices": proj, "3d_vertices": v3[0].squeeze(),
                    "3dmm_params": pred_3dmm}
        return {"3dmm_params": self.readjust_3dmm_to_the_input_image(x, paddings, scale)}

    def postprocess(self, x, cache: Dict[str, Any], *kw: Any) -> Dict[str, Any]:
        predictions = self._get_predictions(self._parse_output(x), cache)
        if "points" in predictions.keys():
            predictions["points"] = np.reshape(predictions["points"], (-1, 2))
        return predictions

    @classmethod
    def dad_3dnet(cls, state_dict: Optional[Dict[str, Tensor]] = None, precision: str = "fp32", cuda_id: int = 0):
        here = os.path.dirname(os.path.abspath(__file__))
        cfg_path = os.path.join(here, "dad_3dnet.yaml")
        config = load_yaml(cfg_path) if os.path.isfile(cfg_path) else dict(DEFAULT_CONFIG)
        return cls(config=config, cuda_id=cuda_id, state_dict=state_dict, precision=precision)

    # ------------------------------------------------------------------ device-side pre-processing (SURVEY §8f row 2)
    def preprocess_batch(self, images) -> Tensor:
        """images: list of HxWx3 uint8 RGB arrays/tensors (any sizes).  -> [B,3,S,S] fp32 on the GPU, bit-identical to
        ``_transform`` (cv2 INTER_LINEAR letter-box + constant-0 pad + imagenet normalisation); only the raw uint8
        pixels cross the PCIe bus."""
        lib = _lib.load()
        S = self._img_size
        mean = (np.array(_MEAN, dtype=np.float32) * 255.0).astype(np.float32)
        inv = np.reciprocal(np.array(_STD, dtype=np.float32) * 255.0, dtype=np.float32)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        if isinstance(images, Tensor) and images.ndim == 4:
            # one [B,H,W,3] uint8 tensor (host, ideally pinned, or device): one copy, one launch
            assert images.dtype == torch.uint8 and images.shape[3] == 3
            B, h, w = int(images.shape[0]), int(images.shape[1]), int(images.shape[2])
            scale = S / float(max(h, w))
            nh, nw = (py3round(h * scale), py3round(w * scale)) if scale != 1.0 else (h, w)
            out = torch.empty(B, 3, S, S, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                d = images.contiguous().to(self.device, non_blocking=True)
                _lib.check(lib.dad3d_preprocess_batch(d.data_ptr(), B, h, w, nh, nw, S, mean.ctypes.data, inv.ctypes.data,
                                                      out.data_ptr(), stream), "dad3d_preprocess_batch")
                d.record_stream(torch.cuda.current_stream(self.device))
            return out
        out = torch.empty(len(images), 3, S, S, dtype=torch.float32, device=self.device)
        keep = []
        with torch.cuda.device(self.device):
            for i, im in enumerate(images):
                t = torch.as_tensor(im)
                assert t.dtype == torch.uint8 and t.ndim == 3 and t.shape[2] == 3
                h, w = int(t.shape[0]), int(t.shape[1])
                scale = S / float(max(h, w))
                nh, nw = (py3round(h * scale), py3round(w * scale)) if scale != 1.0 else (h, w)
                d = t.contiguous().to(self.device, non_blocking=True)
                keep.append(d)
                _lib.check(lib.dad3d_preprocess(d.data_ptr(), h, w, nh, nw, S, mean.ctypes.data, inv.ctypes.data,
                                                out[i].data_ptr(), stream), "dad3d_preprocess")
        return out

    # ------------------------------------------------------------------ batched device-resident API (new)
    def _landmark_index(self, subset: str) -> Tensor:
        subset = str(subset)
        if subset not in self._lm_index:                     # uploaded once (no per-call H2D copy; graph-capture safe)
            if self._static is None:
                self._static = load_flame_static()
            key = {"191": "keypoints_191", "445": "keypoints_445", "565": "keypoints_565"}[subset]
            self._lm_index[subset] = torch.from_numpy(self._static[key].astype(np.int64)).to(self.device)
        return self._lm_index[subset]

    @staticmethod
    def _render_keys(render, to_2d: bool) -> Tuple[str, ...]:
        """``render`` as a canonical tuple (the order of RENDER_KEYS), validated."""
        if render is None:
            return ()
        if isinstance(render, str):
            render = (render,)
        unknown = set(render) - set(RENDER_KEYS)
        if unknown:
            raise ValueError(f"render: unknown maps {sorted(unknown)}; choose from {RENDER_KEYS}")
        keys = tuple(k for k in RENDER_KEYS if k in render)
        if keys and to_2d:
            raise ValueError("render needs to_2d=False: the renderer takes the projected vertices with their depth")
        return keys

    @staticmethod
    def _frame_render_keys(frame_render, to_2d: bool, boxes) -> Tuple[str, ...]:
        """``frame_render`` as a canonical tuple (the order of FRAME_RENDER_KEYS), validated against ``to_2d`` and ``boxes``."""
        if frame_render is None:
            return ()
        if isinstance(frame_render, str):
            frame_render = (frame_render,)
        unknown = set(frame_render) - set(FRAME_RENDER_KEYS)
        if unknown:
            raise ValueError(f"frame_render: unknown maps {sorted(unknown)}; choose from {FRAME_RENDER_KEYS}")
        keys = tuple(k for k in FRAME_RENDER_KEYS if k in frame_render)
        if keys and boxes is None:
            raise ValueError("frame_render needs boxes: it draws the heads of each box into its frame")
        if keys and to_2d:
            raise ValueError("frame_render needs to_2d=False: the renderer takes the projected vertices with their depth")
        return keys

    def _pncc_renderer(self) -> PnccRenderer:
        if self._renderer is None:                           # uploads its tables once (graph-capture safe afterwards)
            self._renderer = PnccRenderer(self.device)
        return self._renderer

    def _lit(self) -> LitRenderer:
        if self._lit_renderer is None:                       # the reference's default lighting; tables uploaded once
            self._lit_renderer = LitRenderer(self.device)
        return self._lit_renderer

    def _check_rois(self, frames, boxes, frame_index) -> Tuple[Tensor, Optional[Tensor]]:
        """Validates the frames + boxes arguments before anything is launched -> (boxes, frame_index) as tensors."""
        if not (isinstance(frames, Tensor) and frames.dtype == torch.uint8 and frames.ndim == 4 and frames.shape[3] == 3):
            raise ValueError("frames: one [F,H,W,3] uint8 tensor")
        if min(frames.shape[:3]) < 1:
            raise ValueError(f"frames: empty shape {tuple(frames.shape)}")
        ints = (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)
        boxes = torch.as_tensor(boxes)
        if boxes.dtype not in ints or boxes.ndim != 2 or boxes.shape[1] != 4:
            raise ValueError(f"boxes: an [R,4] integer tensor of [x, y, w, h], got {boxes.dtype} {tuple(boxes.shape)}")
        R = int(boxes.shape[0])
        if R > MAX_ROIS:
            raise ValueError(f"boxes: at most {MAX_ROIS} per call, got {R}")
        if frame_index is not None:
            frame_index = torch.as_tensor(frame_index)
            if frame_index.dtype not in ints or tuple(frame_index.shape) != (R,):
                raise ValueError(f"frame_index: an [R] integer tensor, got {frame_index.dtype} {tuple(frame_index.shape)}")
            F = int(frames.shape[0])
            if frame_index.device.type == "cpu" and R and (int(frame_index.min()) < 0 or int(frame_index.max()) >= F):
                raise ValueError(f"frame_index: values must lie in [0, {F})")
        c = self.flame_constants
        if c["scale"] != 1 or c["translation"] != 3:
            raise ValueError("boxes need the released 3DMM layout (one scale, three translation parameters)")
        return boxes, frame_index

    def _predict_rois(self, frames, boxes, frame_index, extend, landmark_subset, to_2d, fast_decode,
                      frame_render=()) -> Dict[str, Tensor]:
        """predict_batch with boxes: crop geometry, pre-processing and read-back in csrc/roi.cu, no host synchronisation."""
        boxes, frame_index = self._check_rois(frames, boxes, frame_index)
        ext = np.array(extend_sides(extend), dtype=np.float64)
        frames = frames.to(self.device, non_blocking=True).contiguous()
        boxes = boxes.to(self.device, torch.int32, non_blocking=True).contiguous()
        if frame_index is not None:
            frame_index = frame_index.to(self.device, torch.int32, non_blocking=True).contiguous()
        c = self.flame_constants
        lib = _lib.load()
        S = self._img_size
        F, H, W = (int(d) for d in frames.shape[:3])
        R = int(boxes.shape[0])
        mean = (np.array(_MEAN, dtype=np.float32) * 255.0).astype(np.float32)
        inv = np.reciprocal(np.array(_STD, dtype=np.float32) * 255.0, dtype=np.float32)
        rois = torch.empty(R, ROI_RECORD_BYTES, dtype=torch.uint8, device=self.device)
        x = torch.empty(R, 3, S, S, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check(lib.dad3d_roi_setup(boxes.data_ptr(), frame_index.data_ptr() if frame_index is not None else None, R,
                                           F, H, W, S, ext.ctypes.data, rois.data_ptr(), stream), "dad3d_roi_setup")
            _lib.check(lib.dad3d_preprocess_rois(frames.data_ptr(), H, W, rois.data_ptr(), R, S, mean.ctypes.data,
                                                 inv.ctypes.data, x.data_ptr(), stream), "dad3d_preprocess_rois")
            raw, lms, _ = self.model.forward_raw(x, want_heatmap=False)
            params = torch.empty_like(raw)
            points = torch.empty(R, lms.shape[1], 2, dtype=torch.int64, device=self.device)
            _lib.check(lib.dad3d_readjust_rois(raw.data_ptr(), lms.data_ptr(), rois.data_ptr(), R, raw.shape[1],
                                               lms.shape[1], self.find_3dmm_idx("scale", c),
                                               self.find_3dmm_idx("translation", c), S, params.data_ptr(),
                                               points.data_ptr(), stream), "dad3d_readjust_rois")
        v3, proj = self.head_mesh.decode(params, to_2d=to_2d, hilo=not fast_decode)
        fields = rois.view(torch.int32)                       # x, y, w, h, frame, valid, ... (dad3d_roi)
        out = {"3dmm_params": params, "points": points, "3d_vertices": v3, "projected_vertices": proj,
               "crop_boxes": fields[:, :4].contiguous(), "valid": fields[:, 5] != 0}
        if landmark_subset is not None:
            dec = self.head_mesh.flame.decoder(self.device)
            out[f"landmarks_{landmark_subset}"] = dec.gather(proj, self._landmark_index(landmark_subset))
        if frame_render:
            frame_of_head = torch.where(out["valid"], fields[:, 4], -1)            # invalid boxes draw nothing
            if set(frame_render) - {"lit"}:
                maps = self._pncc_renderer().render_frames(proj, frame_of_head, F, (H, W), pncc="pncc" in frame_render,
                                                           depth="depth" in frame_render,
                                                           tri_index="tri_index" in frame_render,
                                                           head_index="head_index" in frame_render)
                out.update({f"frame_{k}": t for k, t in maps.items()})
            if "lit" in frame_render:
                out["frame_lit"] = self._lit().render_frames(proj, frame_of_head, F, (H, W), frames=frames)["lit"]
        return out

    def predict_batch(self, images: Tensor, landmark_subset: Optional[str] = "445", to_2d: bool = True,
                      fast_decode: bool = True, render=None, boxes=None, frame_index=None,
                      extend=0.0, frame_render=None) -> Dict[str, Tensor]:
        """images: [B,3,256,256] fp32 already letter-boxed + normalised, or raw RGB as the reference's ``__call__`` takes it:
        one [B,H,W,3] uint8 tensor / a list of HxWx3 uint8 images (letter-boxed + normalised on the GPU, bit-identical to
        the reference's albumentations pipeline); host or device.  All outputs stay on the GPU:
        "3dmm_params" [B,413], "points" [B,68,2] (pixels of the 256x256 network input), "3d_vertices" [B,5023,3],
        "projected_vertices" [B,5023,2|3], "landmarks_<subset>" [B,L,2|3].

        ``render``: a subset of ("pncc", "depth", "tri_index", "lit") (needs ``to_2d=False``) adds those maps of every
        head, drawn by :class:`~dad_3dheads_b200.rasterizer.PnccRenderer` from "projected_vertices" at the network input
        size, in the frame of "points": "pncc" [B,S,S,3] uint8, "depth" [B,S,S] fp32, "tri_index" [B,S,S] int32; "lit"
        [B,S,S,3] uint8 is the reference's ``RenderPipeline()`` shaded head on black, with its default lighting
        (:class:`~dad_3dheads_b200.rasterizer.LitRenderer`; other lights: a LitRenderer on "projected_vertices").

        ``boxes``: heads in whole frames.  ``images`` is then one [F,H,W,3] uint8 tensor of frames and ``boxes`` an [R,4]
        integer tensor of head boxes [x, y, w, h] in frame pixels (host or device), on frame ``frame_index[r]`` ([R]
        integers; None: every box is on frame 0).  Each box is cropped as the reference's data pipeline does,
        ``ensure_bbox_boundaries(extend_bbox(box, extend), (H, W))`` (``extend``: a fraction, (width, height) or
        (left, right, top, bottom)), and each crop gives what ``__call__`` gives on it, moved into frame pixels:
        "3dmm_params" readjusted to the frame (translation z = 0), "points" [R,68,2] int64 frame pixels, and
        "projected_vertices" / "landmarks_<subset>" decoded from those parameters; plus "crop_boxes" [R,4] int32 and
        "valid" [R] bool.  A box is invalid when its frame index is out of range, its crop is empty, or a side of its
        letter-box rounds to 0 pixels; its outputs are finite but meaningless.  Nothing waits for the device, so boxes
        computed on the GPU are consumed directly.  At most 65 535 boxes per call; ``render`` is not supported.

        ``frame_render`` (with ``boxes`` and ``to_2d=False``): a subset of ("pncc", "depth", "tri_index", "head_index") adds
        those maps of every whole frame, all its valid boxes' heads drawn from "projected_vertices" into one image and one
        z-buffer (:meth:`~dad_3dheads_b200.rasterizer.PnccRenderer.render_frames`): "frame_pncc" [F,H,W,3] uint8,
        "frame_depth" [F,H,W] fp32 (-z; -1e8 for background), "frame_tri_index" [F,H,W] int32 (the triangle within its
        head) and "frame_head_index" [F,H,W] int32 (the box), -1 for background; "frame_lit" [F,H,W,3] uint8, the heads
        shaded by the reference's default ``RenderPipeline()`` drawn over the frames (it takes ``bg``): each head lit on
        its own, then composited with one z-buffer per frame by the same rule (:meth:`LitRenderer.render_frames
        <dad_3dheads_b200.rasterizer.LitRenderer.render_frames>`; not a loop of RenderPipeline calls, whose fresh depth
        buffers would let a later box paint over a nearer earlier one).  A frame's PNCC maps equal the reference's
        ``PNCCEstimator()(frame, {"3dmm_params": p})`` run for its boxes' frame-space parameters one after the other in box
        order on the same buffers: the nearest head wins, an exact depth tie goes to the earlier box, invalid boxes draw
        nothing.  The reference's ``with_background=True`` overlay is, exactly,
        ``torch.where(out["frame_head_index"][..., None] >= 0, out["frame_pncc"], frames)``."""
        render = self._render_keys(render, to_2d)
        frame_render = self._frame_render_keys(frame_render, to_2d, boxes)
        if boxes is not None:
            if render:
                raise ValueError("render is not supported together with boxes")
            return self._predict_rois(images, boxes, frame_index, extend, landmark_subset, to_2d, fast_decode,
                                      frame_render)
        if isinstance(images, (list, tuple)) or (isinstance(images, Tensor) and images.dtype == torch.uint8):
            x = self.preprocess_batch(images)
        else:
            x = images.to(self.device, torch.float32, non_blocking=True)
        params, lms, _ = self.model.forward_raw(x, want_heatmap=False)
        v3, proj = self.head_mesh.decode(params, to_2d=to_2d, hilo=not fast_decode)
        out = {"3dmm_params": params, "points": lms * float(self._img_size), "3d_vertices": v3,
               "projected_vertices": proj}
        if landmark_subset is not None:
            dec = self.head_mesh.flame.decoder(self.device)
            out[f"landmarks_{landmark_subset}"] = dec.gather(proj, self._landmark_index(landmark_subset))
        if set(render) - {"lit"}:
            out.update(self._pncc_renderer()(proj, self._img_size, pncc="pncc" in render, depth="depth" in render,
                                      tri_index="tri_index" in render))
        if "lit" in render:
            out.update(self._lit()(proj, self._img_size))
        return out

    def _ws_generation(self):
        """Changes whenever the encoder or decoder scratch buffer is reallocated (captured graphs bake in its address)."""
        dec = self.head_mesh.flame.decoder(self.device)
        return (self.model.ws_generation, dec.ws_generation)

    def _capture(self, static_in: Tensor, landmark_subset, to_2d, fast_decode, render=None, rois=None, frame_render=()):
        """Warm up (plans, workspaces, tensor maps, index tables) and capture predict_batch(static_in) into a CUDA graph.
        ``rois`` = (static boxes [R,4] int32, static frame index [R] int32, extend): the graph reads the boxes from those
        buffers on every replay."""
        kw = dict(boxes=rois[0], frame_index=rois[1], extend=rois[2], frame_render=frame_render) if rois is not None else {}
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):
                self.predict_batch(static_in, landmark_subset, to_2d, fast_decode, render, **kw)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = self.predict_batch(static_in, landmark_subset, to_2d, fast_decode, render, **kw)
        return graph, out, self._ws_generation()

    def _roi_buffers(self, R: int, extend):
        """Static boxes / frame index buffers of a captured step with R boxes (zero boxes: every ROI invalid until filled)."""
        return (torch.zeros(R, 4, dtype=torch.int32, device=self.device),
                torch.zeros(R, dtype=torch.int32, device=self.device), extend_sides(extend))

    @staticmethod
    def _fill_rois(rois, boxes: Tensor, frame_index: Optional[Tensor]) -> None:
        rois[0].copy_(boxes, non_blocking=True)
        if frame_index is None:
            rois[1].zero_()
        else:
            rois[1].copy_(frame_index, non_blocking=True)

    def predict_batch_graphed(self, images: Tensor, landmark_subset: Optional[str] = "445", to_2d: bool = True,
                              fast_decode: bool = True, render=None, boxes=None, frame_index=None,
                              extend=0.0, frame_render=None) -> Dict[str, Tensor]:
        """:meth:`predict_batch` replayed from a CUDA graph (one graph per input shape / dtype / option set): the ~110 kernel
        launches of a step become one graph launch, which removes the launch gaps between the many sub-20 us layers.
        ``images`` is copied into the graph's static input buffer (host or device source); the returned tensors are the
        graph's static outputs -- consume or clone them before the next call with the same signature.

        A captured graph holds raw pointers into the encoder / decoder scratch buffers.  Those buffers only ever grow; when a
        later call (a larger batch, eager or graphed) reallocates one, every graph captured against the old buffer is
        re-captured before it is replayed again (``_ws_generation``), so a stale pointer is never dereferenced.

        With ``boxes`` (see :meth:`predict_batch`) the boxes and frame indices are copied into static buffers as well: one
        graph serves every box set of the same frame shape, box count, ``extend`` and ``frame_render``."""
        assert isinstance(images, Tensor), "the graphed path takes one tensor ([B,3,S,S] fp32 or [B,H,W,3] uint8)"
        render = self._render_keys(render, to_2d)
        frame_render = self._frame_render_keys(frame_render, to_2d, boxes)
        key = (tuple(images.shape), images.dtype, landmark_subset, to_2d, fast_decode, render, frame_render)
        if boxes is not None:
            if render:
                raise ValueError("render is not supported together with boxes")
            boxes, frame_index = self._check_rois(images, boxes, frame_index)
            key += (int(boxes.shape[0]), extend_sides(extend))
        ent = self._graphs.get(key)
        if ent is not None and ent[3] != self._ws_generation():
            ent = None                                        # scratch moved since the capture: never replay it
            self._graphs.pop(key)
        if ent is None:
            static_in = torch.empty(images.shape, dtype=images.dtype, device=self.device)
            static_in.copy_(images, non_blocking=True)
            rois = self._roi_buffers(int(boxes.shape[0]), extend) if boxes is not None else None
            if rois is not None:
                self._fill_rois(rois, boxes, frame_index)
            graph, out, gen = self._capture(static_in, landmark_subset, to_2d, fast_decode, render, rois, frame_render)
            ent = (graph, static_in, out, gen, rois)
            self._graphs[key] = ent
        graph, static_in, out, _, rois = ent
        static_in.copy_(images, non_blocking=True)
        if rois is not None:
            self._fill_rois(rois, boxes, frame_index)
        graph.replay()
        return out

    def open_stream(self, shape, dtype=torch.uint8, **kw) -> "BatchStream":
        """A double-buffered pipeline over :meth:`predict_batch` for a fixed batch signature -- see :class:`BatchStream`.
        ``rois=R`` (with optional ``extend`` and ``frame_render``): ``shape`` is that of the frames, and every submit brings R
        boxes."""
        return BatchStream(self, shape, dtype, **kw)


class BatchStream:
    """Software pipeline around the graph replay of ``FaceMeshPredictor.predict_batch`` for one batch signature.

    ``submit(images)`` enqueues, without blocking the host: the H2D copy of the (pinned) host batch on a copy stream, the
    graph replay on the compute stream, the optional all-gather over ``group`` on a communication stream and the D2H copy of
    the requested outputs into pinned host buffers on a fourth stream.  ``collect()`` blocks until the OLDEST submitted batch
    has landed and returns its results.  With ``depth`` slots (default 2) the copies and the collective of batch i overlap
    the encoder of batch i+1, so steady-state throughput is the compute time alone.  Results stay valid until ``depth`` more
    batches have been submitted.  ``render`` is passed to ``predict_batch`` (with ``to_2d=False``); list the maps in
    ``keys`` to have them copied to the host like the other outputs.  With ``rois=R`` each batch is frames plus R boxes
    (``predict_batch``'s ``boxes``): ``submit(frames, boxes=, frame_index=)`` copies the boxes on the copy stream together with
    the frames; "crop_boxes" and "valid" may be listed in ``keys``, and with ``frame_render`` (passed to ``predict_batch``)
    the "frame_<map>" outputs too.
    """

    def __init__(self, predictor: FaceMeshPredictor, shape, dtype=torch.uint8, landmark_subset: Optional[str] = "445",
                 to_2d: bool = True, fast_decode: bool = True, depth: int = 2, render=None,
                 keys=("3dmm_params", "points", "3d_vertices", "landmarks_445"), host_results: bool = True,
                 group=None, gather_keys=("3dmm_params", "3d_vertices", "landmarks_445"), comm=None, rois=None,
                 extend=0.0, frame_render=None):
        self.pred = predictor
        dev = predictor.device
        self.device = dev
        self.depth = int(depth)
        self.keys = tuple(keys)
        self.host_results = host_results
        self.group = group
        self.c_comm = comm                   # optional distributed.Dad3dComm: the gathers then run through the C ABI's NCCL calls
        self.gather_keys = tuple(gather_keys) if group is not None else ()
        self.compute = torch.cuda.Stream(dev)
        self.copy_in = torch.cuda.Stream(dev)
        self.copy_out = torch.cuda.Stream(dev)
        self.comm = torch.cuda.Stream(dev) if group is not None else None
        self._args = (landmark_subset, to_2d, fast_decode, predictor._render_keys(render, to_2d))
        if rois is not None and self._args[3]:
            raise ValueError("render is not supported together with boxes")
        self._frame_render = predictor._frame_render_keys(frame_render, to_2d, rois)
        self.rois = rois
        self.slots = []
        with torch.cuda.device(dev):
            for _ in range(self.depth):
                static_in = torch.zeros(tuple(shape), dtype=dtype, device=dev)
                roi_bufs = predictor._roi_buffers(int(rois), extend) if rois is not None else None
                graph, out, gen = predictor._capture(static_in, *self._args, roi_bufs, self._frame_render)
                slot = {"in": static_in, "rois": roi_bufs, "graph": graph, "out": out, "gen": gen, "busy": False,
                        "h2d": torch.cuda.Event(), "done": torch.cuda.Event(), "comm_done": torch.cuda.Event(),
                        "d2h": torch.cuda.Event(), "gathered": {}, "host": {}}
                if host_results:
                    for k in self.keys:
                        slot["host"][k] = torch.empty(out[k].shape, dtype=out[k].dtype).pin_memory()
                if group is not None:
                    import torch.distributed as dist
                    world = dist.get_world_size(group)
                    for k in self.gather_keys:
                        t = out[k]
                        slot["gathered"][k] = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype,
                                                          device=dev)
                self.slots.append(slot)
            torch.cuda.synchronize(dev)
        self._head = 0          # next slot to submit into
        self._tail = 0          # oldest uncollected
        self._inflight = 0

    def submit(self, images: Tensor, boxes=None, frame_index=None) -> None:
        if self._inflight == self.depth:
            raise RuntimeError("BatchStream: all slots in flight -- collect() before submitting more")
        if (boxes is None) != (self.rois is None):
            raise ValueError("boxes are required exactly when the stream was opened with rois=")
        if boxes is not None:
            boxes, frame_index = self.pred._check_rois(images, boxes, frame_index)
            if int(boxes.shape[0]) != self.rois:
                raise ValueError(f"boxes: this stream takes {self.rois} per batch, got {int(boxes.shape[0])}")
        s = self.slots[self._head]
        if s["gen"] != self.pred._ws_generation():           # scratch reallocated by another caller: re-capture this slot
            torch.cuda.synchronize(self.device)
            s["graph"], s["out"], s["gen"] = self.pred._capture(s["in"], *self._args, s["rois"], self._frame_render)
        with torch.cuda.stream(self.copy_in):
            self.copy_in.wait_event(s["done"])               # the previous replay of this slot has consumed its input
            s["in"].copy_(images, non_blocking=True)
            if boxes is not None:
                self.pred._fill_rois(s["rois"], boxes, frame_index)
            s["h2d"].record(self.copy_in)
        with torch.cuda.stream(self.compute):
            self.compute.wait_event(s["h2d"])
            self.compute.wait_event(s["d2h"])                # its previous results have left the device buffers
            if self.comm is not None:
                self.compute.wait_event(s["comm_done"])
            s["graph"].replay()
            s["done"].record(self.compute)
        last = s["done"]
        if self.comm is not None:
            import torch.distributed as dist
            with torch.cuda.stream(self.comm):
                self.comm.wait_event(s["done"])
                for k in self.gather_keys:
                    if self.c_comm is not None:
                        self.c_comm.all_gather(s["out"][k], s["gathered"][k])
                    else:
                        dist.all_gather_into_tensor(s["gathered"][k], s["out"][k], group=self.group)
                s["comm_done"].record(self.comm)
            last = s["comm_done"]
        with torch.cuda.stream(self.copy_out):
            self.copy_out.wait_event(last)
            if self.host_results:
                for k in self.keys:
                    s["host"][k].copy_(s["out"][k], non_blocking=True)
            s["d2h"].record(self.copy_out)
        s["busy"] = True
        self._head = (self._head + 1) % self.depth
        self._inflight += 1

    def collect(self) -> Dict[str, Tensor]:
        """Results of the oldest in-flight batch: pinned host tensors (``host_results``) or the slot's device outputs;
        gathered tensors (when a group was given) under ``"gathered"``."""
        if self._inflight == 0:
            raise RuntimeError("BatchStream: nothing in flight")
        s = self.slots[self._tail]
        s["d2h"].synchronize()
        s["busy"] = False
        self._tail = (self._tail + 1) % self.depth
        self._inflight -= 1
        res = dict(s["host"]) if self.host_results else {k: s["out"][k] for k in self.keys}
        if s["gathered"]:
            res["gathered"] = s["gathered"]
        return res

    def drain(self) -> None:
        while self._inflight:
            self.collect()
