"""Host side of the DAD-3DNet encoder: weight folding (one time) and the ``model(x) -> dict`` callable the predictor uses.

The reference runs a TorchScript trace of ``FlameRegression`` (predictor.py:72,97-100; flame_regression.py:87-106).  Here the
same ``state_dict`` is folded (eval-mode BatchNorm into the preceding conv, BiFPN depthwise 1x1 scale into the pointwise
conv, fast-normalised fusion weights into scalars) and handed to libdad3d.so, which runs every layer on the GPU.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .encoder_weights import HEAD_OUT, STAGE_UNITS

OUTPUT_2D_LANDMARKS = "OUTPUT_2D_LANDMARKS"               # model_training/data/config.py:16
OUTPUT_LANDMARKS_HEATMAP = "OUTPUT_LANDMARKS_HEATMAP"     # :18
OUTPUT_3DMM_PARAMS = "OUTPUT_3DMM_PARAMS"                 # :21

BN_EPS_RESNET = 1e-5        # pytorchcv ConvBlock
BN_EPS_BIFPN = 4e-5         # bifpn.py:36,66
BIFPN_EPSILON = 1e-4        # bifpn.py:77

PRECISION_PIECES = {"fp32": 3, "bf16x3": 3, "bf16x2": 2, "bf16": 1, "fp16x2": 2, "fp16": 1}
PRECISION_FORMAT = {"fp32": 0, "bf16x3": 0, "bf16x2": 0, "bf16": 0, "fp16x2": 1, "fp16": 1}     # DAD3D_OPERAND_*


def _bn_scale_shift(sd, p, eps):
    g, b = sd[p + ".weight"].double(), sd[p + ".bias"].double()
    m, v = sd[p + ".running_mean"].double(), sd[p + ".running_var"].double()
    s = g / torch.sqrt(v + eps)
    return s, b - m * s


def _khwc(w: Tensor) -> np.ndarray:
    """[cout, cin, R, S] -> contiguous fp32 [cout, R, S, cin]."""
    return np.ascontiguousarray(w.permute(0, 2, 3, 1).to(torch.float32).numpy())


def fold_state_dict(sd: Dict[str, Tensor]) -> Tuple[List[Tuple[str, np.ndarray, np.ndarray]], np.ndarray]:
    """-> ([(layer name, weight [cout,R,S,cin] fp32, bias [cout] fp32)], bifpn fusion weights [2,20] fp32).
    Layer names are the ones include/dad3d.h documents."""
    sd = {k: v.detach().cpu() for k, v in sd.items()}
    layers: List[Tuple[str, np.ndarray, np.ndarray]] = []

    def add(name, w, b):
        layers.append((name, _khwc(w), np.ascontiguousarray(b.to(torch.float32).numpy())))

    def conv_bn(name, p):          # pytorchcv ConvBlock: conv (no bias) -> BN
        s, sh = _bn_scale_shift(sd, p + ".bn", BN_EPS_RESNET)
        add(name, sd[p + ".conv.weight"].double() * s[:, None, None, None], sh)

    conv_bn("stem", "encoder.model.init_block.conv")
    for si, nu in enumerate(STAGE_UNITS):
        for ui in range(nu):
            p = f"encoder.model.stage{si + 1}.unit{ui + 1}"
            n = f"s{si + 1}u{ui + 1}"
            conv_bn(n + "c1", p + ".body.conv1")
            conv_bn(n + "c2", p + ".body.conv2")
            if ui == 0:
                # projection shortcut fused into the last 1x1: out = relu([W3 | Wid] [y ; x] + b3 + bid)
                s3, sh3 = _bn_scale_shift(sd, p + ".body.conv3.bn", BN_EPS_RESNET)
                si_, shi = _bn_scale_shift(sd, p + ".identity_conv.bn", BN_EPS_RESNET)
                w3 = sd[p + ".body.conv3.conv.weight"].double() * s3[:, None, None, None]
                wi = sd[p + ".identity_conv.conv.weight"].double() * si_[:, None, None, None]
                add(n + "c3", torch.cat([w3, wi], dim=1), sh3 + shi)
            else:
                conv_bn(n + "c3", p + ".body.conv3")
    # lateral convs (plain 1x1 + bias, no activation).  P3's lateral feeds exactly one consumer -- the first block's p3_td
    # node, also a 1x1 -- so the two are composed on the host (fp64) and the 64x64x256 lateral map is never materialised
    lat3_w = sd["bifpn.p3.weight"].double()[:, :, 0, 0]
    lat3_b = sd["bifpn.p3.bias"].double()
    for lvl in (4, 5, 6):
        add(f"lat{lvl}", sd[f"bifpn.p{lvl}.weight"].double(), sd[f"bifpn.p{lvl}.bias"].double())
    s, sh = _bn_scale_shift(sd, "bifpn.p7.bn", BN_EPS_BIFPN)       # BiFPNConvBlock: conv(bias) -> BN -> ReLU
    add("lat7", sd["bifpn.p7.conv.weight"].double() * s[:, None, None, None],
        sd["bifpn.p7.conv.bias"].double() * s + sh)
    fusion_w = np.zeros((2, 20), np.float32)
    td_col = {"p6_td": 0, "p5_td": 1, "p4_td": 2, "p3_td": 3}                     # column of w1 each top-down node uses
    for li in range(2):
        fw = {}
        for key, off in (("w1", 0), ("w2", 8)):                                    # bifpn.py:105-108, in fp32 like torch
            w = torch.relu(sd[f"bifpn.bifpn.{li}.{key}"].float())
            w = w / torch.sum(w, dim=0) + BIFPN_EPSILON
            fusion_w[li, off:off + w.numel()] = w.reshape(-1).numpy()
            fw[key] = w.double()
        for node in ("p6_td", "p5_td", "p4_td", "p3_td", "p4_out", "p5_out", "p6_out", "p7_out"):
            p = f"bifpn.bifpn.{li}.{node}"
            s, sh = _bn_scale_shift(sd, p + ".bn", BN_EPS_BIFPN)
            dw = sd[p + ".depthwise.weight"].double().reshape(1, -1, 1, 1)         # per-input-channel scale
            wfull = sd[p + ".pointwise.weight"].double() * dw * s[:, None, None, None]
            name = f"b{li}_{node.replace('_', '')}"
            if node in td_col:
                # top-down node: node(w0*a + w1*up(b)) = relu(W(w0 a) + up(W(w1 b)) + shift) because a 1x1 conv commutes with
                # nearest up-sampling -> two GEMMs (the second at the lower resolution), no separate weighted-sum pass
                j = td_col[node]
                w_main = wfull * fw["w1"][0, j]
                if li == 0 and node == "p3_td":                  # W0' (Wl c2 + bl) = (W0' Wl) c2 + W0' bl
                    w2d = w_main[:, :, 0, 0]
                    add(name, (w2d @ lat3_w)[:, :, None, None], sh + w2d @ lat3_b)
                else:
                    add(name, w_main, sh)
                add(name + "_u", wfull * fw["w1"][1, j], torch.zeros_like(sh))
            else:
                add(name, wfull, sh)
    add("heat", sd["head.heatmap.weight"].double(), sd["head.heatmap.bias"].double())
    wf = sd["fusion_layer.conv1x1.weight"].double()                                # [1024, 1024+68+256, 1, 1]
    n_heat = sd["head.heatmap.weight"].shape[0]
    cx = wf.shape[0]
    wf_p = torch.zeros(wf.shape[0], cx + 128 + (wf.shape[1] - cx - n_heat), 1, 1, dtype=torch.float64)
    wf_p[:, :cx] = wf[:, :cx]
    wf_p[:, cx:cx + n_heat] = wf[:, cx:cx + n_heat]
    wf_p[:, cx + 128:] = wf[:, cx + n_heat:]
    add("fusion", wf_p, sd["fusion_layer.conv1x1.bias"].double())
    names = [n for n, _ in HEAD_OUT]
    w1 = torch.cat([sd[f"{n}.logit_image.0.weight"].double() for n in names], 0)   # [1536, 2048]
    b1 = torch.cat([sd[f"{n}.logit_image.0.bias"].double() for n in names], 0)
    add("mlp1", w1[:, :, None, None], b1)
    hid = sd[f"{names[0]}.logit_image.0.weight"].shape[0]
    nout = sum(o for _, o in HEAD_OUT)
    w2 = torch.zeros(nout, hid * len(names), dtype=torch.float64)
    b2 = torch.zeros(nout, dtype=torch.float64)
    r = 0
    for i, (n, o) in enumerate(HEAD_OUT):
        w2[r:r + o, i * hid:(i + 1) * hid] = sd[f"{n}.logit_image.3.weight"].double()
        b2[r:r + o] = sd[f"{n}.logit_image.3.bias"].double()
        r += o
    add("mlp2", w2[:, :, None, None], b2)
    return layers, fusion_w


class _ConvWeights(C.Structure):
    _fields_ = [("name", C.c_char_p), ("weight_h", C.c_void_p), ("bias_h", C.c_void_p), ("cout", C.c_int32),
                ("cin", C.c_int32), ("R", C.c_int32), ("S", C.c_int32)]


class Dad3dEncoder:
    """``model(x: Tensor[B,3,256,256]) -> {OUTPUT_3DMM_PARAMS, OUTPUT_2D_LANDMARKS, OUTPUT_LANDMARKS_HEATMAP}`` on one GPU.

    precision: "fp32" (= "bf16x3": three-way bf16 split, 6 tensor-core products per tile, fp32-class accuracy -- the
    parity mode), "fp16x2" (fp16 hi/lo, 3 products, 22-bit operands, per-channel scaled weights), "bf16x2" (3 products,
    16-bit operands), "bf16" / "fp16" (one product, throughput modes).
    """

    def __init__(self, state_dict: Dict[str, Tensor], device: Optional[torch.device] = None, precision: str = "fp32",
                 want_heatmap: bool = True):
        self._setup(device, precision, want_heatmap)
        self._create(*fold_state_dict(state_dict))

    def _setup(self, device, precision, want_heatmap):
        if not torch.cuda.is_available():
            raise _lib.Dad3dError("dad_3dheads_b200 needs a CUDA (sm_90a) device: there is no CPU path")
        self.lib = _lib.load()
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise _lib.Dad3dError(f"Dad3dEncoder needs a cuda device, got {self.device}")
        self.precision = precision
        self.want_heatmap = want_heatmap

    @classmethod
    def from_folded(cls, layers: List[Tuple[str, np.ndarray, np.ndarray]], fusion_w: np.ndarray,
                    device: Optional[torch.device] = None, precision: str = "fp32", want_heatmap: bool = True):
        """An encoder over already folded layer records (the output format of :func:`fold_state_dict`), no BN folding:
        tests hand designed weights straight to dad3d_encoder_create."""
        enc = cls.__new__(cls)
        enc._setup(device, precision, want_heatmap)
        enc._create(layers, np.ascontiguousarray(fusion_w, dtype=np.float32))
        return enc

    def _create(self, layers, fusion_w):
        pieces, fmt = PRECISION_PIECES[self.precision], PRECISION_FORMAT[self.precision]
        layers = [(n, np.ascontiguousarray(w, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32))
                  for n, w, b in layers]
        recs = (_ConvWeights * len(layers))()
        keep = []
        for i, (name, w, b) in enumerate(layers):
            keep.append((name.encode(), w, b))
            recs[i].name = keep[-1][0]
            recs[i].weight_h = w.ctypes.data
            recs[i].bias_h = b.ctypes.data
            recs[i].cout, recs[i].R, recs[i].S, recs[i].cin = w.shape
        h = C.c_void_p()
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        _lib.check(self.lib.dad3d_encoder_create(C.byref(h), recs, len(layers), fusion_w.ctypes.data, pieces, fmt, idx),
                   "dad3d_encoder_create")
        self._h = h
        self._ws: Optional[Tensor] = None
        self.ws_generation = 0          # bumped whenever the scratch buffer is reallocated (CUDA graphs bake in its address)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self.lib.dad3d_encoder_destroy(h)
            except Exception:
                pass
            self._h = None

    def eval(self):
        return self

    # ---- live timing of the tile-engine launches (bench.py roofline)
    def set_profile(self, on: bool = True) -> None:
        _lib.check(self.lib.dad3d_encoder_set_profile(self._h, 1 if on else 0), "dad3d_encoder_set_profile")

    def profile_read(self):
        """-> (summed kernel ms, launches, algorithmic FLOPs) of the tile_gemm launches since the last read."""
        ms, n, fl = C.c_double(), C.c_longlong(), C.c_double()
        _lib.check(self.lib.dad3d_encoder_profile_read(self._h, C.byref(ms), C.byref(n), C.byref(fl)),
                   "dad3d_encoder_profile_read")
        return ms.value, n.value, fl.value

    def profile_layers(self):
        """Per-launch records of the current profiling window (call before :meth:`profile_read`): list of dicts with
        name, ms, flops (useful), bytes (algorithmic HBM), M, K, N, products, tiles, block_n, stages, k_blocks."""
        out = []
        name = C.create_string_buffer(64)
        ms, fl, by = C.c_double(), C.c_double(), C.c_double()
        info = (C.c_int32 * 8)()
        i = 0
        while self.lib.dad3d_encoder_profile_layer(self._h, i, name, 64, C.byref(ms), C.byref(fl), C.byref(by), info) == 0:
            out.append(dict(name=name.value.decode(), ms=ms.value, flops=fl.value, bytes=by.value, M=info[0], K=info[1],
                            N=info[2], products=info[3], tiles=info[4], block_n=info[5], stages=info[6], k_blocks=info[7]))
            i += 1
        return out

    # ---- test hooks (include/dad3d.h "test hooks")
    def set_debug(self, keep_all: bool = True) -> None:
        _lib.check(self.lib.dad3d_encoder_set_debug(self._h, 1 if keep_all else 0), "dad3d_encoder_set_debug")

    def read_activation(self, name: str) -> Tensor:
        """fp32 [N,H,W,C] copy of the activation produced by layer ``name`` in the last forward (needs set_debug(True))."""
        dims = (C.c_int32 * 4)()
        _lib.check(self.lib.dad3d_encoder_read_activation(self._h, name.encode(), None, 0, dims, None),
                   "dad3d_encoder_read_activation")
        out = torch.empty(tuple(int(d) for d in dims), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dad3d_encoder_read_activation(self._h, name.encode(), out.data_ptr(), out.numel(), dims,
                                                              torch.cuda.current_stream(self.device).cuda_stream),
                       "dad3d_encoder_read_activation")
        return out

    def describe_plan(self) -> dict:
        """The plan of the last forward: {"B", "pieces", "fp16", "num_sms", "steps": [per step: kind, layer, variant, the
        tensors it touches (in / in2 / in3 / res / out / out_f32 with name, N, H, W, C, planes, f32) and, for conv steps,
        the tile-engine geometry]}."""
        import json
        buf = C.create_string_buffer(1 << 20)
        _lib.check(self.lib.dad3d_encoder_describe_plan(self._h, buf, len(buf)), "dad3d_encoder_describe_plan")
        return json.loads(buf.value.decode())

    def write_activation(self, name: str, x: Tensor) -> None:
        """Overwrite activation ``name`` of the current plan with fp32 NHWC ``x`` (channels padded as stored), split into
        pieces by the library's own split."""
        x = x.to(self.device, torch.float32).contiguous()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dad3d_encoder_write_activation(self._h, name.encode(), x.data_ptr(), x.numel(),
                                                               torch.cuda.current_stream(self.device).cuda_stream),
                       "dad3d_encoder_write_activation")

    def run_steps(self, first: int, count: int = 1, images: Optional[Tensor] = None, params: Optional[Tensor] = None,
                  landmarks: Optional[Tensor] = None, heatmap: Optional[Tensor] = None) -> None:
        """Run steps [first, first + count) of the current plan, exactly as the forward runs them (``heatmap`` selects the
        heat-map variants as in the forward)."""
        ptr = lambda t: t.data_ptr() if t is not None else None     # noqa: E731
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dad3d_encoder_run_steps(self._h, first, count, ptr(images), ptr(params), ptr(landmarks),
                                                        ptr(heatmap), torch.cuda.current_stream(self.device).cuda_stream),
                       "dad3d_encoder_run_steps")

    def _workspace(self, B: int) -> Tensor:
        """The scratch buffer for a batch of B, grown (and ws_generation bumped) when the plan needs more."""
        need = int(self.lib.dad3d_encoder_workspace_bytes(self._h, B))
        if need == 0:
            _lib.check(-1, "dad3d_encoder_workspace_bytes")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            self.ws_generation += 1
        return self._ws

    def forward_raw(self, x: Tensor, want_heatmap: Optional[bool] = None):
        """x: [B,3,256,256] fp32 CUDA.  -> (params [B,413], landmarks [B,68,2], heatmap [B,68,64,64] | None)."""
        assert x.ndim == 4 and x.shape[1:] == (3, 256, 256), x.shape
        x = x.to(self.device, torch.float32).contiguous()
        B = x.shape[0]
        want_heatmap = self.want_heatmap if want_heatmap is None else want_heatmap
        params = torch.empty(B, 413, dtype=torch.float32, device=self.device)
        lms = torch.empty(B, 68, 2, dtype=torch.float32, device=self.device)
        heat = torch.empty(B, 68, 64, 64, dtype=torch.float32, device=self.device) if want_heatmap else None
        if B == 0:
            return params, lms, heat
        ws = self._workspace(B)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dad3d_encoder_forward(self._h, x.data_ptr(), B, params.data_ptr(), lms.data_ptr(),
                                                      heat.data_ptr() if heat is not None else None,
                                                      ws.data_ptr(), ws.numel(),
                                                      torch.cuda.current_stream(self.device).cuda_stream),
                       "dad3d_encoder_forward")
        return params, lms, heat

    def features(self, x: Tensor, want_heatmap: Optional[bool] = None):
        """x: [B,3,256,256] fp32 CUDA -> (features [B,2048], heatmap [B,68,64,64] | None): the pooled stage-4 map
        (F.adaptive_avg_pool2d(fmap, 1)) that the regression heads read, from the forward's steps up to the pool."""
        assert x.ndim == 4 and x.shape[1:] == (3, 256, 256), x.shape
        x = x.to(self.device, torch.float32).contiguous()
        B = x.shape[0]
        want_heatmap = self.want_heatmap if want_heatmap is None else want_heatmap
        feats = torch.empty(B, 2048, dtype=torch.float32, device=self.device)
        heat = torch.empty(B, 68, 64, 64, dtype=torch.float32, device=self.device) if want_heatmap else None
        if B == 0:
            return feats, heat
        ws = self._workspace(B)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dad3d_encoder_features(self._h, x.data_ptr(), B, feats.data_ptr(),
                                                       heat.data_ptr() if heat is not None else None,
                                                       ws.data_ptr(), ws.numel(),
                                                       torch.cuda.current_stream(self.device).cuda_stream),
                       "dad3d_encoder_features")
        return feats, heat

    def __call__(self, x: Tensor) -> Dict[str, Tensor]:
        params, lms, heat = self.forward_raw(x)
        out = {OUTPUT_3DMM_PARAMS: params, OUTPUT_2D_LANDMARKS: lms}
        if heat is not None:
            out[OUTPUT_LANDMARKS_HEATMAP] = heat
        return out
