"""``Sim3DR.lighting.RenderPipeline`` (reference: Sim3DR/lighting.py:23-71) on the GPU: numpy in, numpy out, with the
reference's side effects -- ``bg`` is drawn into in place and returned, and a ``texture`` is multiplied by the light in
place, in its own dtype, on the host, before it is rasterised.

The light is dad_3dheads_b200.rasterizer.light_batch: the reference's float32 arithmetic in its order, except that
(v2v * reflection) ** specular_exp is the correctly rounded power, so ``specular_exp`` must be an integer in [0, 16]
(ValueError otherwise).  Colours, positions and intensities are used as float32, as the reference uses its tuple
defaults."""
from __future__ import annotations

import numpy as np
import torch

from dad_3dheads_b200 import rasterizer as _r


class RenderPipeline(object):
    def __init__(self, **kwargs):
        self._kw = {k: kwargs.get(k, v) for k, v in _r.LIGHTING_DEFAULTS.items()}
        _r.lighting_struct(self._kw)

    def update_light_pos(self, light_pos):
        self._kw["light_pos"] = light_pos
        _r.lighting_struct(self._kw)

    def __getattr__(self, name):
        kw = self.__dict__.get("_kw", {})
        if name in kw:                                     # intensity_ambient, light_pos, ... as the reference stores them
            v = kw[name]
            return np.array(v, dtype=np.float32)[None, :] if isinstance(v, (tuple, list)) else v
        raise AttributeError(name)

    def __call__(self, vertices, triangles, bg, texture=None):
        dev = _r._device(None)
        v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float32)).to(dev)[None]
        t = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int32)).to(dev)
        if texture is None:
            img = torch.from_numpy(np.ascontiguousarray(bg)).to(dev)[None]
            h, w = bg.shape[:2]
            if bg.dtype != np.uint8 or bg.ndim != 3 or bg.shape[2] != 3:
                raise ValueError("bg must be an [H,W,3] uint8 image")
            out = _r.render_lit(v, t, height=h, width=w, lighting=self._kw, image=img)
            np.copyto(bg, out[0].cpu().numpy())
            return bg
        light = _r.light_batch(v, t, lighting=self._kw)[0].cpu().numpy()
        texture *= light
        return _r.rasterize(vertices, triangles, texture, bg=bg)
