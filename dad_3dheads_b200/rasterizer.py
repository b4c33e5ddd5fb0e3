"""GPU drop-in for the reference's ``Sim3DR`` package (Sim3DR/Sim3DR.py:8-29): ``rasterize`` and ``get_normal`` with the same
signatures, numpy in / numpy out, bit-exact with the C++ rasteriser they wrap (csrc/rasterize.cu, SURVEY §8f row 4).  Used by
the reference's ``inference/pncc_estimator.py`` through ``compat/Sim3DR``.  No CPU fallback.

``rasterize_batch`` and ``PnccRenderer`` are the batched, device-resident form: B heads of one topology per call, device
tensors in and out, no host synchronisation (so they run inside a captured CUDA graph); every head equals, bit for bit, what
``rasterize`` gives for that head alone.  With a head -> image map (``rasterize_batch(image_of_head=, num_images=)``,
``PnccRenderer.render_frames``) several heads share one image and one z-buffer, as when a caller of the reference draws the
heads of a whole frame one after the other into the same buffers.

``light_batch`` and ``LitRenderer`` are the reference's ``Sim3DR.RenderPipeline`` (Sim3DR/lighting.py:23-71) in the same
batched form: per-vertex ambient, diffuse and specular light of every head, then the rasteriser with each head's light as
its colours."""
from __future__ import annotations

import os
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib


def _device(cuda_id: Optional[int]) -> torch.device:
    if not torch.cuda.is_available():
        raise _lib.Dad3dError("dad_3dheads_b200.rasterizer needs a CUDA (sm_90a) device: there is no CPU path")
    return torch.device("cuda", torch.cuda.current_device() if cuda_id is None else cuda_id)


def rasterize(vertices: np.ndarray, triangles: np.ndarray, colors: np.ndarray, bg: Optional[np.ndarray] = None,
              height: Optional[int] = None, width: Optional[int] = None, channel: Optional[int] = None, reverse: bool = False,
              cuda_id: Optional[int] = None) -> np.ndarray:
    """Sim3DR.rasterize: z-buffer rendering of per-vertex colours onto ``bg`` (modified in place and returned, like the
    reference) or onto a black ``height x width x channel`` image.  vertices [N,3] float32 (pixels, depth), triangles [M,3] int,
    colors [N,C] in [0,1]."""
    lib = _lib.load()
    dev = _device(cuda_id)
    if bg is not None:
        height, width, channel = bg.shape
    else:
        assert height is not None and width is not None and channel is not None
        bg = np.zeros((height, width, channel), dtype=np.uint8)
    assert bg.dtype == np.uint8
    with torch.cuda.device(dev):
        v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float32)).to(dev)
        t = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int32)).to(dev)
        c = torch.from_numpy(np.ascontiguousarray(colors, dtype=np.float32)).to(dev)
        assert c.shape[1] == channel and v.shape[1] == 3 and t.shape[1] == 3
        img = torch.from_numpy(np.ascontiguousarray(bg)).to(dev)
        depth = torch.full((height, width), -1e8, dtype=torch.float32, device=dev)      # Sim3DR.py:22
        key = torch.empty(height * width, dtype=torch.int64, device=dev)
        _lib.check(lib.dad3d_rasterize(v.data_ptr(), t.data_ptr(), c.data_ptr(), int(t.shape[0]), img.data_ptr(), depth.data_ptr(),
                                       key.data_ptr(), height, width, channel, 1 if reverse else 0,
                                       torch.cuda.current_stream(dev).cuda_stream), "dad3d_rasterize")
        out = img.cpu().numpy()
    np.copyto(bg, out)
    return bg


def vertex_adjacency(triangles: np.ndarray, nver: int):
    """CSR list of the triangles around every vertex, ascending (the order of the reference's accumulation loop)."""
    t = np.asarray(triangles, dtype=np.int64)
    vert = t.reshape(-1)
    tri = np.repeat(np.arange(t.shape[0], dtype=np.int64), 3)
    order = np.lexsort((tri, vert))                       # by vertex, then by triangle index
    counts = np.bincount(vert, minlength=nver)
    offsets = np.zeros(nver + 1, dtype=np.int32)
    offsets[1:] = np.cumsum(counts)
    return offsets, tri[order].astype(np.int32)


def get_normal(vertices: np.ndarray, triangles: np.ndarray, cuda_id: Optional[int] = None) -> np.ndarray:
    """Sim3DR.get_normal: per-vertex normals [N,3] float32."""
    lib = _lib.load()
    dev = _device(cuda_id)
    nver = int(vertices.shape[0])
    off, adj = vertex_adjacency(triangles, nver)
    with torch.cuda.device(dev):
        v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float32)).to(dev)
        t = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int32)).to(dev)
        o = torch.from_numpy(off).to(dev)
        a = torch.from_numpy(adj).to(dev)
        out = torch.empty(nver, 3, dtype=torch.float32, device=dev)
        _lib.check(lib.dad3d_vertex_normals(v.data_ptr(), t.data_ptr(), o.data_ptr(), a.data_ptr(), nver, out.data_ptr(),
                                            torch.cuda.current_stream(dev).cuda_stream), "dad3d_vertex_normals")
        return out.cpu().numpy()


def _check_triangles(triangles: torch.Tensor, nv: int) -> None:
    """Bounds-check the triangle indices against ``nv`` on the host, once per tensor and content version: the kernels index
    vertices through them unchecked.  The first call on a tensor reads it back (a synchronisation); later calls, e.g. inside
    a graph capture after the warm-up, do not."""
    tag = (nv, triangles._version)
    if getattr(triangles, "_dad3d_checked", None) == tag:
        return
    if triangles.numel():
        lo, hi = (int(x) for x in torch.aminmax(triangles))
        if lo < 0 or hi >= nv:
            raise ValueError(f"triangle indices span [{lo}, {hi}], outside the {nv} vertices")
    triangles._dad3d_checked = tag


def _image_map(image_of_head: Optional[torch.Tensor], num_images: Optional[int], B: int, ntri: int, dev):
    """Checks a head -> image map of B heads of ``ntri`` triangles -> (the number of output images, the map made
    contiguous); without a map, B images and None."""
    if (image_of_head is not None) != (num_images is not None):
        raise ValueError("image_of_head and num_images go together")
    if image_of_head is None:
        return B, None
    if image_of_head.shape != (B,) or image_of_head.dtype != torch.int32 or image_of_head.device != dev:
        raise ValueError(f"image_of_head must be a [{B}] int32 tensor on the vertices' device")
    n_out = int(num_images)
    if n_out < 0:
        raise ValueError(f"num_images must be >= 0, got {n_out}")
    if B * ntri > 2 ** 32 - 2:
        raise ValueError(f"{B} heads x {ntri} triangles exceed 2^32 - 2 (head, triangle) pairs")
    return n_out, image_of_head.contiguous()


def _output_image(image: Optional[torch.Tensor], n: int, height: int, width: int, c: int, dev) -> torch.Tensor:
    """The image the heads are drawn over: zeros, or a copy of ``image`` ([n,height,width,c] uint8) on ``dev``."""
    if image is None:
        return torch.zeros(n, height, width, c, dtype=torch.uint8, device=dev)
    if tuple(image.shape) != (n, height, width, c) or image.dtype != torch.uint8:
        raise ValueError(f"image must be [{n},{height},{width},{c}] uint8")
    return image.to(dev, copy=True).contiguous()


def rasterize_batch(vertices: torch.Tensor, triangles: torch.Tensor, colors: Optional[torch.Tensor] = None, *, height: int,
                    width: int, image: Optional[torch.Tensor] = None, depth: bool = True, tri_index: bool = True,
                    reverse: bool = False, negate_z: bool = False, image_of_head: Optional[torch.Tensor] = None,
                    num_images: Optional[int] = None, head_index: bool = True) -> Dict[str, torch.Tensor]:
    """Z-buffer rendering of B heads that share one mesh topology, on the GPU (``dad3d_rasterize_batch``).

    vertices [B,nv,3] float32 (x, y in pixels, z = depth, larger wins; with ``negate_z`` -z is the depth), triangles [ntri,3]
    int32, colors [nv,C] float32 in [0,1] or None (no image), all on one CUDA device.  Returns a dict of the requested maps:
    "image" [B,height,width,C] uint8 (when ``colors`` is given: zeros, or a copy of ``image``, with the heads drawn over it;
    ``reverse`` flips its rows), "depth" [B,height,width] float32 (-1e8 where no triangle covers the pixel), "tri_index"
    [B,height,width] int32 (the winning triangle, -1 for background, in depth-map rows).  Runs on the current stream without
    a host synchronisation, except the first bounds check of a ``triangles`` tensor.

    ``image_of_head`` ([B] int32 on the device) and ``num_images`` draw the heads into ``num_images`` shared images
    (``dad3d_rasterize_frames``): head b goes to image ``image_of_head[b]``, and a head mapped outside [0, num_images) draws
    nothing.  Every map is then [num_images, ...], and "head_index" [num_images,height,width] int32 names the winning head
    (-1 for background; ``head_index=False`` leaves it out).  Each image equals the reference's rasteriser run over its
    heads one after the other in head order with carried buffers: the nearest surface wins, and an exact depth tie goes to
    the lower (head, triangle) pair.  ``reverse`` is not available with a map."""
    if vertices.ndim != 3 or vertices.shape[2] != 3 or vertices.dtype != torch.float32 or not vertices.is_cuda:
        raise ValueError("vertices must be a [B,nv,3] float32 CUDA tensor")
    if triangles.ndim != 2 or triangles.shape[1] != 3 or triangles.dtype != torch.int32 or triangles.device != vertices.device:
        raise ValueError("triangles must be an [ntri,3] int32 tensor on the vertices' device")
    dev = vertices.device
    B, nv = int(vertices.shape[0]), int(vertices.shape[1])
    height, width = int(height), int(width)
    if nv == 0 or height <= 0 or width <= 0 or height * width >= 1 << 31:
        raise ValueError(f"bad shape: nv={nv}, height={height}, width={width}")
    mapped = image_of_head is not None
    n_out, image_of_head = _image_map(image_of_head, num_images, B, int(triangles.shape[0]), dev)
    if mapped and reverse:
        raise ValueError("reverse is not available with image_of_head")
    vertices = vertices.contiguous()
    triangles = triangles.contiguous()
    _check_triangles(triangles, nv)
    out: Dict[str, torch.Tensor] = {}
    c = 1
    if colors is not None:
        if colors.ndim != 2 or colors.shape[0] != nv or colors.dtype != torch.float32 or colors.device != dev:
            raise ValueError("colors must be an [nv,C] float32 tensor on the vertices' device")
        colors = colors.contiguous()
        c = int(colors.shape[1])
        out["image"] = _output_image(image, n_out, height, width, c, dev)
    elif image is not None:
        raise ValueError("image needs colors")
    if depth:
        out["depth"] = torch.full((n_out, height, width), -1e8, dtype=torch.float32, device=dev)     # Sim3DR.py:22
    if tri_index:
        out["tri_index"] = torch.empty(n_out, height, width, dtype=torch.int32, device=dev)
    if mapped and head_index:
        out["head_index"] = torch.empty(n_out, height, width, dtype=torch.int32, device=dev)
    key = torch.empty(n_out * height * width, dtype=torch.int64, device=dev)   # caching allocator: capture-safe
    ptr = lambda name: out[name].data_ptr() if name in out else None           # noqa: E731
    lib = _lib.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        cptr = colors.data_ptr() if colors is not None else None
        if mapped:
            _lib.check(lib.dad3d_rasterize_frames(vertices.data_ptr(), nv, B, triangles.data_ptr(), int(triangles.shape[0]),
                                                  cptr, c, image_of_head.data_ptr(), n_out, height, width,
                                                  1 if negate_z else 0, ptr("image"), ptr("depth"), ptr("tri_index"),
                                                  ptr("head_index"), key.data_ptr(), stream), "dad3d_rasterize_frames")
        else:
            _lib.check(lib.dad3d_rasterize_batch(vertices.data_ptr(), nv, B, triangles.data_ptr(), int(triangles.shape[0]),
                                                 cptr, c, height, width, 1 if reverse else 0, 1 if negate_z else 0,
                                                 ptr("image"), ptr("depth"), ptr("tri_index"), key.data_ptr(), stream),
                       "dad3d_rasterize_batch")
    return out


_RENDER_ASSET = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets", "render_static.json")


def load_render_static() -> Dict[str, np.ndarray]:
    """The reference's PNCC inputs (inference/pncc_estimator.py:66-68), packed by tools/pack_flame_assets.py:
    "faces_wo_ears" [6270,3] int32, FLAME's faces without the ears (stored as row ranges of the packed FLAME faces), and
    "ncc_colors" [5023,3] float32, the NCC colour of every template vertex."""
    import json
    from .flame import load_flame_static
    with open(_RENDER_ASSET) as f:
        d = json.load(f)
    faces = load_flame_static()["faces"]
    rows = np.concatenate([np.arange(a, b) for a, b in d["face_rows"]])
    return {"faces_wo_ears": np.ascontiguousarray(faces[rows], dtype=np.int32),
            "ncc_colors": np.asarray(d["ncc_colors"], dtype=np.float32)}


class PnccRenderer:
    """The reference's PNCC render (inference/pncc_estimator.py:16-43,66-93) for a batch of decoded heads: the FLAME
    template's normalised coordinates as colours over the faces without ears, z negated, on a black background.

    ``__call__(projected_vertices_3d, size)`` takes [B,5023,3] float32 on the device, as ``HeadMesh.decode(...,
    to_2d=False)`` / ``reprojected_vertices(..., to_2d=False)`` return it, and returns {"pncc": [B,S,S,3] uint8, "depth":
    [B,S,S] float32 (-z; -1e8 for background), "tri_index": [B,S,S] int32 (index into ``faces``, -1 for background)}.
    ``faces`` and ``colors`` (:func:`load_render_static`) are uploaded once."""

    def __init__(self, device=None):
        if not torch.cuda.is_available():
            raise _lib.Dad3dError("PnccRenderer needs a CUDA (sm_90a) device: there is no CPU path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        st = load_render_static()
        self.faces = torch.from_numpy(st["faces_wo_ears"]).to(self.device)
        self.colors = torch.from_numpy(st["ncc_colors"]).to(self.device)
        _check_triangles(self.faces, int(self.colors.shape[0]))

    def _render(self, projected_vertices_3d: torch.Tensor, size, pncc: bool, **kw) -> Dict[str, torch.Tensor]:
        """rasterize_batch of [B,nv,3] vertices at ``size`` = (H, W), z negated, with "image" named "pncc"."""
        if projected_vertices_3d.ndim != 3 or projected_vertices_3d.shape[1:] != (self.colors.shape[0], 3):
            raise ValueError(f"expected [B,{self.colors.shape[0]},3] vertices, got {tuple(projected_vertices_3d.shape)}")
        height, width = (int(v) for v in size)
        out = rasterize_batch(projected_vertices_3d, self.faces, self.colors if pncc else None, height=height, width=width,
                              negate_z=True, **kw)
        if pncc:
            out["pncc"] = out.pop("image")
        return out

    def __call__(self, projected_vertices_3d: torch.Tensor, size: int, *, pncc: bool = True, depth: bool = True,
                 tri_index: bool = True) -> Dict[str, torch.Tensor]:
        return self._render(projected_vertices_3d, (size, size), pncc, depth=depth, tri_index=tri_index)

    def render_frames(self, projected_vertices_3d: torch.Tensor, frame_of_head: torch.Tensor, num_frames: int, size, *,
                      pncc: bool = True, depth: bool = True, tri_index: bool = True,
                      head_index: bool = True) -> Dict[str, torch.Tensor]:
        """The frame form: B heads in the pixels of whole frames, drawn into ``num_frames`` frames of ``size`` = (H, W)
        with one z-buffer per frame.  ``frame_of_head`` [B] int32 on the device names each head's frame; a head whose entry
        is outside [0, num_frames) (e.g. -1 for an invalid box) draws nothing.  Returns {"pncc": [F,H,W,3] uint8, "depth":
        [F,H,W] float32 (-z; -1e8 for background), "tri_index": [F,H,W] int32 (index into ``faces`` of the winning head),
        "head_index": [F,H,W] int32 (the winning head)}, -1 for background in both index maps.

        A frame equals the reference's ``PNCCEstimator()(frame, {"3dmm_params": p}, with_background=False)``
        (inference/pncc_estimator.py:88-101) over its heads one after the other in head order, each drawing into the same
        image and depth buffer: the nearest surface wins across heads, and an exact depth tie goes to the lower head.  The
        reference's ``with_background=True`` overlay is ``torch.where(head_index[..., None] >= 0, pncc, frames)``, exactly,
        since alpha = 1 overwrites every covered pixel."""
        return self._render(projected_vertices_3d, size, pncc, depth=depth, tri_index=tri_index, image_of_head=frame_of_head,
                            num_images=num_frames, head_index=head_index)


# RenderPipeline's keyword arguments and defaults (Sim3DR/lighting.py:24-32)
LIGHTING_DEFAULTS = {"intensity_ambient": 0.3, "intensity_directional": 0.6, "intensity_specular": 0.1, "specular_exp": 5,
                     "color_ambient": (1, 1, 1), "color_directional": (1, 1, 1), "light_pos": (0, 0, 5),
                     "view_pos": (0, 0, 5)}
MAX_SPECULAR_EXP = 16


def lighting_struct(lighting: Optional[dict] = None) -> _lib.Lighting:
    """RenderPipeline keyword arguments (None or missing keys: the reference's defaults) -> the ``dad3d_lighting`` the
    kernel takes.  Intensities are scalars, colours and positions 3-sequences, all used as float32 as the reference's
    float32 arithmetic does; ``specular_exp`` must be an integer in [0, 16] (the device computes the correctly rounded power
    only for those).  Raises ValueError otherwise."""
    kw = dict(LIGHTING_DEFAULTS)
    unknown = set(lighting or {}) - set(kw)
    if unknown:
        raise ValueError(f"unknown lighting arguments {sorted(unknown)}; choose from {sorted(kw)}")
    kw.update(lighting or {})
    e = kw["specular_exp"]
    if isinstance(e, (bool, np.bool_)) or not isinstance(e, (int, np.integer)) or not 0 <= int(e) <= MAX_SPECULAR_EXP:
        raise ValueError(f"specular_exp must be an integer in [0, {MAX_SPECULAR_EXP}], got {e!r}")
    L = _lib.Lighting()
    for k in ("intensity_ambient", "intensity_directional", "intensity_specular"):
        x = float(kw[k])
        if x > 0 and np.float32(x) <= 0:       # the reference tests "> 0" before rounding to float32
            raise ValueError(f"{k}={x!r} is positive but rounds to 0 in float32")
        setattr(L, k, float(np.float32(x)))
    L.specular_exp = int(e)
    for k in ("color_ambient", "color_directional", "light_pos", "view_pos"):
        a = np.asarray(kw[k], dtype=np.float32).reshape(-1)
        if a.shape != (3,):
            raise ValueError(f"{k} must have 3 components, got {kw[k]!r}")
        getattr(L, k)[:] = [float(x) for x in a]
    return L


def _adjacency(triangles: torch.Tensor, nv: int):
    """The CSR vertex -> triangle lists of ``triangles`` on its device, built on the host once per tensor and content
    version (the first call synchronises; later calls, e.g. inside a capture after the warm-up, do not)."""
    tag = (nv, triangles._version)
    cached = getattr(triangles, "_dad3d_adj", None)
    if cached is not None and cached[0] == tag:
        return cached[1]
    off, adj = vertex_adjacency(triangles.cpu().numpy(), nv)
    pair = (torch.from_numpy(off).to(triangles.device), torch.from_numpy(adj).to(triangles.device))
    triangles._dad3d_adj = (tag, pair)
    return pair


def _check_mesh(vertices: torch.Tensor, triangles: torch.Tensor):
    if vertices.ndim != 3 or vertices.shape[2] != 3 or vertices.dtype != torch.float32 or not vertices.is_cuda:
        raise ValueError("vertices must be a [B,nv,3] float32 CUDA tensor")
    if triangles.ndim != 2 or triangles.shape[1] != 3 or triangles.dtype != torch.int32 or triangles.device != vertices.device:
        raise ValueError("triangles must be an [ntri,3] int32 tensor on the vertices' device")
    nv = int(vertices.shape[1])
    if nv == 0 or 3 * nv >= 1 << 31:
        raise ValueError(f"bad vertex count {nv}")
    triangles = triangles.contiguous()
    _check_triangles(triangles, nv)
    return vertices.contiguous(), triangles


def light_batch(vertices: torch.Tensor, triangles: torch.Tensor, *, lighting: Optional[dict] = None,
                negate_z: bool = False) -> torch.Tensor:
    """RenderPipeline's per-vertex ``light`` (Sim3DR/lighting.py:38-63) of B heads on the GPU (``dad3d_light_batch``).

    vertices [B,nv,3] float32 (with ``negate_z``, -z is used, as the predictor's renders do), triangles [ntri,3] int32 on
    the same device, ``lighting`` RenderPipeline's keyword arguments (:func:`lighting_struct`).  Returns [B,nv,3] float32 in
    [0,1] (NaN where the reference's arithmetic gives NaN).  Every head is lit on its own: norm_vertices uses that head's
    extent.  Every float32 operation is the reference's, in its order; (v2v * reflection) ** specular_exp is the correctly
    rounded power, which the reference's ``np.power`` misses by one ulp for some inputs.  No host synchronisation except
    the first use of a ``triangles`` tensor (bounds check and adjacency)."""
    L = lighting_struct(lighting)
    vertices, triangles = _check_mesh(vertices, triangles)
    B, nv = int(vertices.shape[0]), int(vertices.shape[1])
    off, adj = _adjacency(triangles, nv)
    out = torch.empty(B, nv, 3, dtype=torch.float32, device=vertices.device)
    lib = _lib.load()
    with torch.cuda.device(vertices.device):
        _lib.check(lib.dad3d_light_batch(vertices.data_ptr(), nv, B, triangles.data_ptr(), off.data_ptr(), adj.data_ptr(),
                                         1 if negate_z else 0, L, out.data_ptr(),
                                         torch.cuda.current_stream(vertices.device).cuda_stream), "dad3d_light_batch")
    return out


def render_lit(vertices: torch.Tensor, triangles: torch.Tensor, *, height: int, width: int, lighting: Optional[dict] = None,
               negate_z: bool = False, image: Optional[torch.Tensor] = None, image_of_head: Optional[torch.Tensor] = None,
               num_images: Optional[int] = None) -> torch.Tensor:
    """Lit render of B heads (``dad3d_render_lit``): :func:`light_batch`, then the z-buffer rasteriser with each head's light
    as its colours, alpha = 1.  Returns [N,height,width,3] uint8: zeros, or a copy of ``image`` ([N,height,width,3] uint8),
    with the heads drawn over it.  Without ``image_of_head`` N = B and image b is RenderPipeline()(head b, triangles, bg)
    exactly.  With ``image_of_head`` ([B] int32 on the device) and ``num_images`` = N, as :func:`rasterize_batch`: each head
    is lit on its own, then all heads of an image share one z-buffer, the nearest surface wins and an exact tie goes to the
    lower head; heads mapped outside [0, N) draw nothing.  That is the reference's ``_rasterize`` run once on the union mesh
    with the heads' lights as colours, NOT a loop of RenderPipeline calls (each call starts a fresh depth buffer, so a later
    head would paint over a nearer earlier one)."""
    L = lighting_struct(lighting)
    vertices, triangles = _check_mesh(vertices, triangles)
    dev = vertices.device
    B, nv, ntri = int(vertices.shape[0]), int(vertices.shape[1]), int(triangles.shape[0])
    height, width = int(height), int(width)
    if height <= 0 or width <= 0 or height * width >= 1 << 31:
        raise ValueError(f"bad image size {height} x {width}")
    n_out, image_of_head = _image_map(image_of_head, num_images, B, ntri, dev)
    out = _output_image(image, n_out, height, width, 3, dev)
    if B == 0 or n_out == 0:
        return out
    off, adj = _adjacency(triangles, nv)
    light = torch.empty(B * nv * 3, dtype=torch.float32, device=dev)            # caching allocator: capture-safe
    key = torch.empty(max(n_out, 1) * height * width, dtype=torch.int64, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        _lib.check(lib.dad3d_render_lit(vertices.data_ptr(), nv, B, triangles.data_ptr(), ntri, off.data_ptr(),
                                        adj.data_ptr(), 1 if negate_z else 0, L,
                                        image_of_head.data_ptr() if image_of_head is not None else None, n_out, height, width,
                                        light.data_ptr(), out.data_ptr(), key.data_ptr(),
                                        torch.cuda.current_stream(dev).cuda_stream), "dad3d_render_lit")
    return out


class LitRenderer:
    """The reference's ``RenderPipeline(**lighting)`` (Sim3DR/lighting.py:23-71) for a batch of decoded heads, drawn as
    the predictor's PNCC render draws them: z negated (a larger -z is nearer), on a black background.

    ``triangles`` None means the PNCC faces without ears with the winding reversed (``faces_wo_ears[:, [0, 2, 1]]``):
    negating z reflects the mesh, which reverses the orientation of FLAME's counter-clockwise faces, so their normals would
    face away from the light at +z (DESIGN §4.6).  Lighting keyword arguments as RenderPipeline's (:func:`lighting_struct`).
    Adjacency and tables are uploaded once, so both methods are safe inside a CUDA graph capture after one warm-up call;
    neither synchronises the host."""

    def __init__(self, device=None, triangles=None, **lighting):
        if not torch.cuda.is_available():
            raise _lib.Dad3dError("LitRenderer needs a CUDA (sm_90a) device: there is no CPU path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.lighting = dict(lighting)
        lighting_struct(self.lighting)                          # validate now, before any launch
        st = load_render_static()
        self.nv = int(st["ncc_colors"].shape[0])
        if triangles is None:
            triangles = st["faces_wo_ears"][:, [0, 2, 1]]
        self.faces = torch.as_tensor(np.ascontiguousarray(np.asarray(triangles), dtype=np.int32)).to(self.device)
        _check_triangles(self.faces, self.nv)
        _adjacency(self.faces, self.nv)

    def _check(self, v: torch.Tensor) -> None:
        if v.ndim != 3 or v.shape[1:] != (self.nv, 3):
            raise ValueError(f"expected [B,{self.nv},3] vertices, got {tuple(v.shape)}")

    def __call__(self, projected_vertices_3d: torch.Tensor, size: int) -> Dict[str, torch.Tensor]:
        """[B,5023,3] float32 on the device (``HeadMesh.decode(..., to_2d=False)``) -> {"lit": [B,S,S,3] uint8}, each head
        equal to ``RenderPipeline(**lighting)(v, triangles, zeros)`` with z negated."""
        self._check(projected_vertices_3d)
        return {"lit": render_lit(projected_vertices_3d, self.faces, height=size, width=size, lighting=self.lighting,
                                  negate_z=True)}

    def render_frames(self, projected_vertices_3d: torch.Tensor, frame_of_head: torch.Tensor, num_frames: int, size,
                      frames: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """B heads in frame pixels into ``num_frames`` frames of ``size`` = (H, W): {"lit": [F,H,W,3] uint8}, drawn over a
        copy of ``frames`` ([F,H,W,3] uint8) or over black.  ``frame_of_head`` [B] int32 on the device names each head's
        frame; entries outside [0, F) draw nothing.  Each head is lit by its own RenderPipeline, which normalises that
        head's vertices; then the heads of a frame share one z-buffer: the nearest surface wins and an exact depth tie goes
        to the earlier head, the rule of ``PnccRenderer.render_frames``.  This is the reference's ``_rasterize`` run once
        on the union mesh with the heads' lights as colours.  It is not a loop of RenderPipeline calls, where each call
        starts a fresh depth buffer and a later head paints over a nearer earlier one."""
        self._check(projected_vertices_3d)
        height, width = (int(v) for v in size)
        return {"lit": render_lit(projected_vertices_3d, self.faces, height=height, width=width, lighting=self.lighting,
                                  negate_z=True, image=frames, image_of_head=frame_of_head, num_images=num_frames)}
