"""-m "not gpu": tests/lit_model.py against the reference's own, unmodified RenderPipeline (Sim3DR/lighting.py,
byte-compiled into oracle/_ref by oracle/lighting_ref.py, over the reference's C++ normals and rasteriser).  With the
host's np.power the model is the reference bit for bit; with the correctly rounded power (what the device computes) it
differs only where np.power is not correctly rounded, which is counted and bounded here."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import lighting_ref
from tests import lit_model as LM

F = np.float32
needs_ref = pytest.mark.skipif(not lighting_ref.available(), reason="oracle/_ref lighting.pyc / libsim3dr_ref.so not built")
HOST_POW = lambda a, e: a ** e                                         # noqa: E731 -- what lighting.py:59 evaluates


def same_bits(a, b) -> bool:
    """Equal bit for bit, except that any NaN equals any NaN (the payload of a NaN is not part of the contract)."""
    a, b = np.asarray(a, F), np.asarray(b, F)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


def reference_light(v, t, texture=None, **kw):
    """(light the reference's rasterize receives, its image) for RenderPipeline(**kw)(v, t, bg, texture)."""
    mod = lighting_ref.load()
    seen = {}
    orig = mod.rasterize

    def spy(vertices, triangles, colors, bg=None, **k):
        seen["colors"] = np.array(colors, copy=True)
        return orig(vertices, triangles, colors, bg=bg, **k)
    mod.rasterize = spy
    try:
        bg = np.zeros((64, 64, 3), np.uint8)
        img = mod.RenderPipeline(**kw)(v, t, bg, texture)
    finally:
        mod.rasterize = orig
    return seen["colors"], img


def demo_head():
    """The demo image's head as the oracle decodes it (tests/golden/reference_predictor.npz), z negated: what the
    predictor renders; it lands at x 213-379, y 451-600 of a 640 x 420 image."""
    import os
    import torch
    from oracle.flame_oracle import FlameOracle, load_static
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_predictor.npz"))
    p = torch.from_numpy(z["params_3dmm"]).double()
    v = FlameOracle(load_static(), image_size=256).reprojected_vertices(p, to_2d=False)[0].numpy().astype(F)
    v[:, 2] *= -1
    return np.ascontiguousarray(v)


def pncc_faces():
    from dad_3dheads_b200.rasterizer import load_render_static
    return load_render_static()["faces_wo_ears"]


def designed_meshes():
    """name -> (vertices [nv,3] float32, triangles, lighting kwargs)."""
    g = np.random.default_rng(5)
    # a bumpy 6 x 6 grid: front- and back-facing vertices, plus an unused vertex and a zero-area triangle (normal 1e-6)
    xs, ys = np.meshgrid(np.arange(6, dtype=F) * 9 + 3, np.arange(6, dtype=F) * 9 + 3)
    z = g.uniform(-8, 8, xs.shape).astype(F)
    grid = np.c_[xs.reshape(-1), ys.reshape(-1), z.reshape(-1)].astype(F)
    tris = []
    for r in range(5):
        for c in range(5):
            a = r * 6 + c
            tris += [[a, a + 1, a + 6], [a + 1, a + 7, a + 6]] if (r + c) % 3 else [[a, a + 6, a + 1], [a + 1, a + 6, a + 7]]
    grid = np.r_[grid, [[30, 30, 0], [10, 10, 1]]].astype(F)          # 36: unused; 37: only in a zero-area triangle
    tris += [[37, 37, 37]]
    tris = np.array(tris, np.int32)
    # a flat square (normals +z, vn_z = 0): a light in its plane gives cos == 0 exactly, a light behind gives cos < 0
    flat = np.array([[2, 2, 4], [40, 2, 4], [2, 40, 4], [40, 40, 4]], F)
    ft = np.array([[0, 1, 2], [1, 3, 2]], np.int32)
    vn = flat.copy()
    vn -= vn.min(0)
    vn /= vn.max()
    vn *= 2
    vn -= vn.max(0) / 2
    return {
        "grid_default": (grid, tris, {}),
        "grid_custom": (grid, tris, dict(intensity_ambient=0.25, intensity_directional=0.7, intensity_specular=0.35,
                                         specular_exp=3, color_ambient=(0.9, 0.8, 1.0), color_directional=(1.0, 0.7, 0.5),
                                         light_pos=(1, 2, 3), view_pos=(-1, 0.5, 4))),
        "grid_exp0": (grid, tris, dict(specular_exp=0, intensity_specular=0.5)),
        "grid_exp16": (grid, tris, dict(specular_exp=16, intensity_specular=0.9)),
        "grid_no_ambient": (grid, tris, dict(intensity_ambient=0)),
        "grid_no_directional": (grid, tris, dict(intensity_directional=0)),
        "grid_no_specular": (grid, tris, dict(intensity_specular=0.0)),
        "flat_cos_zero": (flat, ft, dict(light_pos=(5, 0, 0))),
        "flat_back_facing": (flat, ft, dict(light_pos=(0, 0, -5), intensity_specular=0.8)),
        "flat_nan_norm": (flat, ft, dict(light_pos=tuple(float(x) for x in vn[0]))),       # light on vertex 0: 0 / 0
    }


def test_sum_order_is_left_to_right():
    """np.sum(axis=1) over 3 float32 columns adds left to right on this numpy: lit_model relies on it."""
    g = np.random.default_rng(0)
    a = (g.standard_normal((200_000, 3)) * np.exp(g.uniform(-20, 20, (200_000, 3)))).astype(F)
    b = g.standard_normal((200_000, 3)).astype(F)
    for x in (a * b, a ** 2, a):
        assert same_bits(np.sum(x, axis=1), (x[:, 0] + x[:, 1]) + x[:, 2])


def _fraction_round(r: Fraction) -> float:
    """Nearest float32 to the rational r by comparing it with float32 neighbours, ties to an even significand."""
    guess = F(float(r)) if abs(r) < Fraction(2) ** 130 else F(math.copysign(math.inf, r))
    best = None
    for c in (np.nextafter(guess, F(-np.inf)), guess, np.nextafter(guess, F(np.inf))):
        if not np.isfinite(c):
            continue
        d = abs(Fraction(float(c)) - r)
        key = (d, int(np.asarray(c, F).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return float(best[1])


def test_exact_power_against_fractions():
    g = np.random.default_rng(1)
    xs = np.r_[g.uniform(-1, 1, 400), g.uniform(-3, 3, 200), np.exp(g.uniform(-12, 3, 100)) * g.choice([-1, 1], 100),
               [1 + 2 ** -12, -(1 + 2 ** -12), 1 + 2 ** -8, 1.5, 0.5, -0.75, 3 * 2 ** -20, 2 ** -9]].astype(F)
    for e in range(17):
        got = LM.exact_pow(xs, e)
        for x, y in zip(xs, got):
            want = 1.0 if e == 0 else _fraction_round(Fraction(float(x)) ** e)
            assert float(y) == want and math.copysign(1, float(y)) == math.copysign(1, want), (float(x), e, float(y), want)
    # exact midpoints: (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 lies halfway between two floats and goes to the even one
    assert float(LM.exact_pow(np.array([1 + 2 ** -12], F), 2)[0]) == 1 + 2 ** -11
    # (1 + 3*2^-12)^2 = 1 + 6*2^-12 + 2^-21 + 2^-24: again a midpoint, and the even neighbour is the lower one
    assert float(LM.exact_pow(np.array([1 + 3 * 2 ** -12], F), 2)[0]) == 1 + 6 * 2 ** -12 + 2 ** -21
    # (1 + 2^-12 + 2^-23)^2 = 1 + 4098.5005 * 2^-23: just above a midpoint, rounds up
    assert float(LM.exact_pow(np.array([1 + 2 ** -12 + 2 ** -23], F), 2)[0]) == 1 + 4099 * 2 ** -23
    # near midpoints: the inputs whose exact fifth power lies closest to a midpoint, rounded both ways correctly
    x = g.uniform(0.5, 1, 50_000).astype(F)
    dist = []
    for v in x[:3000]:
        r = Fraction(float(v)) ** 5
        lo = Fraction(float(_fraction_round(r)))
        ulp = Fraction(float(np.spacing(F(float(lo)))))
        dist.append(abs(abs(r - lo) / ulp - Fraction(1, 2)))
    near = x[:3000][np.argsort([float(d) for d in dist])[:20]]
    for v in near:
        assert float(LM.exact_pow(np.array([v], F), 5)[0]) == _fraction_round(Fraction(float(v)) ** 5)
    # special values follow the plain product
    sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], F)
    for e in (1, 2, 5):
        assert same_bits(LM.exact_pow(sp, e), np.array([s ** e for s in sp], F))


def test_host_power_mismatches_are_at_most_one_ulp():
    """How far the host's float32 x ** 5 is from correctly rounded: the only difference allowed between the device's light
    and the live reference's."""
    x = np.random.default_rng(2).uniform(-1, 1, 20_000).astype(F)
    host, exact = HOST_POW(x, 5), LM.exact_pow(x, 5)
    ulps = np.abs(host.astype(np.float64) - exact.astype(np.float64)) / np.spacing(np.abs(exact)).astype(np.float64)
    print(f"host float32 x**5: {int((host != exact).sum())} of {x.size} not correctly rounded, max {ulps.max():.2f} ulp")
    assert ulps.max() <= 1.0


@needs_ref
def test_normals_equal_reference():
    mod = lighting_ref.load()
    for name, (v, t, _) in designed_meshes().items():
        assert same_bits(LM.vertex_normals(v, t), mod.get_normal(v, t)), name
    v, t = demo_head(), pncc_faces()
    assert same_bits(LM.vertex_normals(v, t), mod.get_normal(v, t))


@needs_ref
@pytest.mark.parametrize("name", sorted(designed_meshes()))
def test_model_equals_reference_on_designed_meshes(name):
    v, t, kw = designed_meshes()[name]
    want, _ = reference_light(v, t, **kw)
    got = LM.light(v, t, kw, pow=HOST_POW)
    assert same_bits(got, want), name
    if name == "flat_nan_norm":
        assert np.isnan(got[0]).all() and not np.isnan(got[1:]).any()
    if name == "flat_cos_zero":
        assert same_bits(got, np.full_like(got, F(0.3)))                   # no diffuse, no specular: ambient only
    if name == "flat_back_facing":
        assert (got == F(0.3)).all()


@needs_ref
@pytest.mark.parametrize("kw", [{}, dict(specular_exp=2, intensity_specular=0.4, light_pos=(0.3, -1, 4)),
                                dict(intensity_ambient=0.1, color_directional=(0.2, 0.9, 0.6), view_pos=(2, 2, 2))])
def test_model_equals_reference_on_the_demo_head(kw):
    v, t = demo_head(), np.ascontiguousarray(pncc_faces()[:, [0, 2, 1]])
    want, _ = reference_light(v, t, **kw)
    assert same_bits(LM.light(v, t, kw, pow=HOST_POW), want)
    exact = LM.light(v, t, kw)
    diff = exact != want
    print(f"demo head {kw}: {int(diff.any(1).sum())} of {len(v)} vertex lights differ with the correctly rounded power, "
          f"max {np.abs(exact - want).max():.3g}")
    assert np.abs(exact - want).max() <= 1e-6


@needs_ref
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_texture_path(dtype):
    """texture *= light in place, in the texture's dtype; the rasteriser receives the product."""
    v, t, _ = designed_meshes()["grid_default"]
    tex = np.random.default_rng(3).uniform(0, 1, v.shape).astype(dtype)
    before = tex.copy()
    seen, _ = reference_light(v, t, texture=tex)
    light = LM.light(v, t, pow=HOST_POW)
    assert tex.dtype == dtype and np.array_equal(tex, before * light)
    assert np.array_equal(seen, tex)


@needs_ref
def test_winding_of_the_default_faces():
    """The predictor renders -z: a reflection of the projected (rotated) model space, so FLAME's counter-clockwise faces
    turn clockwise and their normals face away from the light at +z.  With the winding reversed most covered pixels are
    drawn from vertices that face the light."""
    from tests import raster_model
    v = demo_head()
    ccw = np.ascontiguousarray(pncc_faces())
    frac = {}
    for name, t in (("ccw", ccw), ("reversed", np.ascontiguousarray(ccw[:, [0, 2, 1]]))):
        n = LM.vertex_normals(v, t)
        vn = v - v.min(0)
        vn = vn / vn.max() * F(2)
        vn = vn - vn.max(0) / F(2)
        d = np.array([[0, 0, 5]], F) - vn
        cos = ((n * d).sum(1))
        _, _, tri = raster_model.rasterize(v, t, None, 640, 420)
        verts = t[tri[tri >= 0]].reshape(-1)
        frac[name] = float((cos[verts] > 0).mean())
    print("share of covered pixels' vertices with cos > 0:", frac)
    assert frac["reversed"] > 0.8 > 0.2 > frac["ccw"]
