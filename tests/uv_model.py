"""Exact numpy model of csrc/uv_texture.cu (TEST INFRASTRUCTURE): the fp64 vertex normals' z and the texel gather, in the
kernels' operation order.  numpy's float64 element-wise operations round once each and are never contracted, so the model
equals the kernels bit for bit and -- by the same order -- the reference's ``_compute_texture_map`` on tests/psbody_mesh.py's ``Mesh``."""
import numpy as np


def vertex_normals_z(v, faces, row, col):
    """v [V,3] fp32/fp64, faces [NF,3], CSR (row [V+1], col [nnz]) of each vertex's distinct faces ascending -> [V] fp64:
    z of (sum over the row of m * cross(v1 - v0, v2 - v0)) / norm, m = how often the face lists the vertex, the sum from
    +0 in row order, norm = sqrt((x^2 + y^2) + z^2) and 1 where that is 0."""
    v = np.asarray(v, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    a, b = p1 - p0, p2 - p0
    n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                  a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)
    V = v.shape[0]
    row = np.asarray(row, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    deg = row[1:] - row[:-1]
    s = np.zeros((V, 3))
    verts = np.arange(V)
    for k in range(int(deg.max(initial=0))):
        has = deg > k
        e = row[:-1][has] + k
        fc = col[e]
        m = (f[fc] == verts[has, None]).sum(1).astype(np.float64)
        s[has] = s[has] + m[:, None] * n[fc]
    norm = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2])
    norm[norm == 0] = 1.0
    return s[:, 2] / norm


def texture(v, nz, frame, texel, vids, bary, img_size):
    """One head: v [V,3], nz [V] (vertex_normals_z), frame [H,W,3] uint8 and the compacted table -> [S,S,3] uint8."""
    v = np.asarray(v, dtype=np.float64)
    a, b, c = vids[:, 0], vids[:, 1], vids[:, 2]
    b0, b1, b2 = bary[:, 0], bary[:, 1], bary[:, 2]
    n_dot_view = -((nz[a] * b0 + nz[b] * b1) + nz[c] * b2)
    px = (v[a, 0] * b0 + v[b, 0] * b1) + v[c, 0] * b2
    py = (v[a, 1] * b0 + v[b, 1] * b1) + v[c, 1] * b2
    x, y = np.rint(px), np.rint(py)
    H, W = frame.shape[:2]
    with np.errstate(invalid="ignore"):
        keep = ~(n_dot_view < 0) & (x > 0) & (x < W) & (y > 0) & (y < H)
    out = np.zeros((img_size * img_size, 3), dtype=np.uint8)
    out[texel[keep]] = frame[y[keep].astype(np.int64), x[keep].astype(np.int64)]
    return out.reshape(img_size, img_size, 3)


def textures(vertices, frames, frame_index, valid, faces, row, col, texel, vids, bary, img_size):
    """The kernels' [R,S,S,3] output: heads that are not valid or whose frame index is outside [0, F) are all zero."""
    R = vertices.shape[0]
    F = frames.shape[0]
    out = np.zeros((R, img_size, img_size, 3), dtype=np.uint8)
    for r in range(R):
        fi = 0 if frame_index is None else int(frame_index[r])
        if (valid is not None and not valid[r]) or not (0 <= fi < F):
            continue
        nz = vertex_normals_z(vertices[r], faces, row, col)
        out[r] = texture(vertices[r], nz, frames[fi], texel, vids, bary, img_size)
    return out


# ------------------------------------------------------------------------------------------------ shared test inputs
def reference_table_path():
    """The reference's texture_data.npy (its source tree, or the byte-compiled twin's data copy), or None."""
    import os
    from oracle import ref_harness as R
    root = R.root()
    p = None if root is None else os.path.join(root, "inference", "texture_data.npy")
    return p if p is not None and os.path.isfile(p) else None


def reference_texture_map(frame, vertices, faces, table):
    """The reference's own ``UVTextureCreator._compute_texture_map(frame, Mesh(vertices, faces))`` (uv_texture.py:21-47,
    run live through oracle/ref_harness on tests/psbody_mesh.py's ``Mesh``), with ``table`` the dict of texture_data.npy."""
    from oracle import ref_harness as R
    R.activate()
    from inference.uv_texture import UVTextureCreator
    from tests.psbody_mesh import Mesh
    creator = UVTextureCreator.__new__(UVTextureCreator)            # __init__ would also load generic_model.pkl
    creator.texture_data = table
    return creator._compute_texture_map(frame, Mesh(vertices, faces))


def flame_heads(n, seed=0):
    """[n,5023,3] fp32: FLAME heads decoded by the oracle at sampled parameters, projected to_2d=False (256-px frame)."""
    from oracle.flame_oracle import FlameOracle, sample_params
    p = sample_params(n, seed=seed)
    return FlameOracle().reprojected_vertices(p, to_2d=False).numpy().astype(np.float32)


def yawed(v, degrees):
    """v [V,3] rotated about the vertical axis through its centroid, in fp64, rounded to fp32."""
    v = np.asarray(v, dtype=np.float64)
    c = v.mean(0)
    t = np.deg2rad(degrees)
    rot = np.array([[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]])
    return ((v - c) @ rot.T + c).astype(np.float32)


def rough(v, seed=0):
    """v [V,3] fp32 with per-vertex noise whose scale spans 1e-3 .. 1e4.  The face normals of a plain fp32 head are exact
    in fp64 and so are most of their sums, whatever the order; these are not, so the sum order shows in the normals."""
    g = np.random.default_rng(seed)
    scale = (10.0 ** g.integers(0, 8, (v.shape[0], 1))).astype(np.float32)
    return v + g.standard_normal(v.shape).astype(np.float32) * np.float32(1e-3) * scale


def designed_heads(faces, seed=0, fp64=False):
    """{name: (vertices [5023,3] fp32, frame [H,W,3] uint8)} for the edge cases of the texel kernel; ``fp64`` adds
    "huge_fp64", an fp64 head with vertices at +-1e300."""
    rng = np.random.default_rng(seed)
    base = flame_heads(3, seed)
    frame = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)   # noqa: E731
    out = {"frontal": (base[0], frame(256, 256)),
           "rough_normals": (rough(base[0], seed), frame(256, 256)),
           "yaw_plus_85": (yawed(base[1], 85.0), frame(256, 256)),
           "yaw_minus_88": (yawed(base[2], -88.0), frame(240, 270)),
           "facing_away": (yawed(base[0], 180.0), frame(256, 256))}
    v = base[1].copy()
    v[:, 0] += 120.0
    out["partly_off_image"] = (v, frame(256, 256))
    v = base[2].copy()
    v[:, :2] -= v[:, :2].mean(0) - 2.0                                  # straddles row 0 and column 0
    out["straddles_0"] = (v, frame(200, 190))
    v = base[0].copy()
    v[:, 0] += 190.0 - v[:, 0].mean()                                   # straddles columns W-1 / W and rows H-1 / H
    v[:, 1] += 150.0 - v[:, 1].mean()
    out["straddles_W_H"] = (v, frame(161, 197))
    v = base[1].copy()
    v[:, :2] = np.round(v[:, :2] * 2.0) / 2.0                           # half-integer grid: exact .5 ties
    out["half_ties"] = (v, frame(256, 256))
    v = base[2].copy()
    v[faces[100, 0]] = np.nan
    v[faces[2000, 1], 0] = np.inf
    v[faces[3000, 2], 1] = -np.inf
    v[faces[4000, 0], 0] = np.float32(3e38)                             # the kernel's fp32 input: near its largest magnitude
    v[faces[5000, 1], 1] = -np.float32(3e38)
    v[faces[6000, 2], 2] = np.float32(3e38)
    out["nonfinite"] = (v, frame(256, 256))
    if fp64:                                                            # the reference's Mesh.v is fp64: magnitudes fp32 lacks
        v = base[0].astype(np.float64)
        v[faces[500, 0], 0] = 1e300
        v[faces[1500, 1], 1] = -1e300
        v[faces[2500, 2], 2] = 1e300
        v[faces[3500, 0], 0] = -1e300
        out["huge_fp64"] = (v, frame(256, 256))
    out["frame_1x1"] = (base[0] * np.float32(0.01), frame(1, 1))
    return out
