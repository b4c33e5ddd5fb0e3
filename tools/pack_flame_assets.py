#!/usr/bin/env python
"""Pack the reference's static FLAME assets into one fp32 ``.npz`` the product path and the oracle both read.

Run in the build container (where /root/reference exists); the GPU box only sees the packed file.

What is read (reference data assets, not source):
  model_training/model/static/flame.pkl                      -> v_template, shapedirs, posedirs, J_regressor,
                                                               kintree_table, weights, f   (model/utils.py:84-89,
                                                               flame.py:124-180 say how the reference consumes them)
  model_training/model/static/indices_2d.npy                 -> indices_2d (flame.py:132)
  model_training/model/static/face_keypoints/keypoints_{191,445}/*.npy   (demo_utils.py:37-47, model_training/utils.py:81-105)
  model_training/model/static/flame_static_embedding.pkl, flame_dynamic_embedding.npy (data/utils.py:120-206)

and, into a second small text file ``render_static.json`` (read by ``rasterizer.load_render_static``), the two inputs of the
reference's PNCC renderer (inference/pncc_estimator.py:46-60,66-68):
  model_training/model/static/flame_indices/faces_wo_ears_remapped.npy  -> ``face_rows``: that file is FLAME's face list
  with the ear faces removed, in order, so it is stored as [start, stop) row ranges of ``faces`` in flame_static.npz
  ``ncc_colors`` [5023,3]: the template normalised to the unit cube over the vertices those faces use, computed in fp64 from
  the fp64 template of flame.pkl and rounded to fp32 once (as Sim3DR.rasterize does); from the packed fp32 template the
  last bits would differ.  Written as the shortest decimals that read back to the same fp32 values.

The pickle is python-2 era and references ``chumpy.ch.Ch`` + ``scipy.sparse.csc.csc_matrix``; chumpy is not installed, so
a restricted unpickler substitutes a stub for it (its array payload is attribute ``x``).
"""
import argparse
import io
import os
import pickle
import sys
import types

import numpy as np

REF = "/root/reference"
STATIC = "model_training/model/static"


class _ChStub:
    """Stand-in for chumpy.ch.Ch: keeps whatever state the pickle gives it; payload is ``x``."""

    def __setstate__(self, state):
        self.__dict__.update(state)


class _Unpickler(pickle.Unpickler):
    _ALLOWED_PREFIX = ("numpy", "scipy.sparse", "collections", "__builtin__", "builtins", "copy_reg", "copyreg")

    def find_class(self, module, name):
        if module.startswith("chumpy"):
            return _ChStub
        if module in ("scipy.sparse.csc", "scipy.sparse._csc") and name == "csc_matrix":
            import scipy.sparse
            return scipy.sparse.csc_matrix
        if module == "__builtin__":
            module = "builtins"
        if module == "copy_reg":
            module = "copyreg"
        if not module.startswith(self._ALLOWED_PREFIX):
            raise pickle.UnpicklingError(f"refusing to unpickle {module}.{name}")
        return super().find_class(module, name)


def _load_pickle(path):
    with open(path, "rb") as f:
        return _Unpickler(f, encoding="latin1").load()


def _np(x, dtype=None):
    if isinstance(x, _ChStub):
        x = x.x
    if hasattr(x, "todense"):
        x = np.asarray(x.todense())
    x = np.asarray(x)
    return x.astype(dtype) if dtype is not None else x


def _indices_from_npy(path):
    data = np.load(path, allow_pickle=True)[()]
    out = []
    for v in data.values():
        out += list(v)
    return out


def _keypoint_subset(dirpath, exclude=()):
    names = sorted(x[:-4] for x in os.listdir(dirpath) if x.endswith(".npy"))
    idx, per_file = [], {}
    for n in names:
        if n in exclude:
            continue
        cur = _indices_from_npy(os.path.join(dirpath, n + ".npy"))
        per_file[n] = len(cur)
        idx += cur
    return np.asarray(idx, dtype=np.int32), per_file


def ncc_color_codes(template: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """(template - lo) / (hi - lo) per axis, lo / hi the extent of the vertices ``faces`` uses with 0 included (the
    ``initial=0`` of pncc_estimator.py:53-54), in the template's own precision."""
    sub = template[np.unique(faces)]
    lo = sub.min(axis=0, keepdims=True, initial=0)
    hi = sub.max(axis=0, keepdims=True, initial=0)
    return (template - lo) / (hi - lo)


def face_row_ranges(faces: np.ndarray, subset: np.ndarray) -> list:
    """[start, stop) row ranges of ``faces`` whose concatenation is ``subset`` (which must be an ordered subset of rows)."""
    rows = {tuple(r): i for i, r in enumerate(faces.tolist())}
    idx = np.array([rows[tuple(r)] for r in subset.tolist()])
    if not np.all(np.diff(idx) > 0):
        raise ValueError("subset is not an ordered subset of the face rows")
    cut = np.flatnonzero(np.diff(idx) != 1) + 1
    return [[int(r[0]), int(r[-1]) + 1] for r in np.split(idx, cut)]


def pack_render_static(st: str, out_path: str) -> None:
    import json
    fl = _load_pickle(os.path.join(st, "flame.pkl"))
    template = _np(fl["v_template"], np.float64)
    flame_faces = _np(fl["f"]).astype(np.int32)
    faces = np.load(os.path.join(st, "flame_indices", "faces_wo_ears_remapped.npy")).astype(np.int32)
    ranges = face_row_ranges(flame_faces, faces)
    colors = ncc_color_codes(template, faces).astype(np.float32)
    dec = [[np.format_float_positional(x, unique=True, trim="-") for x in row] for row in colors]
    back = np.array([[float(x) for x in row] for row in dec], np.float32)
    assert np.array_equal(back.view(np.uint32), colors.view(np.uint32)), "decimal round trip"
    with open(out_path, "w") as f:
        f.write('{"face_rows": ' + json.dumps(ranges, separators=(",", ":")) + ',\n "ncc_colors": [\n')
        f.write(",\n".join("[" + ",".join(row) + "]" for row in dec))
        f.write("]}\n")
    print("wrote", os.path.abspath(out_path), os.path.getsize(out_path) / 1e3, "kB")


def main():
    assets = os.path.join(os.path.dirname(__file__), "..", "dad_3dheads_b200", "assets")
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF)
    ap.add_argument("--out", default=os.path.join(assets, "flame_static.npz"))
    ap.add_argument("--render-out", default=os.path.join(assets, "render_static.json"))
    ap.add_argument("--only", choices=("flame_static", "render_static"), default=None,
                    help="write one of the two files (default: both)")
    args = ap.parse_args()
    st = os.path.join(args.ref, STATIC)
    if args.only != "flame_static":
        pack_render_static(st, args.render_out)
    if args.only == "render_static":
        return

    fl = _load_pickle(os.path.join(st, "flame.pkl"))
    v_template = _np(fl["v_template"], np.float32)                      # [5023,3]
    shapedirs = _np(fl["shapedirs"], np.float32)                        # [5023,3,400]
    posedirs_raw = _np(fl["posedirs"], np.float64)                      # [5023,3,36]
    # flame.py:171-173: posedirs = reshape(posedirs, [-1, 36]).T -> [36, 15069]
    posedirs = np.reshape(posedirs_raw, [-1, posedirs_raw.shape[-1]]).T.astype(np.float32)
    j_regressor = _np(fl["J_regressor"], np.float32)                    # [5,5023]
    kintree = _np(fl["kintree_table"]).astype(np.int64)
    parents = kintree[0].copy()
    parents[0] = -1                                                      # flame.py:176-178
    weights = _np(fl["weights"], np.float32)                            # [5023,5]
    faces = _np(fl["f"]).astype(np.int32)                               # [9976,3]

    indices_2d = np.load(os.path.join(st, "indices_2d.npy")).astype(np.int32)
    kp191, files191 = _keypoint_subset(os.path.join(st, "face_keypoints", "keypoints_191"))
    kp445, files445 = _keypoint_subset(os.path.join(st, "face_keypoints", "keypoints_445"), exclude=("cheeks",))
    kp565, _ = _keypoint_subset(os.path.join(st, "face_keypoints", "keypoints_445"))

    stat = _load_pickle(os.path.join(st, "flame_static_embedding.pkl"))
    dyn = np.load(os.path.join(st, "flame_dynamic_embedding.npy"), allow_pickle=True, encoding="latin1")[()]
    static_face_idx = _np(stat["lmk_face_idx"]).astype(np.int32)         # [51]
    static_bcoords = _np(stat["lmk_b_coords"], np.float32)               # [51,3]
    dyn_face_idx = _np(dyn["lmk_face_idx"]).astype(np.int32)             # [79,17]
    dyn_bcoords = _np(dyn["lmk_b_coords"], np.float32)                   # [79,17,3]

    out = dict(
        v_template=v_template, shapedirs=shapedirs, posedirs=posedirs, J_regressor=j_regressor,
        parents=parents.astype(np.int32), lbs_weights=weights, faces=faces, indices_2d=indices_2d,
        keypoints_191=kp191, keypoints_445=kp445, keypoints_565=kp565,
        static_lmk_face_idx=static_face_idx, static_lmk_b_coords=static_bcoords,
        dynamic_lmk_face_idx=dyn_face_idx, dynamic_lmk_b_coords=dyn_bcoords,
    )
    for sub in ("head", "face", "face_w_ears", "eyeballs"):
        p = os.path.join(st, "flame_indices", sub + ".npy")
        if os.path.exists(p):
            out["flame_indices_" + sub] = np.load(p).astype(np.int32)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez(args.out, **out)
    for k, v in out.items():
        print(f"{k:28s} {str(v.dtype):8s} {v.shape}")
    print("191 files:", files191)
    print("445 files:", files445)
    print("indices_2d == keypoints_191:", bool(np.array_equal(indices_2d, kp191)))
    print("wrote", os.path.abspath(args.out), os.path.getsize(args.out) / 1e6, "MB")


if __name__ == "__main__":
    main()
