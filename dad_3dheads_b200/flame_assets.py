"""Readers of the reference's static FLAME assets (model_training/model/utils.py:80-89 ``get_flame_indices`` /
``get_flame_model``; flame.py:124-180 says how ``FLAMELayer.__init__`` consumes the pickle).

``flame.pkl`` is a python-2 era pickle that references ``chumpy.ch.Ch`` and ``scipy.sparse.csc.csc_matrix``; chumpy is not a
dependency of this package, so a restricted unpickler substitutes a stub for it (payload attribute ``x``) and refuses every
global outside a short whitelist (numpy array reconstruction, scipy csc_matrix, plain containers).  ``load_flame_pickle`` returns the same fp32 arrays the packed
``assets/flame_static.npz`` holds (tests/test_oracle_pinned.py checks the two bit for bit against the reference's own
FLAMELayer buffers), so ``FLAMELayer(consts, flame_path=".../flame.pkl")`` works at run time exactly like the reference's.
"""
from __future__ import annotations

import os
import pickle
from typing import Any, Dict, List, Optional, Tuple

import numpy as np


class _ChStub:
    """Stand-in for chumpy.ch.Ch: keeps whatever state the pickle gives it; the array payload is ``x``."""

    def __setstate__(self, state):
        self.__dict__.update(state)


class _RestrictedUnpickler(pickle.Unpickler):
    """Whitelist of exactly the globals FLAME-style pickles need (flame.pkl / generic_model.pkl of the reference:
    numpy.dtype, numpy.ndarray, numpy.core.multiarray._reconstruct, scipy.sparse csc_matrix, chumpy.ch.Ch, builtins set) plus
    the inert container / scalar types protocol-2 pickles of numpy data may name.  A module PREFIX is not enough: "builtins"
    also holds eval / exec / __import__, "numpy" holds load / fromfile -- everything else is refused."""

    _ALLOWED = {
        "builtins": {"set", "frozenset", "list", "dict", "tuple", "object", "slice", "range", "complex", "int", "float", "bool",
                     "str", "bytes", "bytearray"},
        "collections": {"OrderedDict", "defaultdict"},
        "copyreg": {"_reconstructor"},
        "_codecs": {"encode"},                      # how protocol-2 pickles written by python 3 carry numpy's raw bytes
        "numpy": {"dtype", "ndarray"},
        "numpy.core.multiarray": {"_reconstruct", "scalar"},
        "numpy._core.multiarray": {"_reconstruct", "scalar"},
        "numpy.core.numeric": {"_frombuffer"},
        "numpy._core.numeric": {"_frombuffer"},
    }

    def find_class(self, module, name):
        if module in ("chumpy.ch", "chumpy") and name == "Ch":
            return _ChStub
        if module in ("scipy.sparse.csc", "scipy.sparse._csc") and name == "csc_matrix":
            import scipy.sparse
            return scipy.sparse.csc_matrix
        module = {"__builtin__": "builtins", "copy_reg": "copyreg"}.get(module, module)
        if name not in self._ALLOWED.get(module, ()):
            raise pickle.UnpicklingError(f"refusing to unpickle {module}.{name}")
        return super().find_class(module, name)


def _np(x, dtype=None) -> np.ndarray:
    if isinstance(x, _ChStub):
        x = x.x
    if hasattr(x, "todense"):
        x = np.asarray(x.todense())
    x = np.asarray(x)
    return x.astype(dtype) if dtype is not None else x


def load_pickle(path: str):
    with open(path, "rb") as f:
        return _RestrictedUnpickler(f, encoding="latin1").load()


def load_flame_pickle(path: str) -> Dict[str, np.ndarray]:
    """flame.pkl -> {v_template [V,3], shapedirs [V,3,400], posedirs [36,3V], J_regressor [5,V], parents [5], lbs_weights
    [V,5], faces [F,3]} in fp32 / int32, with the reference's reshapes (flame.py:171-178)."""
    fl = load_pickle(path)
    posedirs_raw = _np(fl["posedirs"], np.float64)                       # [V,3,36]
    parents = _np(fl["kintree_table"]).astype(np.int64)[0].copy()
    parents[0] = -1                                                       # flame.py:176-178
    out = {
        "v_template": _np(fl["v_template"], np.float32),
        "shapedirs": _np(fl["shapedirs"], np.float32),
        "posedirs": np.reshape(posedirs_raw, [-1, posedirs_raw.shape[-1]]).T.astype(np.float32),   # flame.py:171-173
        "J_regressor": _np(fl["J_regressor"], np.float32),
        "parents": parents.astype(np.int32),
        "lbs_weights": _np(fl["weights"], np.float32),
        "faces": _np(fl["f"]).astype(np.int32),
    }
    here = os.path.dirname(os.path.abspath(path))
    idx = os.path.join(here, "indices_2d.npy")                           # flame.py:132 (get_flame_indices("indices_2d"))
    if os.path.isfile(idx):
        out["indices_2d"] = np.load(idx).astype(np.int32)
    return out


def load_indices_from_npy(filepath: str):
    """model_training/utils.py:99-105: an .npy holding an (ordered) dict of index lists -> their concatenation, in dict order."""
    groups = np.load(filepath, allow_pickle=True)[()]          # 0-d object array -> the dict it wraps
    return [i for indices in groups.values() for i in indices]


def get_list_of_npy_files(config: Dict) -> list:
    """model_training/utils.py:81-96.  ``2d_keys == "all"`` (the default): every file of ``2d_subset_path``, named by its stem,
    except the stems listed in ``2d_keys_exclude`` (a name or a list; default "cheeks"; None keeps everything), returned as
    ``<folder>/<stem>.npy``.  Any other ``2d_keys`` value is handed back unchanged, as the reference does."""
    folder = str(config.get("2d_subset_path"))
    keys = config.get("2d_keys", "all")
    entries = os.listdir(folder)                          # (the reference lists the folder before looking at the keys, too)
    if not (isinstance(keys, str) and keys == "all"):
        return keys
    dropped = config.get("2d_keys_exclude", "cheeks")
    dropped = [] if dropped is None else [dropped] if isinstance(dropped, str) else list(dropped)
    stems = [name.split(".")[0] for name in entries]
    for stem in dropped:
        if stem in stems:
            stems.remove(stem)                            # first occurrence only, like list.remove in the reference
    return [os.path.join(folder, stem + ".npy") for stem in stems]


def load_2d_indices(config: Dict) -> Optional[List[int]]:
    """model_training/utils.py:62-78: the 2D keypoint subset -- None for ``2d_subset_name == "multipie_keypoints"`` (the 68
    barycentric landmarks), else the index lists of ``get_list_of_npy_files`` concatenated over the SORTED file names."""
    if config["2d_subset_name"] == "multipie_keypoints":
        return None
    indices: List[int] = []
    for filename in sorted(get_list_of_npy_files(config)):
        if not os.path.exists(filename):
            raise ValueError(f"[{filename.split('.')[0].split('/')[-1]}] class of keypoints doesn't exist")
        indices += load_indices_from_npy(filename)
    return indices


def indices_reweighing(weights_and_indices: Dict[str, Any]) -> Tuple[List, List]:
    """model_training/utils.py:108-117: the (weight, index array) pairs of the loss subsets, in the order of the
    ``flame_indices.files`` mapping, for every file whose key has a weight."""
    weights_dict = weights_and_indices["weights"]
    weights, indices = [], []
    for key, value in weights_and_indices["flame_indices"]["files"].items():
        if key in weights_dict.keys():
            indices.append(np.load(os.path.join(weights_and_indices["flame_indices"]["folder"], value)))
            weights.append(weights_dict[key])
    return weights, indices


def load_static(path: Optional[str], default_npz: str) -> Dict[str, np.ndarray]:
    """``path`` None -> the packed npz; ``*.pkl`` -> the reference's pickle (landmark tables etc. are then taken from the packed
    npz, which holds everything else the path needs); anything else -> an npz in the packed format."""
    def npz(p):
        with np.load(p) as z:
            return {k: z[k] for k in z.files}
    def extras(st):
        # static/head_indices.npy (benchmark evaluator: get_flame_indices() default, dad_3dheads_benchmark/utils.py:310-311)
        # lives beside the packed npz as a small file of its own
        hp = os.path.join(os.path.dirname(default_npz), "head_indices.npy")
        if "head_indices" not in st and os.path.isfile(hp):
            st["head_indices"] = np.load(hp)
        return st
    if path is None:
        return extras(npz(default_npz))
    if str(path).endswith(".pkl"):
        st = extras(npz(default_npz)) if os.path.isfile(default_npz) else {}
        st.update(load_flame_pickle(path))
        return st
    return extras(npz(path))
