"""-m "not gpu": host-side logic that needs no device -- the restricted unpickler behind ``FLAMELayer(flame_path=...)``
(model/utils.py:84-89 loads the same file with a plain ``pickle.load``), the FLAME index-file readers, the decode kernel's
row permutation."""
import io
import os
import pickle

import numpy as np
import pytest

from dad_3dheads_b200 import flame_assets as FA


class _Evil:
    def __reduce__(self):
        return (eval, ("__import__('os').getpid()",))


@pytest.mark.parametrize("payload", [
    pickle.dumps(_Evil(), protocol=2),                                        # builtins.eval through REDUCE
    b"cos\nsystem\n(S'true'\ntR.",                                           # os.system
    b"cnumpy\nload\n(S'/etc/passwd'\ntR.",                                  # a numpy function that opens files
    b"cbuiltins\n__import__\n(S'os'\ntR.",
    b"c__builtin__\nexec\n(S'pass'\ntR.",
    b"csubprocess\nPopen\n((S'true'\nttR.",
])
def test_restricted_unpickler_refuses_everything_but_array_data(payload):
    with pytest.raises(pickle.UnpicklingError):
        FA._RestrictedUnpickler(io.BytesIO(payload), encoding="latin1").load()


def test_restricted_unpickler_reads_numpy_scipy_and_chumpy_payloads(tmp_path):
    import scipy.sparse
    data = {"v": np.arange(12, dtype=np.float64).reshape(4, 3), "f": np.arange(6, dtype=np.uint32).reshape(2, 3),
            "J": scipy.sparse.csc_matrix(np.eye(3)), "s": {1, 2}, "name": "x", "n": 3, "t": (1.5, None)}
    for proto in (2, 4):
        p = tmp_path / f"a{proto}.pkl"
        p.write_bytes(pickle.dumps(data, protocol=proto))
        got = FA.load_pickle(str(p))
        assert np.array_equal(got["v"], data["v"]) and got["f"].dtype == np.uint32 and got["s"] == {1, 2}
        assert np.array_equal(FA._np(got["J"]), np.eye(3)) and got["t"] == (1.5, None)
    # a chumpy object: class chumpy.ch.Ch with its array in attribute x (what flame.pkl's posedirs / v_template are)
    ch = b"(dp0\nS'a'\np1\nccopy_reg\n_reconstructor\np2\n(cchumpy.ch\nCh\np3\nc__builtin__\nobject\np4\nNtp5\nRp6\n(dp7\nS'x'\np8\nI7\nsbs."
    got = FA._RestrictedUnpickler(io.BytesIO(ch), encoding="latin1").load()
    assert isinstance(got["a"], FA._ChStub) and got["a"].x == 7 and FA._np(got["a"]) == 7


def test_index_file_readers(tmp_path):
    """model_training/utils.py:81-105: ``get_list_of_npy_files`` (config dict; "all" = every file of the folder minus
    ``2d_keys_exclude``, default cheeks) and ``load_indices_from_npy`` (an .npy holding an ordered dict of index lists)."""
    import collections
    np.save(tmp_path / "face.npy", collections.OrderedDict(a=[3, 1], b=[2]), allow_pickle=True)
    np.save(tmp_path / "cheeks.npy", collections.OrderedDict(c=[9]), allow_pickle=True)
    np.save(tmp_path / "nose.npy", collections.OrderedDict(n=[5, 6]), allow_pickle=True)
    files = FA.get_list_of_npy_files({"2d_subset_path": str(tmp_path)})
    assert sorted(os.path.basename(f) for f in files) == ["face.npy", "nose.npy"]
    assert sorted(os.path.basename(f) for f in FA.get_list_of_npy_files({"2d_subset_path": str(tmp_path), "2d_keys_exclude": None})) == \
        ["cheeks.npy", "face.npy", "nose.npy"]
    assert FA.get_list_of_npy_files({"2d_subset_path": str(tmp_path), "2d_keys": ["x.npy"]}) == ["x.npy"]   # explicit lists pass through
    assert FA.load_indices_from_npy(str(tmp_path / "face.npy")) == [3, 1, 2]


def test_decode_row_permutation_is_a_bijection_with_equal_residues_per_warp():
    """flame_decode.cuh ``dec_phys_row`` / ``dec_head_of`` (restated): physical coefficient row of head h inside its 256-head
    block = 128 t + 32 wq + l with residue h mod 8 = 4 t + wq, l = (h mod 256) / 8 -- every accumulator row quarter of a row tile holds
    32 heads that are equal mod 8 (the premise of the per-lane sector-aligned stores)."""
    def phys(h):
        return (h & ~255) + ((h & 7) >> 2) * 128 + (h & 3) * 32 + ((h & 255) >> 3)

    def head_of(m_tile, wq, lane):
        return (m_tile >> 1) * 256 + lane * 8 + (m_tile & 1) * 4 + wq

    n = 1024
    rows = [phys(h) for h in range(n)]
    assert sorted(rows) == list(range(n))
    for h in range(n):
        r = rows[h]
        m_tile, u = r // 128, r % 128
        assert head_of(m_tile, u // 32, u % 32) == h
    for m_tile in range(8):
        for wq in range(4):
            res = {head_of(m_tile, wq, l) % 8 for l in range(32)}
            assert len(res) == 1
            # row pitch 15069 floats: 8 heads further the sector phase repeats, so one residue = one phase
            assert len({(head_of(m_tile, wq, l) * 15069) % 8 for l in range(32)}) == 1
