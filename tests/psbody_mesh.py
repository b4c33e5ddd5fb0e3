"""psbody.mesh's ``Mesh(v, f)`` as inference/uv_texture.py uses it (``v``, ``estimate_vertex_normals``), restated from
psbody-mesh's published ``Mesh.estimate_vertex_normals``, ``geometry.tri_normals.TriNormalsScaled`` and
``Mesh.faces_by_vertex(as_sparse_matrix=True)`` (TEST INFRASTRUCTURE).  psbody is not installed here, so this restatement
is not pinned against it (DESIGN §2).  The reference's ``_compute_texture_map`` takes the mesh as an argument, so the tests
pass this class to it directly; the import-only stub in oracle/ref_shims is what its module imports."""
import numpy as np
import scipy.sparse as sp


class Mesh:
    def __init__(self, v=None, f=None):
        self.v = np.array(v, dtype=np.float64)                   # psbody keeps its vertices as float64
        self.f = np.require(f, dtype=np.uint32)

    def faces_by_vertex(self, as_sparse_matrix=True):
        if not as_sparse_matrix:
            raise NotImplementedError("only the sparse form estimate_vertex_normals uses")
        row = self.f.flatten()
        col = np.array([range(self.f.shape[0])] * 3).T.flatten()
        data = np.ones(len(col))
        return sp.csr_matrix((data, (row, col)), shape=(self.v.shape[0], len(self.f)))

    def estimate_vertex_normals(self, face_to_verts_sparse_matrix=None):
        f = self.f.astype(np.int64)
        v = self.v.reshape(-1, 3)
        face_normals = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]).reshape(-1, 3)   # TriNormalsScaled
        ftov = face_to_verts_sparse_matrix if face_to_verts_sparse_matrix is not None \
            else self.faces_by_vertex(as_sparse_matrix=True)
        non_scaled_normals = ftov * face_normals
        norms = (np.sum(non_scaled_normals ** 2.0, axis=1) ** 0.5).T
        norms[norms == 0] = 1.0
        return (non_scaled_normals.T / norms).T
