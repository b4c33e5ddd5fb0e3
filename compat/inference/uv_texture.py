"""reference path: inference/uv_texture.py -> dad_3dheads_b200.uv_texture.

``UVTextureCreator()(image, predictions)`` keeps the reference's signature and bytes: the texture of the head decoded from
``predictions["3dmm_params"]`` with ``to_2d=False`` (uv_texture.py:49-51), computed by the GPU kernel instead of the
per-texel loop.  The table is the reference's ``texture_data.npy`` from its inference/ directory; neither psbody nor chumpy
is needed, because the faces are FLAME's packed ones (``generic_model.pkl['f']``)."""
import os

import numpy as np
import torch

from dad_3dheads_b200.uv_texture import UvTextureTable, uv_textures
from model_training.head_mesh import HeadMesh


def _reference_file(name: str) -> str:
    """``name`` in the first inference/ directory of the package path that holds it (the reference's)."""
    import inference
    for d in inference.__path__:
        p = os.path.join(d, name)
        if os.path.isfile(p):
            return p
    raise FileNotFoundError(f"{name} not found in the reference's inference/ directory ({list(inference.__path__)})")


class UVTextureCreator:
    def __init__(self):
        self.head_mesh = HeadMesh()
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.table = UvTextureTable.load(_reference_file("texture_data.npy"), self.device)

    def get_mesh(self, predicted_mesh):
        """The head's [5023,3] projected vertices with depth (uv_texture.py:49-51 without the psbody Mesh)."""
        return self.head_mesh.reprojected_vertices(params_3dmm=predicted_mesh["3dmm_params"], to_2d=False)[0]

    def __call__(self, image, mesh, *args, **kwargs):
        v = self.get_mesh(mesh).to(self.device, torch.float32).contiguous()[None]
        frame = torch.from_numpy(np.ascontiguousarray(image[..., :3], dtype=np.uint8)).to(self.device)[None]
        return uv_textures(self.table, frame.contiguous(), v)[0].cpu().numpy()
