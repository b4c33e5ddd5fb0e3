#!/usr/bin/env python
"""Copy the reference's UV-texture data into ``oracle/_ref/inference/`` (TEST INFRASTRUCTURE).

``inference/texture_data.npy`` (the texel table of ``UVTextureCreator``) and ``inference/generic_model.pkl`` (its mesh,
whose faces the tests compare with the packed asset) sit beside the byte-compiled ``inference/*.pyc`` that
oracle/build_ref.py writes, so the tests and the unchanged ``demo.py … uv_texture`` find them where the reference does
(``get_relative_path``).  ``oracle/_ref/`` is git-ignored: the files never enter history.

Run by ``__graft_entry__.build()`` after oracle/build_ref.py; a no-op where the reference is absent.
"""
import os
import shutil

from oracle.build_ref import OUT, REF

FILES = ("inference/texture_data.npy", "inference/generic_model.pkl")


def build(ref: str = REF, out: str = OUT) -> bool:
    if not os.path.isdir(ref):
        return False
    for rel in FILES:
        src, dst = os.path.join(ref, rel), os.path.join(out, rel)
        if not os.path.isfile(src):
            continue
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not (os.path.isfile(dst) and os.path.getsize(dst) == os.path.getsize(src)):
            shutil.copyfile(src, dst)
    return True


if __name__ == "__main__":
    print("oracle/_ref UV data copied" if build() else f"{REF} absent: nothing to do")
