"""reference path: inference/ -- uv_texture.py here (the GPU texture kernel); every other module, and the data files, from
the reference's own inference/ directory, which this package's ``__path__`` also covers."""
import os
import sys

_HERE = os.path.realpath(os.path.dirname(os.path.abspath(__file__)))
for _entry in list(sys.path):
    _dir = os.path.realpath(os.path.join(_entry or os.getcwd(), "inference"))
    if os.path.isdir(_dir) and _dir != _HERE and _dir not in __path__:
        __path__.append(_dir)
