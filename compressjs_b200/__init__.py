"""compressjs_b200 -- GPU-native (H100) drop-in for the bzip2 block pipeline of cscott/compressjs.

Mirrors the reference's package surface for that path (main.js:1-29): ``Bzip2``, ``BWT`` and (experimental)
``BWTC`` with the reference's member names and argument meaning.  All compute runs
in libb2bz.so (hand-written CUDA for sm_90a) through the C ABI in include/b2bz.h; there is no
CPU fallback.
"""
from . import _native
from .bzip2 import Bzip2, Bzip2Error
from .bwt import BWT
from .bwtc import BWTC

version = "0.0.1"  # main.js:5

__all__ = ["Bzip2", "BWT", "BWTC", "Bzip2Error", "version"]
