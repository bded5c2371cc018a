"""compressjs.BWTC on the GPU (lib/BWTC.js:10-231): same two entry points and the same container bytes.

New in round 1 (see the header of csrc/bwtc.cu for what has been verified where).  The block stages (sentinel BWT, MTF, zero runs) are
the block-parallel kernels of the bzip2 path; the range coder is one serial chain over the file, so this path is
bound by a single GPU thread."""
import ctypes as C

import numpy as np

from . import _native
from ._pump import Pump, is_stream_pair
from ._streams import coerce_input, deliver_output


def _take(L, p, n):
    arr = np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else np.zeros(0, dtype=np.uint8)
    L.b2_free(p)
    return arr


def _level(props):
    """props: block size in units of 100 000 bytes, 1..9; anything else means 9 (lib/BWTC.js:16-19)."""
    if isinstance(props, (int, float)) and not isinstance(props, bool) and 1 <= props <= 9:
        return int(props)
    return 9


def _error(rc):
    if rc == -102:
        return ValueError("Bad magic")   # lib/Util.js:151-153
    return RuntimeError("libb2bz: %s (code %d)" % (_native.last_error(), rc))


def _compress(entry, input, props):
    L = _native.lib()
    data = coerce_input(input)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = getattr(L, entry)(data.ctypes.data if data.size else None, data.size, _level(props), C.byref(out), C.byref(n))
    if rc:
        raise _error(rc)
    return _take(L, out, n)


def _stream_size(input):
    """The header's size field of a stream (lib/Util.js:119-124): its ``size`` when it has a non-negative one, else -1,
    "size unknown"."""
    size = getattr(input, "size", None)
    if isinstance(size, (int, float)) and not isinstance(size, bool) and size >= 0:
        return int(size)
    return -1


def _compress_unsized(input, props=None):
    """BWTC.compressFile of an input stream without a size (lib/Util.js:119-124): the header says "size unknown".  The
    command line writes this for a pipe or an empty file, as bin/compressjs does.  Returns bytes."""
    return _compress("b2_bwtc_compress_unsized", input, props).tobytes()


class BWTC:
    MAGIC = "bwtc"  # lib/BWTC.js:11

    @staticmethod
    def compressFile(input, output=None, props=None):
        """lib/BWTC.js:12-139.  props: block size in units of 100 000 bytes, 1..9; anything else means 9 (:16-19).  When
        input has readByte and output has writeByte, the input is read and the output written as the encode goes, in
        bounded memory, and the header has the input's ``size`` if it has one, else "size unknown" (lib/Util.js:119-124)."""
        if is_stream_pair(input, output):
            pump = Pump(input, output)
            rc = _native.lib().b2_bwtc_compress_stream(pump.read_fn, pump.write_fn, None, _level(props), _stream_size(input))
            pump.check(rc, _error)
            return output
        return deliver_output(output, _compress("b2_bwtc_compress", input, props))

    @staticmethod
    def decompressFile(input, output=None):
        """lib/BWTC.js:141-231.  Raises ValueError("Bad magic") like lib/Util.js:151-153 throws Error("Bad magic").  When
        input has readByte and output has writeByte, the input is read and the output written as the decode goes, in
        bounded memory; on a decode error the output has the blocks decoded before it when the error is raised, as the
        reference writes each block as it ends (lib/BWTC.js:228)."""
        if is_stream_pair(input, output):
            pump = Pump(input, output)
            rc = _native.lib().b2_bwtc_decompress_stream(pump.read_fn, pump.write_fn, None)
            pump.check(rc, _error)
            return output
        L = _native.lib()
        data = coerce_input(input)
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        rc = L.b2_bwtc_decompress(data.ctypes.data if data.size else None, data.size, C.byref(out), C.byref(n))
        if rc:
            raise _error(rc)
        return deliver_output(output, _take(L, out, n))
