"""compressjs.Bzip2 on the GPU: same four entry points as lib/Bzip2.js:879-933, and decompressBlocks (decompressBlock at
many positions in one pass)."""
import ctypes as C
from collections import namedtuple

import numpy as np

from . import _native
from ._pump import Pump, is_stream_pair
from ._streams import coerce_input, deliver_output


class Bzip2Error(TypeError):
    """Decode errors are TypeErrors carrying ``errorCode`` (lib/Bzip2.js:82-88)."""

    def __init__(self, code, msg):
        super().__init__(msg)
        self.errorCode = code


class Err:  # lib/Bzip2.js:62-72
    OK = 0
    LAST_BLOCK = -1
    NOT_BZIP_DATA = -2
    UNEXPECTED_INPUT_EOF = -3
    UNEXPECTED_OUTPUT_EOF = -4
    DATA_ERROR = -5
    OUT_OF_MEMORY = -6
    OBSOLETE_INPUT = -7
    END_OF_BLOCK = -8


def _error(rc):
    msg = _native.last_error()
    if rc == -100:
        return ValueError(msg or "Invalid block size multiplier")  # `new Error(...)` lib/Bzip2.js:888-890
    if rc in (Err.NOT_BZIP_DATA, Err.UNEXPECTED_INPUT_EOF, Err.DATA_ERROR, Err.OBSOLETE_INPUT):
        return Bzip2Error(rc, msg)
    return RuntimeError("libb2bz: %s (code %d)" % (msg, rc))


def _raise(rc):
    raise _error(rc)


def _level(props):
    """compressFile's block size multiplier: props if it is a number (9 otherwise), 1..9 (lib/Bzip2.js:881-890)."""
    level = 9
    if isinstance(props, (int, float)) and not isinstance(props, bool):
        level = props
    if level < 1 or level > 9 or int(level) != level:
        raise ValueError("Invalid block size multiplier")
    return int(level)


# The flavors (include/b2bz.h B2_BZ2_*): compressFile writes the bytes of compressjs (the default) or of libbz2, and
# decompressFile reads as compressjs (the default) or as bzip2 -d reads
FLAVORS = {"compressjs": 0, "libbz2": 1}


def _flavor(flavor):
    if not isinstance(flavor, str) or flavor not in FLAVORS:
        raise ValueError("unknown bzip2 flavor %r (expected one of %s)" % (flavor, ", ".join(sorted(FLAVORS))))
    return FLAVORS[flavor]


def _take(L, p, n):
    arr = np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else np.zeros(0, dtype=np.uint8)
    L.b2_free(p)
    return arr


def _partial(call):
    """Run a b2_bzip2_decompress*_partial call: (decoded bytes, None), or on a decode error (the bytes the reference has
    written by the time it throws -- lib/Bzip2.js:405-448 writes as it decodes --, the error)."""
    L = _native.lib()
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = call(C.byref(out), C.byref(n))
    if rc and not out:
        _raise(rc)
    err = _error(rc) if rc else None   # before `output` can call into the library again
    return _take(L, out, n), err


def _file(input, multistream=False, flavor=0):
    L = _native.lib()
    data = coerce_input(input)
    return _partial(lambda out, n: L.b2_bzip2_decompress_partial_flavor(
        data.ctypes.data if data.size else None, data.size, int(bool(multistream)), out, n, flavor))


def _block(input, pos):
    L = _native.lib()
    data = coerce_input(input)
    return _partial(lambda out, n: L.b2_bzip2_decompress_block_partial(
        data.ctypes.data if data.size else None, data.size, int(pos), out, n))


# Bzip2.recover's rows (include/b2bz.h b2_recovered_block), with the status as a string
RecoveredBlock = namedtuple("RecoveredBlock", "bitpos endbit out_off size crc got status")
REC_STATUS = ("INTACT", "BAD_CRC", "DATA_ERROR", "OBSOLETE", "INSIDE")


def _rows(L, rows, count):
    out = [RecoveredBlock(r.bitpos, r.endbit, r.out_off, r.size, r.crc, r.got, REC_STATUS[r.status])
           for r in (rows[i] for i in range(count.value))]
    L.b2_free(rows)
    return out


def _deliver(output, data, err):
    """On a decode error `output` gets the bytes decoded before it first, then the error is raised."""
    if err is not None:
        deliver_output(output, data, partial=True)
        raise err
    return deliver_output(output, data)


class Bzip2:
    Err = Err

    @staticmethod
    def compressFile(input, output=None, props=None, *, flavor="compressjs"):
        """lib/Bzip2.js:879-929.  props: block size multiplier 1..9 (default 9).  When input has readByte and output
        has writeByte, the input is read and the output written as the encode goes, in bounded memory.
        flavor: "compressjs" writes the bytes of compressjs; "libbz2" those of libbz2 (``bzip2 -N``, Python's
        ``bz2.compress(data, N)``), whose block cut and Huffman tables differ."""
        fl = _flavor(flavor)   # before anything is read
        if is_stream_pair(input, output):
            level = _level(props)
            pump = Pump(input, output)
            rc = _native.lib().b2_bzip2_compress_stream_flavor(pump.read_fn, pump.write_fn, None, level, fl)
            pump.check(rc, _error)
            return output
        L = _native.lib()
        data = coerce_input(input)
        level = _level(props)
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        rc = L.b2_bzip2_compress_flavor(data.ctypes.data if data.size else None, data.size, int(level), C.byref(out), C.byref(n), fl)
        if rc:
            _raise(rc)
        return deliver_output(output, _take(L, out, n))

    @staticmethod
    def decompressFile(input, output=None, multistream=False, *, flavor="compressjs"):
        """lib/Bzip2.js:454-481 (Bunzip.decode).  On a decode error the output receives the bytes decoded before it.
        When input has readByte and output has writeByte, the input is read and the output written as the decode goes,
        in bounded memory.
        flavor: "compressjs" decodes as compressjs does; "libbz2" as ``bzip2 -d`` does: it decodes randomised blocks,
        raises errorCode -3 (Err.UNEXPECTED_INPUT_EOF) for a file cut off where a magic is due, ignores trailing
        garbage behind a member, and rejects two streams compressjs accepts (include/b2bz.h states the rules)."""
        fl = _flavor(flavor)   # before anything is read
        if is_stream_pair(input, output):
            pump = Pump(input, output)
            rc = _native.lib().b2_bzip2_decompress_stream_flavor(pump.read_fn, pump.write_fn, None, int(bool(multistream)), fl)
            pump.check(rc, _error)
            return output
        return _deliver(output, *_file(input, multistream, fl))

    @staticmethod
    def decompressBlock(input, pos, output=None):
        """lib/Bzip2.js:482-503 (Bunzip.decodeBlock): decode the single block whose magic starts at bit `pos`.  A block
        whose only failure is its CRC delivers its bytes before the error is raised."""
        return _deliver(output, *_block(input, pos))

    @staticmethod
    def decompressBlocks(input, positions, output=None):
        """GPU extension: decompressBlock at every bit position of `positions`, in one pass.  The result is that of
        ``[decompressBlock(input, p) for p in positions]`` (output None: a list of bytes), or of
        ``for p in positions: decompressBlock(input, p, output)`` with a writeByte stream, which is returned.  On an error
        the stream first receives what that loop would have written, then the first failing position's error is raised.
        Positions may repeat and come in any order; every block is held to the dbufSize of the file's first header."""
        if output is not None and not hasattr(output, "writeByte"):
            raise TypeError("decompressBlocks writes to a stream (writeByte) or returns a list: output must be one or None")
        L = _native.lib()
        data = coerce_input(input)
        pos = np.array([int(p) & 0xFFFFFFFFFFFFFFFF for p in positions], dtype=np.uint64)   # as c_uint64 takes decompressBlock's pos
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        ends, done = C.POINTER(C.c_uint64)(), C.c_size_t()
        rc = L.b2_bzip2_decompress_blocks(data.ctypes.data if data.size else None, data.size, pos.ctypes.data if pos.size else None,
                                          pos.size, C.byref(out), C.byref(n), C.byref(ends), C.byref(done))
        if rc and not out:
            _raise(rc)
        err = _error(rc) if rc else None
        stops = [int(ends[i]) for i in range(done.value)]
        L.b2_free(ends)
        buf = _take(L, out, n)
        if output is not None:
            deliver_output(output, buf, partial=err is not None)
        if err is not None:
            raise err
        if output is not None:
            return output
        return [buf[s:e].tobytes() for s, e in zip([0] + stops[:-1], stops)]

    @staticmethod
    def recover(input, output=None, *, repair=False):
        """GPU extension: recover the intact blocks of a damaged bzip2 file.  Every block magic of the input is a
        candidate, decoded as decompressBlock decodes a block of a BZh9 file and walked in position order
        (include/b2bz.h b2_bzip2_recover gives the rules).  Returns (output, blocks): output receives the intact blocks'
        decoded bytes, or with `repair` one bzip2 stream made of their bits, and blocks has one RecoveredBlock per
        candidate, whose status is "INTACT", "BAD_CRC", "DATA_ERROR", "OBSOLETE" or "INSIDE" (it starts inside an intact
        block).  Damage is a result, not an error.  When input has readByte and output has writeByte, the input is read
        and the output written as the recovery goes, in bounded memory."""
        L = _native.lib()
        mode = 1 if repair else 0
        rows, count = C.POINTER(_native.RecoveredBlock)(), C.c_size_t()
        if is_stream_pair(input, output):
            pump = Pump(input, output)
            rc = L.b2_bzip2_recover_stream(pump.read_fn, pump.write_fn, None, mode, C.byref(rows), C.byref(count))
            pump.check(rc, _error)
            return output, _rows(L, rows, count)
        data = coerce_input(input)
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        rc = L.b2_bzip2_recover(data.ctypes.data if data.size else None, data.size, mode, C.byref(out), C.byref(n),
                                C.byref(rows), C.byref(count))
        if rc:
            _raise(rc)
        blocks = _rows(L, rows, count)
        return deliver_output(output, _take(L, out, n)), blocks

    @staticmethod
    def table(input, callback, multistream=False):
        """lib/Bzip2.js:508-548: callback(bit position, decoded bytes) once per block.  On a decode error the callback
        has been called for every block in front of the failing one when the error is raised."""
        L = _native.lib()
        data = coerce_input(input)
        bp, sz, cnt = C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint32)(), C.c_size_t()
        rc = L.b2_bzip2_table_partial(data.ctypes.data if data.size else None, data.size, int(bool(multistream)), C.byref(bp), C.byref(sz), C.byref(cnt))
        if rc and not bp:
            _raise(rc)
        err = _error(rc) if rc else None
        rows = [(int(bp[i]), int(sz[i])) for i in range(cnt.value)]
        L.b2_free(bp)
        L.b2_free(sz)
        for pos, size in rows:
            callback(pos, size)
        if err is not None:
            raise err
