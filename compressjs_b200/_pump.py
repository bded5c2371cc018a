"""The read / write callbacks of the stream entry points (b2_bzip2_compress_stream, b2_bzip2_decompress_stream) over
the reference's streams (lib/Stream.js).

An input stream is read with ``read(buf, bufOffset, length)`` when it has one (it returns how many bytes it put, 0 at
the end), else byte by byte with ``readByte()`` (-1 at the end).  An output stream is written with
``write(buf, bufOffset, length)`` when it has one, else with ``writeByte(b)``.  ``buf`` is a writable memoryview of the
library's input buffer for ``read``, and a ``bytes`` object for ``write``.

A ctypes callback that raises returns 0, which the library would take for the end of the input: the output would be
silently cut short.  So every exception raised inside a callback is caught, the call is aborted, and the exception is
raised again once the call has returned (``Pump.check``).
"""
import ctypes as C

from . import _native

EOF_BYTE = -1
READ_CHUNK = 1 << 24   # most bytes asked of a read() stream at once
BYTE_CHUNK = 1 << 16   # most bytes taken from a readByte() stream in one callback


def is_stream_pair(input, output):
    """The case where the reference itself streams: input has readByte and output has writeByte."""
    return hasattr(input, "readByte") and hasattr(output, "writeByte")


def read_into(stream, mv):
    """Put up to len(mv) bytes of `stream` into the writable memoryview `mv`: (how many, whether the stream ended)."""
    if hasattr(stream, "read"):
        k = int(stream.read(mv, 0, min(len(mv), READ_CHUNK)) or 0)
        if k > len(mv):
            raise ValueError("read() returned more bytes than it was asked for")
        return max(k, 0), k <= 0
    got = bytearray()
    ended = False
    for _ in range(min(len(mv), BYTE_CHUNK)):
        b = stream.readByte()
        if b is None or b == EOF_BYTE:
            ended = True
            break
        got.append(b & 0xFF)
    mv[:len(got)] = got
    return len(got), ended


def write_from(stream, data):
    """Hand the bytes `data` to `stream`."""
    if hasattr(stream, "write"):
        stream.write(data, 0, len(data))
        return
    for b in data:
        stream.writeByte(b)


class Pump:
    """The two callbacks of one stream call between `input` and `output`.  Pass ``read_fn`` and ``write_fn`` to the
    call, then ``check(rc)`` its return code."""

    def __init__(self, input, output):
        self.input, self.output = input, output
        self.error = None
        self.ended = False
        self.read_fn = _native.READ_FN(self._read)
        self.write_fn = _native.WRITE_FN(self._write)

    def _read(self, user, buf, cap):
        if self.error is not None:
            return -1
        if self.ended:
            return 0
        try:
            mv = memoryview((C.c_uint8 * cap).from_address(C.cast(buf, C.c_void_p).value)).cast("B")
            k, self.ended = read_into(self.input, mv)   # after the end, the stream is not asked again
            return k
        except BaseException as e:   # noqa: B036 -- re-raised by check()
            self.error = e
            return -1

    def _write(self, user, buf, n):
        if self.error is not None:
            return 1
        try:
            write_from(self.output, C.string_at(buf, n))
            return 0
        except BaseException as e:   # noqa: B036 -- re-raised by check()
            self.error = e
            return 1

    def check(self, rc, error):
        """After the call: a callback's exception first, else error(rc) for a non-zero rc."""
        if self.error is not None:
            e, self.error = self.error, None
            raise e
        if rc:
            raise error(rc)
