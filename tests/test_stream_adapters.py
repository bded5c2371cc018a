"""The Python side of the bzip2 stream calls, without the library: the read / write callbacks over the reference's
streams (compressjs_b200/_pump.py) and the command line's streams (bin/compressjs:60-120)."""
import ctypes as C
import os

import pytest

from compressjs_b200 import _pump as P
from compressjs_b200 import cli


class ByteIn:
    """A readByte-only stream (-1 at the end)."""

    def __init__(self, data):
        self.data, self.pos, self.calls = data, 0, 0

    def readByte(self):
        self.calls += 1
        if self.pos >= len(self.data):
            return -1
        self.pos += 1
        return self.data[self.pos - 1]


class ChunkIn:
    """A read(buf, off, len) stream whose reads return at most `most` bytes each (short reads)."""

    def __init__(self, data, most):
        self.data, self.pos, self.most, self.asked = data, 0, most, []

    def readByte(self):
        raise AssertionError("read() is there: readByte must not be used")

    def read(self, buf, off, length):
        self.asked.append(length)
        k = min(length, self.most, len(self.data) - self.pos)
        buf[off:off + k] = self.data[self.pos:self.pos + k]
        self.pos += k
        return k


class ByteOut:
    def __init__(self):
        self.b = bytearray()

    def writeByte(self, x):
        self.b.append(x)


class ChunkOut(ByteOut):
    def __init__(self):
        super().__init__()
        self.calls = 0

    def writeByte(self, x):
        raise AssertionError("write() is there: writeByte must not be used")

    def write(self, buf, off, length):
        self.calls += 1
        self.b += buf[off:off + length]
        return length


def pull(pump, cap):
    """Call the read callback as the library does, until it returns 0: (the bytes, the return values)."""
    buf = (C.c_uint8 * cap)()
    out, rets = bytearray(), []
    while True:
        k = pump.read_fn(None, C.cast(buf, C.POINTER(C.c_uint8)), cap)
        rets.append(k)
        if k <= 0:
            return bytes(out), rets
        assert k <= cap
        out += bytes(buf[:k])


def push(pump, data):
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    return pump.write_fn(None, C.cast(buf, C.POINTER(C.c_uint8)), len(data))


DATA = bytes((i * 7 + i // 300) & 0xFF for i in range(100003))


def test_stream_pair_is_the_reference_case():
    assert P.is_stream_pair(ByteIn(b""), ByteOut())
    assert not P.is_stream_pair(b"abc", ByteOut())
    assert not P.is_stream_pair(ByteIn(b""), None)
    assert not P.is_stream_pair(ByteIn(b""), bytearray(3))


@pytest.mark.parametrize("cap", [1, 7, 4096, 200000])
def test_read_byte_stream_in_chunks(cap):
    s = ByteIn(DATA)
    got, rets = pull(P.Pump(s, ByteOut()), cap)
    assert got == DATA and rets[-1] == 0
    assert all(0 < k <= min(cap, P.BYTE_CHUNK) for k in rets[:-1])
    # once the end is seen the stream is not asked again
    assert s.calls == len(DATA) + 1


@pytest.mark.parametrize("cap,most", [(1, 5), (13, 5), (4096, 1000), (1 << 20, 65536)])
def test_read_method_short_reads_are_not_the_end(cap, most):
    s = ChunkIn(DATA, most)
    got, rets = pull(P.Pump(s, ByteOut()), cap)
    assert got == DATA
    assert rets[-1] == 0 and all(0 < k <= min(cap, most) for k in rets[:-1])
    assert all(a <= min(cap, P.READ_CHUNK) for a in s.asked)


def test_empty_input():
    assert pull(P.Pump(ByteIn(b""), ByteOut()), 64) == (b"", [0])
    assert pull(P.Pump(ChunkIn(b"", 9), ByteOut()), 64) == (b"", [0])


def test_write_adapters():
    o = ByteOut()
    p = P.Pump(ByteIn(b""), o)
    for piece in (b"a", DATA[:999], DATA[999:]):
        assert push(p, piece) == 0
    assert bytes(o.b) == b"a" + DATA
    o = ChunkOut()
    p = P.Pump(ByteIn(b""), o)
    assert push(p, DATA[:10]) == 0 and push(p, DATA[10:]) == 0
    assert bytes(o.b) == DATA and o.calls == 2


class Boom(Exception):
    pass


def test_exception_in_read_aborts_and_is_raised_again():
    class Bad(ByteIn):
        def readByte(self):
            if self.pos == 10:
                raise Boom("read failed")
            return super().readByte()

    p = P.Pump(Bad(DATA), ByteOut())
    buf = (C.c_uint8 * 64)()
    assert p.read_fn(None, C.cast(buf, C.POINTER(C.c_uint8)), 64) == -1      # an abort, never 0 (the end)
    assert p.read_fn(None, C.cast(buf, C.POINTER(C.c_uint8)), 64) == -1      # and it stays aborted
    with pytest.raises(Boom):
        p.check(-103, lambda rc: AssertionError("the callback's exception comes first"))
    p.check(0, None)   # raised once


def test_exception_in_write_aborts_and_is_raised_again():
    class Bad(ByteOut):
        def writeByte(self, x):
            raise Boom("disk full")

    p = P.Pump(ByteIn(b""), Bad())
    assert push(p, b"xyz") != 0
    with pytest.raises(Boom):
        p.check(-103, lambda rc: AssertionError())


def test_a_read_that_claims_too_much_aborts():
    class Liar(ChunkIn):
        def read(self, buf, off, length):
            return length + 1

    p = P.Pump(Liar(DATA, 10), ByteOut())
    buf = (C.c_uint8 * 8)()
    assert p.read_fn(None, C.cast(buf, C.POINTER(C.c_uint8)), 8) == -1
    with pytest.raises(ValueError):
        p.check(-103, None)


def test_check_raises_the_call_error():
    p = P.Pump(ByteIn(b""), ByteOut())
    with pytest.raises(KeyError):
        p.check(-5, lambda rc: KeyError(rc))


# ---- the command line's streams ----
class File:
    def __init__(self):
        self.b = bytearray()
        self.flushes = 0

    def write(self, b):
        self.b += b

    def flush(self):
        self.flushes += 1


def test_cli_in_stream_reads_chunks(tmp_path):
    f = tmp_path / "f"
    f.write_bytes(DATA)
    fd = os.open(f, os.O_RDONLY)
    try:
        got, rets = pull(P.Pump(cli.InStream(fd), ByteOut()), 4099)
    finally:
        os.close(fd)
    assert got == DATA and rets[-1] == 0
    r, w = os.pipe()
    os.write(w, b"piped" * 100)
    os.close(w)
    try:
        got, _ = pull(P.Pump(cli.InStream(r), ByteOut()), 7)
    finally:
        os.close(r)
    assert got == b"piped" * 100


@pytest.mark.parametrize("pieces", [[1], [4096], [4097], [4095, 1, 1], [3, 8190, 4096, 5], [12288], [12289, 4095], [100003]])
def test_cli_out_stream_flushes_whole_buffers_only_when_the_next_byte_comes(pieces):
    """bin/compressjs:100-116: after T bytes the file holds the first 4096 * ((T - 1) // 4096); flush() writes the rest.
    write() of a piece behaves as writeByte of each of its bytes."""
    data = DATA[:sum(pieces)]
    f, g = File(), File()
    s, t = cli.OutStream(f), cli.OutStream(g)
    o = 0
    for k in pieces:
        assert s.write(data, o, k) == k
        for b in data[o:o + k]:
            t.writeByte(b)
        o += k
        assert bytes(f.b) == bytes(g.b) == data[:cli.FLUSH * ((o - 1) // cli.FLUSH)]
    s.flush()
    assert bytes(f.b) == data and f.flushes == 1


def test_cli_out_stream_through_the_pump():
    f = File()
    p = P.Pump(ByteIn(b""), cli.OutStream(f))
    for a, b in ((0, 5000), (5000, 5001), (5001, 9000)):
        assert push(p, DATA[a:b]) == 0
    assert bytes(f.b) == DATA[:8192]   # the error path: nothing flushes the last, partial buffer
