"""What a failed GPU decode delivers before it raises, as compressjs does: the reference writes every decoded byte to its
output stream as it goes (lib/Bzip2.js:405-448) and calls table's callback once per good block (:508-548), so the
blocks in front of an error are out when it throws, and so are the bytes of a block whose CRC fails.  Every expected
prefix comes from the model or the oracle decoder of tests/partial_cases.py, which tests/test_decode_partial_oracle.py
pins to each other; the error code is always the one the call raised before."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import bz2synth as W
from tests import partial_cases as P
from tests import util as T

pytestmark = pytest.mark.gpu

FILES = {name: (f, ms) for name, f, ms in P.files()}
STREAM_MAX = 1 << 20   # larger prefixes are checked through buffers only (writeByte is one Python call per byte)


class Sink:
    def __init__(self):
        self.buf = bytearray()

    def writeByte(self, b):
        self.buf.append(b)


def _B():
    from compressjs_b200 import Bzip2
    return Bzip2


def _code(fn):
    """fn() must raise a Bzip2Error: its errorCode."""
    from compressjs_b200 import Bzip2Error
    with pytest.raises(Bzip2Error) as e:
        fn()
    return e.value.errorCode


def _check_decode(data, ms, code, prefix):
    """decompressFile(data) raises `code` after handing `prefix` to a stream, a longer and a shorter buffer."""
    B = _B()
    if len(prefix) <= STREAM_MAX:
        s = Sink()
        assert _code(lambda: B.decompressFile(data, s, ms)) == code
        assert bytes(s.buf) == prefix
    longer = bytearray(b"\xa5" * (len(prefix) + 100))
    assert _code(lambda: B.decompressFile(data, longer, ms)) == code
    assert longer[:len(prefix)] == prefix and longer[len(prefix):] == b"\xa5" * 100
    k = len(prefix) // 2
    shorter = np.full(k, 0xA5, np.uint8)
    assert _code(lambda: B.decompressFile(data, shorter, ms)) == code
    assert shorter.tobytes() == prefix[:k]
    for out in (None, len(prefix)):   # nothing observable, as there
        assert _code(lambda: B.decompressFile(data, out, ms)) == code


def _check_table(data, ms, code, rows):
    got = []
    assert _code(lambda: _B().table(data, lambda p, s: got.append((p, s)), ms)) == code
    assert got == rows


@pytest.mark.parametrize("name", sorted(FILES))
def test_synthetic_case_partial(name):
    f, ms = FILES[name]
    exp = f.expect(ms)
    if exp[0] == "err":
        _check_decode(f.data, ms, exp[1], P.expect_partial(f, ms))
    t = f.expect_table()
    if t[0] == "err":
        _check_table(f.data, False, t[1], P.expect_table_partial(f))
    if ms:   # the table over every member: the oracle
        o = P.oracle_table(f.data, True)
        if o[0] == "err":
            _check_table(f.data, True, o[1], o[2])
    for pos, b in f.member_blocks[0]:
        e = P.block_expect(b)
        if e[0] == "err" and e[2]:   # fails on its CRC only
            s = Sink()
            assert _code(lambda: _B().decompressBlock(f.data, pos, s)) == e[1], pos
            assert bytes(s.buf) == e[2], pos


def _against_oracle(z, ms=False, out_len=None):
    """decompressFile and table of z equal the oracle: the result, or the error code and what went out before it."""
    B = _B()
    o = P.oracle_decompress(z, ms)
    if o[0] == "ok":
        assert B.decompressFile(z, None, ms) == o[1]
    else:
        out = bytearray(b"\xa5" * ((out_len or len(o[2])) + 64))
        assert _code(lambda: B.decompressFile(z, out, ms)) == o[1]
        assert out[:len(o[2])] == o[2] and out[len(o[2]):] == b"\xa5" * (len(out) - len(o[2]))
    o = P.oracle_table(z, ms)
    got = []
    if o[0] == "ok":
        B.table(z, lambda p, s: got.append((p, s)), ms)
        assert got == o[1]
    else:
        _check_table(z, ms, o[1], o[2])


def _mixed_level1():
    data = T.ascii_random(150000, 11) + T.runs(150000, 12) + T.texty(200000, 13) + T.ascii_random(60000, 14)
    z, tr = O.bzip2_compress(data, 1, trace=True)
    assert len(tr) >= 5
    return data, z, tr


def _flip(z, bit, mask=None):
    b = bytearray(z)
    b[bit // 8] ^= (0x80 >> (bit % 8)) if mask is None else mask
    return bytes(b)


def test_truncation_sweep():
    data, z, tr = _mixed_level1()
    cuts = set(range(5))
    for t in tr:
        m = t.bit_start // 8
        cuts |= {m + d for d in range(7)}
        cuts.add((t.bit_start + t.bit_len // 2) // 8)
    eos = (tr[-1].bit_start + tr[-1].bit_len) // 8
    cuts |= set(range(eos, len(z)))      # inside the end-of-stream magic and the stream CRC, up to one byte short
    for cut in sorted(cuts):
        assert cut < len(z)
        _against_oracle(z[:cut], out_len=len(data))


def _block_bytes(z, pos):
    """decompressBlock of a block whose only failure is its CRC: the bytes it delivered."""
    s = Sink()
    assert _code(lambda: _B().decompressBlock(z, pos, s)) == W.DATA_ERROR
    return bytes(s.buf)


def test_corrupted_block_crc_stream_crc_and_tables():
    data, z, tr = _mixed_level1()
    B = _B()
    rows = O.bzip2_table(z)
    for k in (0, len(tr) // 2, len(tr) - 1):
        t = tr[k]
        bad = _flip(z, t.bit_start + 48)      # stored block CRC
        _check_decode(bad, False, W.DATA_ERROR, data[:t.raw_start + t.raw_len])
        _check_table(bad, False, W.DATA_ERROR, rows[:k])
        block = _block_bytes(bad, t.bit_start)
        assert block == data[t.raw_start:t.raw_start + t.raw_len]
    bad = _flip(z, tr[-1].bit_start + tr[-1].bit_len + 48)   # stored stream CRC
    _check_decode(bad, False, W.DATA_ERROR, data)
    got = []
    B.table(bad, lambda p, s: got.append((p, s)))             # table does not check it
    assert got == rows
    # a byte of the middle block's selectors, code lengths or codes: an error inside the block, none of its bytes go out
    t = tr[len(tr) // 2]
    start = t.bit_start // 8
    hit = 0
    for j in range(start + 60, start + 3000, 97):
        bad = _flip(z, 8 * j, 0xFF)
        o = P.oracle_decompress(bad)
        if o[0] == "err" and len(o[2]) == t.raw_start:
            _check_decode(bad, False, o[1], data[:t.raw_start])
            _check_table(bad, False, o[1], rows[:len(tr) // 2])
            hit += 1
    assert hit >= 3


def test_multistream_tails():
    first = T.texty(30000, 21)
    z1 = O.bzip2_compress(first, 1)
    z2 = O.bzip2_compress(T.ascii_random(250000, 22), 2)
    for name, tail, code in (("BZh0", b"BZh0" + z2[4:], W.NOT_BZIP), ("garbage", b"\x00garbage\xff" * 20, W.NOT_BZIP),
                             ("truncated", z2[:len(z2) // 2], None)):
        cat = z1 + tail
        o = P.oracle_decompress(cat, True)
        assert o[0] == "err" and o[2][:len(first)] == first, name
        if code is not None:
            assert o[1] == code and o[2] == first, name
        _check_decode(cat, True, o[1], o[2])
        _against_oracle(cat, True)


_SEAM_SCRIPT = r"""
import sys
sys.path.insert(0, %(root)r)
from compressjs_b200 import Bzip2, Bzip2Error
from tests import bz2synth as W, partial_cases as P, synth_corpus as SC
blocks = [W.from_content(SC.rand_bytes(300 + 40 * i, 700 + i, 97, 100)) for i in range(40)]
variants = [list(blocks), list(blocks)]
variants[0][30] = P.with_crc(blocks[30], blocks[30].crc ^ 4)
variants[1][30] = W.from_content(SC.rand_bytes(900, 799, 97, 100), rand=1)
for v in variants:
    f = W.File(W.Member(v))
    exp, prefix = f.expect(), P.expect_partial(f)
    assert exp[0] == "err" and len(prefix) > 0
    out = bytearray(b"\xa5" * (len(prefix) + 10))
    try:
        Bzip2.decompressFile(f.data, out)
        raise SystemExit("no error")
    except Bzip2Error as e:
        assert e.errorCode == exp[1], (e.errorCode, exp)
    assert out[:len(prefix)] == prefix and out[len(prefix):] == b"\xa5" * 10
    rows = []
    try:
        Bzip2.table(f.data, lambda p, s: rows.append((p, s)))
        raise SystemExit("no error")
    except Bzip2Error as e:
        assert e.errorCode == f.expect_table()[1]
    assert rows == P.expect_table_partial(f) and len(rows) == 30, len(rows)
print("ok")
"""


@pytest.mark.parametrize("env", [{"B2_DEC_BATCH": "7"}, {"B2_DEC_KEEP_CLS": "5"}])
def test_batch_seams(env):
    """40 small blocks, the failure in block 30, in decode batches of 7 blocks / with the count-byte classes
    recomputed at expansion.  A child process, because the library reads the hooks per call but the tests share it."""
    r = subprocess.run([sys.executable, "-c", _SEAM_SCRIPT % {"root": T.ROOT}], env=dict(os.environ, **env),
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stdout + r.stderr[-3000:]


def test_scale_256mib():
    from compressjs_b200 import _native
    B = _B()
    data = T.ascii_random(192 << 20, 31) + T.runs(64 << 20, 32)
    z = B.compressFile(data, None, 9)
    tr = _native.last_trace()
    assert len(tr) >= 200
    bits = np.unpackbits(np.frombuffer(z[tr[-1].bit_start // 8:tr[-1].bit_start // 8 + 8], np.uint8))
    ph = tr[-1].bit_start % 8
    assert int("".join(map(str, bits[ph:ph + 48])), 2) == W.BLOCK_MAGIC
    src = np.frombuffer(data, np.uint8)
    out = np.full(len(data), 0xA5, np.uint8)
    # the stored CRC of the second-to-last block: everything through that block
    t = tr[-2]
    end = t.raw_start + t.raw_len
    assert _code(lambda: B.decompressFile(_flip(z, t.bit_start + 48), out)) == W.DATA_ERROR
    assert np.array_equal(out[:end], src[:end]) and bool((out[end:] == 0xA5).all())
    # cut inside the last block: the blocks before it, then what the reference makes of the cut block
    t = tr[-1]
    cut = z[:(t.bit_start + t.bit_len // 2) // 8]
    o = P.oracle_decompress_block(cut, t.bit_start)
    assert o[0] == "err"
    out[:] = 0xA5
    assert _code(lambda: B.decompressFile(cut, out)) == o[1]
    k = t.raw_start + len(o[2])
    assert np.array_equal(out[:t.raw_start], src[:t.raw_start])
    assert out[t.raw_start:k].tobytes() == o[2] and bool((out[k:] == 0xA5).all())


def test_all_or_nothing_entry_points_are_unchanged():
    """b2_bzip2_decompress / _block / _table return nothing on an error; the partial calls equal them on valid streams."""
    from compressjs_b200 import _native
    L = _native.lib()
    data, z, tr = _mixed_level1()
    bad = _flip(z, tr[1].bit_start + 48)
    u8p, u64p, u32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
    out, n = u8p(), C.c_size_t(0)
    assert L.b2_bzip2_decompress(bad, len(bad), 0, C.byref(out), C.byref(n)) == W.DATA_ERROR
    assert not out and n.value == 0
    assert L.b2_bzip2_decompress_block(bad, len(bad), tr[1].bit_start, C.byref(out), C.byref(n)) == W.DATA_ERROR
    assert not out and n.value == 0
    bp, sz, cnt = u64p(), u32p(), C.c_size_t(0)
    assert L.b2_bzip2_table(bad, len(bad), 0, C.byref(bp), C.byref(sz), C.byref(cnt)) == W.DATA_ERROR
    assert not bp and not sz and cnt.value == 0
    assert "Bad block CRC" in _native.last_error()
    # the partial call on the same stream: the bytes through the failing block, to be freed
    assert L.b2_bzip2_decompress_partial(bad, len(bad), 0, C.byref(out), C.byref(n)) == W.DATA_ERROR
    assert C.string_at(out, n.value) == data[:tr[1].raw_start + tr[1].raw_len]
    L.b2_free(out)

    def both(fn_old, fn_new, z, arg):
        res = []
        for fn in (fn_old, fn_new):
            o, m = u8p(), C.c_size_t()
            assert fn(z, len(z), arg, C.byref(o), C.byref(m)) == 0, _native.last_error()
            res.append(C.string_at(o, m.value))
            L.b2_free(o)
        return res

    for k in range(5):
        zk = T.fixture("sample%d.bz2" % k)
        a, b = both(L.b2_bzip2_decompress, L.b2_bzip2_decompress_partial, zk, 0)
        assert a == b == T.fixture("sample%d.ref" % k)
        rows = []
        for fn in (L.b2_bzip2_table, L.b2_bzip2_table_partial):
            p, s, c = u64p(), u32p(), C.c_size_t()
            assert fn(zk, len(zk), 0, C.byref(p), C.byref(s), C.byref(c)) == 0
            rows.append([(p[i], s[i]) for i in range(c.value)])
            L.b2_free(p)
            L.b2_free(s)
        assert rows[0] == rows[1] and len(rows[0]) >= 1
    a, b = both(L.b2_bzip2_decompress_block, L.b2_bzip2_decompress_block_partial, T.fixture("sample2.bz2"), 544888)
    assert a == b == T.fixture("sample2.544888")
