"""Bzip2.decompressBlocks / b2_bzip2_decompress_blocks: decompressBlock at a list of bit positions in one GPU pass.

The oracle is the loop the call replaces, `for p in positions: decompressBlock(input, p, stream)`, whose every step
the other decode tests pin to the reference: the same bytes per position, the same error code and message at the
first failing position in list order, and the same bytes in a stream when the error is raised."""
import bz2
import ctypes as C
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import bz2synth as W
from tests import partial_cases as P
from tests import synth_corpus as SC
from tests import util as T

gpu = pytest.mark.gpu


class Sink:
    def __init__(self):
        self.buf = bytearray()
        self.writeByte = self.buf.append


def _B():
    from compressjs_b200 import Bzip2
    return Bzip2


def _one(data, pos):
    """decompressBlock(data, pos) into a stream: ('ok', bytes) or ('err', code, message, bytes written)."""
    from compressjs_b200 import Bzip2Error
    s = Sink()
    try:
        _B().decompressBlock(data, pos, s)
    except Bzip2Error as e:
        return ("err", e.errorCode, str(e), bytes(s.buf))
    return ("ok", bytes(s.buf))


def _loop(data, positions, memo=None):
    """What the per-position loop gives: ('ok', [bytes per position]) or ('err', code, message, stream bytes)."""
    memo = {} if memo is None else memo
    done = []
    for p in positions:
        if p not in memo:
            memo[p] = _one(data, p)
        r = memo[p]
        if r[0] == "err":
            return ("err", r[1], r[2], b"".join(done) + r[3])
        done.append(r[1])
    return ("ok", done)


def _check(data, positions, memo=None, stream=True):
    """decompressBlocks(data, positions) with no output and with a stream equals the loop; returns the loop's result."""
    from compressjs_b200 import Bzip2Error
    B = _B()
    exp = _loop(data, positions, memo)
    if exp[0] == "ok":
        assert B.decompressBlocks(data, positions) == exp[1]
        if stream:
            s = Sink()
            assert B.decompressBlocks(data, positions, s) is s
            assert bytes(s.buf) == b"".join(exp[1])
        return exp
    with pytest.raises(Bzip2Error) as e:
        B.decompressBlocks(data, positions)
    assert (e.value.errorCode, str(e.value)) == exp[1:3]
    if stream:
        s = Sink()
        with pytest.raises(Bzip2Error) as e:
            B.decompressBlocks(data, positions, s)
        assert (e.value.errorCode, str(e.value)) == exp[1:3]
        assert bytes(s.buf) == exp[3]
    return exp


def _magics(data):
    bm, em = W.magic_positions(data)
    return sorted(bm + em)


# ---- reference fixtures ------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("k", range(5))
def test_table_positions_of_reference_fixtures(k):
    """The .bzt positions (test/bzip2-table.js) in one call: the loop's bytes, the .bzt sizes, and together the .ref."""
    z = T.fixture("sample%d.bz2" % k)
    rows = [tuple(map(int, l.split("\t"))) for l in T.fixture("sample%d.bzt" % k).decode().strip().split("\n")]
    got = _check(z, [p for p, _ in rows], stream=False)[1]
    assert [len(b) for b in got] == [s for _, s in rows]
    assert b"".join(got) == T.fixture("sample%d.ref" % k)


@gpu
def test_block_extracts_reversed_with_repeats():
    """The extracts of test/bzip2-block.js, several blocks of a file in one call, reversed and repeated."""
    for f, poss in (("sample2", [544888, 32, 544888]), ("sample4", [2342106, 1596228, 32, 1596228, 2342106, 2342106])):
        z = T.fixture(f + ".bz2")
        got = _B().decompressBlocks(z, poss)
        for p, b in zip(poss, got):
            if (f, p) != ("sample2", 32):
                assert b == T.fixture("%s.%d" % (f, p)), (f, p)
        assert got == _loop(z, poss)[1]


# ---- the synthetic corpus ------------------------------------------------------------------------------------------
def _corpus_files():
    out = [(name, SC.build(name).file) for name in sorted(SC.CASES)]
    for name, f in list(out):
        v = P.crc_flipped(f)
        if v is not None:
            out.append((name + "+crc", v))
    obsolete = W.from_content(SC.rand_bytes(900, 799, 97, 100), rand=1)   # the randomised bit (lib/Bzip2.js:143)
    out.append(("obsolete", W.File(W.Member([P.lead(), obsolete, P.lead(seed=1)]))))
    return out


CORPUS = dict(_corpus_files())


@functools.lru_cache(maxsize=None)
def _results(name):
    """{position: decompressBlock result} for every magic of a corpus file."""
    f = CORPUS[name]
    return {p: _one(f.data, p) for p in _magics(f.data)}


@gpu
@pytest.mark.parametrize("name", sorted(CORPUS))
def test_synthetic_corpus(name):
    """Every magic of the file (blocks, end-of-stream magics, planted ones), shuffled: the list up to the first position
    the loop fails on must succeed; then that failing position in the middle of the good ones must raise the loop's error
    after the loop's bytes (for a CRC-only failure, including the failing block's own)."""
    f = CORPUS[name]
    memo = dict(_results(name))
    poss = sorted(memo)
    T.rng(len(poss)).shuffle(poss)
    good = [p for p in poss if memo[p][0] == "ok"]
    bad = [p for p in poss if memo[p][0] == "err"]
    first_bad = next((i for i, p in enumerate(poss) if memo[p][0] == "err"), len(poss))
    small = sum(len(r[-1]) for r in memo.values()) <= (4 << 20)   # larger outputs are compared as lists only
    assert _check(f.data, poss[:first_bad], memo, stream=small)[0] == "ok"
    for p in bad:
        lst = good[:len(good) // 2] + [p] + good[len(good) // 2:]
        exp = _check(f.data, lst, memo, stream=small)
        assert exp[0] == "err" and exp[1] == memo[p][1]


@gpu
def test_error_kinds_of_the_corpus_are_reached():
    """The corpus gives a failing position for every kind of block error: origPtr, code hole, the obsolete bit, the
    dbufSize bound, and a CRC-only failure (which delivers the block's bytes)."""
    msgs = set()
    for name in CORPUS:
        for r in _results(name).values():
            if r[0] == "err":
                msgs.add((r[1], r[2] if "CRC" not in r[2] else "crc", bool(r[3])))
    assert (W.DATA_ERROR, "Data error: initial position out of bounds", False) in msgs
    assert (W.DATA_ERROR, "Data error", False) in msgs                     # code hole, dbufSize bound, origPtr >= n
    assert (-7, "Obsolete (pre 0.9.5) bzip format not supported.", False) in msgs
    assert (W.DATA_ERROR, "crc", True) in msgs


@gpu
def test_positions_off_a_magic_and_past_the_end():
    f = CORPUS["orig_0"]
    good = f.block_starts[0]
    n8 = len(f.data) * 8
    for bad in (good + 1, good - 1, n8, n8 + 100, n8 - 1, 2 ** 64 - 1):
        exp = _check(f.data, [good, bad, good])
        assert exp[:3] == ("err", W.NOT_BZIP, "Not bzip data")


# ---- multistream ---------------------------------------------------------------------------------------------------
@gpu
def test_multistream_positions_use_the_first_header():
    """A level-1 member then a level-9 one: every position is held to the first header's dbufSize, so a block of the
    second member that fits only its own level fails and a small one decodes."""
    f = SC.multistream_file()
    assert f.members[0].level < f.members[1].level
    memo = {}
    poss = _magics(f.data)
    res = {p: _one(f.data, p) for p in poss}
    memo.update(res)
    big = f.member_blocks[1][0][0]
    assert res[big][0] == "err" and res[big][1] == W.DATA_ERROR   # fits level 9, not level 1
    good = [p for p in poss if res[p][0] == "ok"]
    assert f.member_blocks[1][1][0] in good                        # a small block of the second member decodes
    _check(f.data, good[::-1], memo)
    _check(f.data, good[:1] + [big] + good[1:], memo)
    # libbz2 members of levels 1 and 9: the second member's 300k block fails under level 1
    a, b = T.texty(150000, 31), T.ascii_random(300000, 32)
    z = bz2.compress(a, 1) + bz2.compress(b, 9)
    rows = []
    _B().table(z, lambda p, s: rows.append(p), True)
    assert len(rows) == 3
    assert _check(z, rows[:2], stream=False)[0] == "ok"
    assert _check(z, [rows[1], rows[2], rows[0]], stream=False)[1] == W.DATA_ERROR


# ---- scale and batch seams -----------------------------------------------------------------------------------------
_SCALE_SCRIPT = r"""
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import torch
from compressjs_b200 import Bzip2
from tests import util as T
nb = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 20
data = T.ascii_random(nb * 99000, 41)
z = Bzip2.compressFile(data, None, 1)
rows = []
Bzip2.table(z, lambda p, s: rows.append((p, s)))
assert len(rows) > nb - 20, len(rows)
assert Bzip2.decompressFile(z) == data
offs = np.concatenate([[0], np.cumsum([s for _, s in rows])])
slices = {p: data[offs[i]:offs[i + 1]] for i, (p, _) in enumerate(rows)}
order = [p for p, _ in rows]
T.rng(5).shuffle(order)
got = Bzip2.decompressBlocks(z, order)
assert len(got) == len(order)
for p, b in zip(order, got):
    assert b == slices[p], p
print("ok", len(order))
"""


@gpu
@pytest.mark.parametrize("env", [{}, {"B2_DEC_BATCH": "7"}, {"B2_DEC_KEEP_CLS": "0"}])
def test_scale_all_positions_shuffled(env):
    """A level-1 stream of more than 2 x SM-count blocks, all positions shuffled in one call, equals the table's slices
    of decompressFile: by default, in decode batches of 7 blocks, and with the count-byte classes recomputed at expansion.
    A child process, because the library reads the hooks per call but the tests share it."""
    r = subprocess.run([sys.executable, "-c", _SCALE_SCRIPT % {"root": T.ROOT}], env=dict(os.environ, **env),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stdout + r.stderr[-3000:]


# ---- the C ABI -----------------------------------------------------------------------------------------------------
def _abi(z, poss, null_pos=False):
    from compressjs_b200 import _native
    L = _native.lib()
    a = np.array(poss, dtype=np.uint64)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t(77)
    ends, done = C.POINTER(C.c_uint64)(), C.c_size_t(77)
    rc = L.b2_bzip2_decompress_blocks(z, len(z), None if null_pos else (a.ctypes.data if a.size else None), len(poss),
                                      C.byref(out), C.byref(n), C.byref(ends), C.byref(done))
    if not out:
        return rc, None, None, None
    data = C.string_at(out, n.value)
    e = [ends[i] for i in range(done.value)]
    L.b2_free(out)
    L.b2_free(ends)
    return rc, data, e, done.value


@gpu
def test_c_abi_done_ends_and_out_n():
    from compressjs_b200 import _native
    data, z, tr = _mixed_level1()
    poss = [t.bit_start for t in tr]
    rc, out, ends, done = _abi(z, poss[::-1])
    assert rc == 0 and done == len(poss)
    exp = [data[t.raw_start:t.raw_start + t.raw_len] for t in tr[::-1]]
    assert ends == list(np.cumsum([len(b) for b in exp])) and out == b"".join(exp)
    # a CRC-only failure at position k: done == k, ends of the k before it, *out_n with the failing block's bytes
    k = 2
    bad = bytearray(z)
    bit = tr[k].bit_start + 48
    bad[bit // 8] ^= 0x80 >> (bit % 8)
    bad = bytes(bad)
    rc, out, ends, done = _abi(bad, poss)
    assert rc == W.DATA_ERROR and "Bad block CRC" in _native.last_error()
    assert done == k and ends == [tr[i].raw_start + tr[i].raw_len for i in range(k)]
    assert out == data[:tr[k].raw_start + tr[k].raw_len]
    # an error inside a block at position k: only the positions before it
    rc, out, ends, done = _abi(z, poss[:k] + [poss[k] + 3] + poss[k:])
    assert rc == W.NOT_BZIP and _native.last_error() == "Not bzip data"
    assert done == k and out == data[:tr[k].raw_start] and len(ends) == k


def _mixed_level1():
    from oracle import oracle as O
    data = T.ascii_random(150000, 11) + T.runs(150000, 12) + T.texty(200000, 13)
    z, tr = O.bzip2_compress(data, 1, trace=True)
    assert len(tr) >= 4
    return data, z, tr


def test_c_abi_empty_list_and_null_positions():
    """No position: nothing is decoded, not even a bad header.  Positions without an array: B2_ERR_BAD_ARG."""
    rc, out, ends, done = _abi(b"not a bzip2 file", [])
    assert (rc, out, ends, done) == (0, b"", [], 0)
    assert _abi(b"not a bzip2 file", [32], null_pos=True)[0] == -101


def test_python_empty_list_and_output_types():
    from compressjs_b200 import Bzip2
    assert Bzip2.decompressBlocks(b"BZh0 bad header", []) == []
    s = Sink()
    assert Bzip2.decompressBlocks(b"garbage", [], s) is s and s.buf == b""
    for out in (5, bytearray(5), np.zeros(5, np.uint8), True, "x"):
        with pytest.raises(TypeError) as e:
            Bzip2.decompressBlocks(b"garbage", [32], out)
        assert type(e.value) is TypeError   # raised before the library: not a Bzip2Error
