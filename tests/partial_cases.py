"""Synthetic streams whose decode fails after some output, for the tests of what a failed decode delivers first
(the reference writes every decoded byte as it goes, lib/Bzip2.js:405-448, and throws only after that).

Every corpus case (tests/synth_corpus.py) is taken as it is, and once more behind a good block with the CRC of its
first block that has an output flipped, so that the bytes of a block whose CRC fails are delivered.  The multistream
file is also taken behind a good member, and with its stream CRC flipped.

What the reference has delivered when it throws comes from two sides: the model of tests/bz2synth.py
(`expect_partial`, `expect_table_partial`: the walk of `File.expect` / `File.expect_table`, returning what it has
accumulated), and the CPU oracle's decoder with that output handed back (tests/host/bz2_partial_host.c, built on first
use into a temporary directory; `oracle_decompress`, `oracle_decompress_block`, `oracle_table`)."""
import atexit
import copy
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from tests import bz2synth as W
from tests import synth_corpus as SC
from tests import util as T


def with_crc(b, crc):
    """Block b with its stored CRC replaced (the model then expects its bytes, then a data error)."""
    c = copy.copy(b)
    c.bits = b.bits.copy()
    c.bits[48:80] = W.bits_of(crc, 32)
    c.crc = crc
    return c


def lead(level=9, seed=0):
    return W.from_content(SC.rand_bytes(700, 900 + seed, 97, 123), level=level)


def crc_flipped(f):
    """f's first member behind a good block, the first block with an output carrying a wrong CRC; None if none has one."""
    m = f.members[0]
    k = next((i for i, b in enumerate(m.blocks) if b.out is not None), None)
    if k is None:
        return None
    blocks = list(m.blocks)
    blocks[k] = with_crc(blocks[k], blocks[k].crc ^ 0x80000001)
    return W.File(W.Member([lead(m.level)] + blocks, m.level, level_byte=m.level_byte))


def files():
    """(name, File, multistream) of every case and variant."""
    out = []
    for name in sorted(SC.CASES):
        f = SC.build(name).file
        out.append((name, f, False))
        v = crc_flipped(f)
        if v is not None:
            out.append((name + "+crc", v, False))
    ms = SC.multistream_file()
    out.append(("multistream", ms, True))
    out.append(("multistream+crc", W.File([ms.members[0], crc_flipped(W.File(ms.members[1])).members[0]]), True))
    m1 = ms.members[1]
    out.append(("multistream+stream_crc", W.File([ms.members[0], W.Member(m1.blocks, m1.level, stream_crc=m1.stream_crc ^ 1)]), True))
    out.append(("multistream+level0", W.File([ms.members[0], W.Member(m1.blocks, m1.level, level_byte=ord("0"))]), True))
    return out


def block_expect(b):
    """decompressBlock of block b: ('ok', bytes) or ('err', code, bytes delivered before the error)."""
    if b.err is not None:
        return ("err", b.err, b"")
    if W.crc32(b.out) != b.crc:
        return ("err", W.DATA_ERROR, b.out)
    return ("ok", b.out)


# ---- the model ----------------------------------------------------------------------------------------------------
def expect_partial(f, multistream=False):
    """The bytes written in front of the error that f.expect(multistream) returns (all of them when it returns 'ok')."""
    out = []
    for m in f.members[: None if multistream else 1]:
        if not 1 <= m.level_byte - ord("0") <= 9:
            break
        for b in m.blocks:
            if b.err is not None:
                return b"".join(out)
            out.append(b.out)        # a block's bytes are written before its CRC is checked
            if W.crc32(b.out) != b.crc:
                return b"".join(out)
        if not m.crc_ok:
            break
    return b"".join(out)


def expect_table_partial(f):
    """The (bit position, size) rows reported in front of the error that f.expect_table() returns."""
    rows = []
    for pos, b in f.member_blocks[0]:
        if b.err is not None or W.crc32(b.out) != b.crc:
            break
        rows.append((pos, len(b.out)))
    return rows


# ---- the oracle ---------------------------------------------------------------------------------------------------
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="bz2partial")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libbz2partial.so")
        subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-pthread", "-fvisibility=hidden", "-w",
                               os.path.join(T.ROOT, "tests", "host", "bz2_partial_host.c"), "-o", so])
        L = C.CDLL(so)
        u8pp, szp = C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)
        L.part_bzip2_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, u8pp, szp]
        L.part_bzip2_decompress_block.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, u8pp, szp]
        L.part_bzip2_table.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.POINTER(C.c_uint64)),
                                       C.POINTER(C.POINTER(C.c_uint32)), szp]
        L.orc_free.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def _bytes_call(fn, data, arg):
    L = _lib()
    a = np.frombuffer(bytes(data), np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = fn(a.ctypes.data if a.size else None, a.size, arg, C.byref(out), C.byref(n))
    res = C.string_at(out, n.value) if n.value else b""
    L.orc_free(out)
    return ("err", rc, res) if rc else ("ok", res)


def oracle_decompress(data, multistream=False):
    """('ok', bytes) or ('err', code, the bytes written before the error)."""
    return _bytes_call(_lib().part_bzip2_decompress, data, int(multistream))


def oracle_decompress_block(data, pos):
    return _bytes_call(_lib().part_bzip2_decompress_block, data, int(pos))


def oracle_table(data, multistream=False):
    """('ok', rows) or ('err', code, the rows reported before the error)."""
    L = _lib()
    a = np.frombuffer(bytes(data), np.uint8)
    bp, sz, cnt = C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint32)(), C.c_size_t()
    rc = L.part_bzip2_table(a.ctypes.data if a.size else None, a.size, int(multistream), C.byref(bp), C.byref(sz), C.byref(cnt))
    rows = [(int(bp[i]), int(sz[i])) for i in range(cnt.value)]
    L.orc_free(bp)
    L.orc_free(sz)
    return ("err", rc, rows) if rc else ("ok", rows)
