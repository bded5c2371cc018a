"""ctypes binding of oracle/liboracle.so -- the CPU restatement of the reference path.

TEST INFRASTRUCTURE ONLY.  Imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never by compressjs_b200 (the product).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("bz2_oracle.c", "bwtc_oracle.c")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B", "liboracle.so"])
    return so


class BlockTrace(C.Structure):
    _fields_ = [("n", C.c_int32), ("pidx", C.c_int32), ("m", C.c_int32), ("alpha", C.c_int32),
                ("ngroups", C.c_int32), ("nsel", C.c_int32), ("crc", C.c_uint32), ("pad", C.c_uint32),
                ("raw_start", C.c_uint64), ("raw_len", C.c_uint64), ("bit_start", C.c_uint64),
                ("bit_len", C.c_uint64)]


class BwtcBlockTrace(C.Structure):
    """orc_bwtc_block_t (bwtc_oracle.c): counters of one block of orc_bwtc_compress_trace."""
    _fields_ = [(f, C.c_uint32) for f in ("n", "alpha", "nsym", "ntriples", "rescales", "rescales_esc", "rescales_ff00",
                                          "rescales_noesc", "escapes", "last_escape", "reescapes", "esc_lane31",
                                          "ds_rebuilds", "ds_esc_cap", "max_tot", "carries", "help_carry", "help_nocarry")] + \
        [("corr", C.c_uint32 * 3), ("max_help", C.c_uint32), ("help_in", C.c_uint32), ("resolved_in", C.c_uint32),
         ("help", C.c_uint64), ("bytes_out", C.c_uint64),
         ("bytecount", C.c_uint64)]


class BwtcFileTrace(C.Structure):
    """orc_bwtc_file_t (bwtc_oracle.c)."""
    _fields_ = [(f, C.c_uint32) for f in ("nblocks", "max_help", "first_carry", "finish_carry", "finish_round", "corr2")] + \
        [("coder_bytes", C.c_uint64), ("bytecount", C.c_uint64)]


def lib():
    global _LIB
    if _LIB is None:
        so = build()
        L = C.CDLL(so)
        u8p, szp = C.POINTER(C.c_uint8), C.POINTER(C.c_size_t)
        L.orc_last_error.restype = C.c_char_p
        L.orc_crc32.restype = C.c_uint32
        L.orc_crc32.argtypes = [C.c_void_p, C.c_size_t]
        L.orc_bwt_cyclic.restype = C.c_int32
        L.orc_bwt_cyclic.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.orc_bwt_sentinel.restype = C.c_int32
        L.orc_bwt_sentinel.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.orc_unbwt_sentinel.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        L.orc_suffixsort.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.orc_huffman_code_lengths.restype = None
        L.orc_huffman_code_lengths.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.orc_bzip2_compress_ex.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(u8p), szp,
                                            C.c_void_p, C.c_size_t, szp]
        L.orc_bzip2_compress_mt.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(u8p), szp]
        L.orc_bzip2_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(u8p), szp]
        L.orc_bzip2_decompress_block.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.POINTER(u8p), szp]
        L.orc_bzip2_table.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.POINTER(C.c_uint64)),
                                      C.POINTER(C.POINTER(C.c_uint32)), szp]
        L.orc_rle1_split.restype = C.c_size_t
        L.orc_rle1_split.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_size_t, C.c_void_p, C.c_size_t]
        L.orc_compress_block_stages.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.POINTER(u8p), szp]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_bwtc_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(u8p), szp]
        L.orc_bwtc_decompress.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(u8p), szp]
        L.orc_bwtc_compress_trace.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(u8p), szp, C.c_void_p, C.c_size_t,
                                              C.POINTER(BwtcFileTrace)]
        _LIB = L
    return _LIB


class OracleError(Exception):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.errorCode = code


def _buf(data):
    a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)
    return a, a.ctypes.data if a.size else None


def _take(L, p, n):
    out = C.string_at(p, n.value) if n.value else b""
    L.orc_free(p)
    return out


def crc32(data):
    a, p = _buf(data)
    return lib().orc_crc32(p, a.size)


def bwt_cyclic(data):
    a, p = _buf(data)
    u = np.empty(max(a.size, 1), dtype=np.uint8)
    pidx = lib().orc_bwt_cyclic(p, u.ctypes.data, a.size)
    return u[:a.size].tobytes(), pidx


def bwt_sentinel(data):
    a, p = _buf(data)
    u = np.empty(max(a.size, 1), dtype=np.uint8)
    pidx = lib().orc_bwt_sentinel(p, u.ctypes.data, a.size)
    return u[:a.size].tobytes(), pidx


def unbwt_sentinel(data, pidx):
    a, p = _buf(data)
    u = np.empty(max(a.size, 1), dtype=np.uint8)
    lib().orc_unbwt_sentinel(p, u.ctypes.data, a.size, pidx)
    return u[:a.size].tobytes()


def suffixsort(data):
    a, p = _buf(data)
    sa = np.empty(max(a.size, 1), dtype=np.int32)
    lib().orc_suffixsort(p, sa.ctypes.data, a.size)
    return sa[:a.size]


def huffman_code_lengths(freqs, maxlen):
    arr = np.array(freqs, dtype=np.int32)
    lib().orc_huffman_code_lengths(arr.ctypes.data, arr.size, maxlen)
    return arr.tolist()


def block_cap(n, level):
    """Upper bound on the number of blocks of an n-byte input: a block holds at least 4/5 of blockSize raw bytes
    (runs of exactly four give 5 RLE1 bytes per 4 raw bytes), the last one may be short."""
    bs = max(level * 100000 - 19, 1)
    return n // max(bs * 4 // 5, 1) + 2


def bzip2_compress(data, level=9, legacy_sort=False, trace=False, threads=0):
    L = lib()
    a, p = _buf(data)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    if threads and not trace and not legacy_sort:
        rc = L.orc_bzip2_compress_mt(p, a.size, level, threads, C.byref(out), C.byref(n))
        if rc:
            raise OracleError(rc, "more blocks than the block arrays hold" if rc == -101 else "Invalid block size multiplier")
        return _take(L, out, n)
    cap = block_cap(a.size, level)
    tr = (BlockTrace * cap)()
    nt = C.c_size_t()
    rc = L.orc_bzip2_compress_ex(p, a.size, level, int(legacy_sort), C.byref(out), C.byref(n), tr, cap, C.byref(nt))
    if rc:
        raise OracleError(rc, L.orc_last_error().decode())
    res = _take(L, out, n)
    if trace:
        return res, [tr[i] for i in range(nt.value)]
    return res


def bzip2_decompress(data, multistream=False):
    L = lib()
    a, p = _buf(data)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = L.orc_bzip2_decompress(p, a.size, int(multistream), C.byref(out), C.byref(n))
    if rc:
        raise OracleError(rc, L.orc_last_error().decode())
    return _take(L, out, n)


def bzip2_decompress_block(data, bitpos):
    L = lib()
    a, p = _buf(data)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = L.orc_bzip2_decompress_block(p, a.size, bitpos, C.byref(out), C.byref(n))
    if rc:
        raise OracleError(rc, L.orc_last_error().decode())
    return _take(L, out, n)


def bzip2_table(data, multistream=False):
    L = lib()
    a, p = _buf(data)
    bp, sz, cnt = C.POINTER(C.c_uint64)(), C.POINTER(C.c_uint32)(), C.c_size_t()
    rc = L.orc_bzip2_table(p, a.size, int(multistream), C.byref(bp), C.byref(sz), C.byref(cnt))
    if rc:
        raise OracleError(rc, L.orc_last_error().decode())
    res = [(int(bp[i]), int(sz[i])) for i in range(cnt.value)]
    L.orc_free(bp)
    L.orc_free(sz)
    return res


def rle1_split(data, level=9, stride=None):
    """Returns (raw_starts, lens, crcs, blocks[nb, stride])."""
    L = lib()
    a, p = _buf(data)
    stride = stride or level * 100000
    cap = block_cap(a.size, level)
    starts = np.zeros(cap, dtype=np.uint64)
    lens = np.zeros(cap, dtype=np.uint32)
    crcs = np.zeros(cap, dtype=np.uint32)
    blocks = np.zeros((cap, stride), dtype=np.uint8)
    nb = L.orc_rle1_split(p, a.size, level, starts.ctypes.data, lens.ctypes.data, crcs.ctypes.data, cap,
                          blocks.ctypes.data, stride)
    return starts[:nb], lens[:nb], crcs[:nb], blocks[:nb]


def compress_block_stages(block, legacy_sort=False):
    """One post-RLE1 block -> dict(trace, sym, sel, lens, bits, nbits)."""
    L = lib()
    a, p = _buf(block)
    n = a.size
    tr = BlockTrace()
    sym = np.zeros(n + 2, dtype=np.uint16)
    sel = np.zeros((n + 1) // 50 + 2, dtype=np.uint8)
    lens = np.zeros(6 * 258, dtype=np.uint8)
    out, nbits = C.POINTER(C.c_uint8)(), C.c_size_t()
    L.orc_compress_block_stages(p, n, int(legacy_sort), C.byref(tr), sym.ctypes.data, sel.ctypes.data,
                                lens.ctypes.data, C.byref(out), C.byref(nbits))
    nb = C.c_size_t((nbits.value + 7) // 8)
    bits = _take(L, out, nb)
    return dict(trace=tr, sym=sym[:tr.m].copy(), sel=sel[:tr.nsel].copy(),
                lens=lens.reshape(6, 258)[:tr.ngroups, :tr.alpha + 2].copy(), bits=bits, nbits=nbits.value)


def bwtc_compress(data, level=9, trace=False):
    """BWTC.compressFile (lib/BWTC.js:12-139).  With `trace`: (stream, [BwtcBlockTrace per block], BwtcFileTrace)."""
    L = lib()
    a, p = _buf(data)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    if trace:
        bs = (level if 1 <= level <= 9 else 9) * 100000
        cap = a.size // bs + 1
        tr, ft = (BwtcBlockTrace * cap)(), BwtcFileTrace()
        rc = L.orc_bwtc_compress_trace(p, a.size, level, C.byref(out), C.byref(n), tr, cap, C.byref(ft))
    else:
        rc = L.orc_bwtc_compress(p, a.size, level, C.byref(out), C.byref(n))
    if rc:
        raise OracleError(rc, "bwtc compress failed")
    if trace:
        return _take(L, out, n), [tr[i] for i in range(ft.nblocks)], ft
    return _take(L, out, n)


def bwtc_decompress(data):
    """BWTC.decompressFile (lib/BWTC.js:141-231)."""
    L = lib()
    a, p = _buf(data)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = L.orc_bwtc_decompress(p, a.size, C.byref(out), C.byref(n))
    if rc:
        raise OracleError(rc, "Bad magic" if rc == -2 else "bwtc decompress failed")
    return _take(L, out, n)
