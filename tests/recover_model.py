"""Model of block recovery (include/b2bz.h b2_bzip2_recover), for the tests of the GPU recovery.

It follows the definition the C ABI states, from two independent parts:
  - candidates: every 48-bit block magic at any bit position, from a plain numpy scan of the bytes;
  - decodes: the CPU oracle's decompressBlock of B = b"BZh9" + input at p + 32 (decode_block: oracle/bz2_oracle.c,
    included unchanged by tests/host/bz2_recover_host.c, which also hands back the bit behind the end-of-block code and
    the CRC of the bytes it decoded).
The walk keeps `end` (0 at first): a candidate with p < end is INSIDE, any other is decoded and is INTACT when that
raises nothing (end moves behind it), else BAD_CRC ("Bad block CRC"), OBSOLETE (-7) or DATA_ERROR.  The recovered bytes
are the INTACT blocks' bytes in position order; the repaired stream is "BZh9", the bits [p, endbit) of every intact
block, the end-of-stream magic, the combined CRC (crc = rotl1(crc) ^ stored CRC) and zero bits to the next byte."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from collections import namedtuple

import numpy as np

from tests import util as T

BLOCK_MAGIC = 0x314159265359
EOS_MAGIC = 0x177245385090
INTACT, BAD_CRC, DATA_ERROR, OBSOLETE, INSIDE = "INTACT", "BAD_CRC", "DATA_ERROR", "OBSOLETE", "INSIDE"

# the fields of b2_recovered_block / Bzip2.recover's rows
Row = namedtuple("Row", "bitpos endbit out_off size crc got status")
Recovery = namedtuple("Recovery", "rows data stream")


_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="bz2recover")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libbz2recover.so")
        subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-pthread", "-fvisibility=hidden", "-w",
                               os.path.join(T.ROOT, "tests", "host", "bz2_recover_host.c"), "-o", so])
        L = C.CDLL(so)
        L.rec_bzip2_decompress_block.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.POINTER(C.POINTER(C.c_uint8)),
                                                 C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.orc_last_error.restype = C.c_char_p
        L.orc_free.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def decode_block(B, bitpos):
    """The oracle's decompressBlock of B at bitpos: (code, message, bytes, endbit, got).  bytes, endbit (the bit behind
    the end-of-block code) and got (the CRC of the bytes) are set when the block decoded up to its CRC check, whether
    that passed (code 0) or not; otherwise they are b"", 0, 0."""
    L = _lib()
    a = np.frombuffer(bytes(B), np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    endbit, got = C.c_uint64(), C.c_uint32()
    rc = L.rec_bzip2_decompress_block(a.ctypes.data if a.size else None, a.size, bitpos, C.byref(out), C.byref(n),
                                      C.byref(endbit), C.byref(got))
    msg = L.orc_last_error().decode() if rc else ""
    res = C.string_at(out, n.value) if n.value else b""
    L.orc_free(out)
    return rc, msg, res, int(endbit.value), int(got.value)


def candidates(data):
    """Bit positions of every block magic that lies wholly inside data, in order."""
    a = np.frombuffer(bytes(data), np.uint8)
    n = a.size
    if n < 6:
        return []
    pad = np.concatenate([a, np.zeros(7, np.uint8)]).astype(np.uint64)
    v = np.zeros(n, np.uint64)
    for k in range(7):   # v[i] = the 56 bits from byte i on
        v = (v << np.uint64(8)) | pad[k:k + n]
    found = []
    for ph in range(8):
        w = (v >> np.uint64(8 - ph)) & np.uint64((1 << 48) - 1)
        found += [8 * int(i) + ph for i in np.nonzero(w == np.uint64(BLOCK_MAGIC))[0]]
    return sorted(p for p in found if p + 48 <= 8 * n)


def bits_at(data, pos, k):
    """The k bits of data from bit pos on (bits past the end read as zeros)."""
    b = bytes(data[pos // 8:(pos + k + 7) // 8 + 1]).ljust((pos % 8 + k + 7) // 8 + 1, b"\0")
    return (int.from_bytes(b, "big") >> (8 * len(b) - pos % 8 - k)) & ((1 << k) - 1)


def rotl1(v):
    return ((v << 1) | (v >> 31)) & 0xFFFFFFFF


def walk(data):
    """The rows of every candidate and the bytes of the intact ones: (rows, [(bitpos, endbit, bytes) of the intact])."""
    data = bytes(data)
    B = b"BZh9" + data
    rows, intact = [], []
    end = total = 0
    for p in candidates(data):
        stored = bits_at(data, p + 48, 32)
        if p < end:
            rows.append(Row(p, 0, total, 0, stored, 0, INSIDE))
            continue
        rc, msg, out, eb, got = decode_block(B, p + 32)
        if rc == 0 or "Bad block CRC" in msg:
            st = INTACT if rc == 0 else BAD_CRC
            rows.append(Row(p, eb - 32, total, len(out), stored, got, st))
            if st == INTACT:
                intact.append((p, eb - 32, out))
                end = eb - 32
                total += len(out)
        else:
            rows.append(Row(p, 0, total, 0, stored, 0, OBSOLETE if rc == -7 else DATA_ERROR))
    return rows, intact


def repaired_stream(data, intact):
    """"BZh9", the intact blocks' bits back to back, the end-of-stream magic, the combined CRC, zero bits to a byte."""
    bits = np.unpackbits(np.frombuffer(bytes(data), np.uint8))
    parts = [np.unpackbits(np.frombuffer(b"BZh9", np.uint8))]
    crc = 0
    for p, e, _ in intact:
        parts.append(bits[p:e])
        crc = rotl1(crc) ^ bits_at(data, p + 48, 32)
    tail = (EOS_MAGIC << 32) | crc
    parts.append(np.array([(tail >> (79 - i)) & 1 for i in range(80)], np.uint8))
    return np.packbits(np.concatenate(parts)).tobytes()


def recover(data):
    """Recovery(rows, recovered bytes, repaired stream) of data."""
    rows, intact = walk(data)
    return Recovery(rows, b"".join(o for _, _, o in intact), repaired_stream(data, intact))


def libbz2_language(data, rows):
    """False when an intact block is outside libbz2's language: its bytes end on four equal bytes without a count byte
    (a compressjs block can; libbz2 rejects it).  The block's RLE1 bytes are not kept, so this is judged from the
    decoded bytes: a block whose bytes end on four or more equal bytes is taken as possibly outside."""
    B = b"BZh9" + bytes(data)
    for r in rows:
        if r.status == INTACT:
            out = decode_block(B, r.bitpos + 32)[2]
            if len(out) >= 4 and len(set(out[-4:])) == 1:
                return False
    return True
