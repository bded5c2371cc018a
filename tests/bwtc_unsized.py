"""The BWTC stream compressjs writes for an input stream without a size (lib/Util.js:119-124: fileSize = -1, so the size
field is writeUnsignedNumber(0), the single group 0x80), obtained from the oracle's stream of the same input with its size.

The size field's last group is not written: it is the range coder's initial `buffer` (RangeCoder.js:66-72), which the
coder writes out once, as it is or plus a carry, at its first byte (:40-61, or :118-144 if no byte came out before).
`buffer` never enters `low` or `range`, so the two streams differ only there: "bwtc" + the written size groups + the
first coder byte become "bwtc" + 0x80 plus the same carry.  The oracle's decoder, which accepts a size field of 0,
checks every stream made here (`unsized` decodes it back)."""
from oracle import oracle as O


def unsized(data, level=9):
    z = O.bwtc_compress(data, level)
    v, groups = len(data) + 1, 1
    while v >= 128:
        v >>= 7
        groups += 1
    i = 4 + groups - 1                              # the coder's first byte, after the written size groups
    carry = (z[i] - (0x80 | ((len(data) + 1) & 0x7F))) & 0xFF
    assert carry in (0, 1), carry
    out = b"bwtc" + bytes([0x80 + carry]) + z[i + 1:]
    assert O.bwtc_decompress(out) == bytes(data)
    return out
