"""Damage corpus of the block recovery tests: each case is a seeded input and the condition it is named for, which
`check` asserts through the model's rows (tests/recover_model.py).  cases() -> [Case]."""
import bz2
import functools
from collections import namedtuple

import numpy as np

from oracle import oracle as O
from tests import bz2synth as W
from tests import recover_model as M
from tests import util as T

Case = namedtuple("Case", "name data check")


def flip(data, bit):
    b = bytearray(data)
    b[bit // 8] ^= 0x80 >> (bit % 8)
    return bytes(b)


def statuses(rows):
    return [r.status for r in rows]


def three(level=1, seed=1, n=330000):
    """bz2.compress of seeded text: four blocks at level 1."""
    return bz2.compress(T.texty(n, seed), level)


def _huffman_flip(want, seed):
    """A flipped bit in the second half of block 1 of three() whose model status is `want`."""
    z = three()
    c = M.candidates(z)
    g = T.rng(seed)
    for _ in range(400):
        bit = int(g.integers(c[1] + (c[2] - c[1]) // 2, c[2] - 8))
        d = flip(z, bit)
        if M.walk(d)[0][1].status == want:
            return d
    raise AssertionError("no flip gives " + want)


def _insert_bits(z, seed):
    """The blocks of z with 8 k bytes and a few bits of seeded garbage in front of block k (k >= 1), so that block k
    starts at bit phase k mod 8."""
    bits = np.unpackbits(np.frombuffer(z, np.uint8))
    c = M.candidates(z)
    g = T.rng(seed)
    parts, prev, shift = [], 0, 0
    for k, p in enumerate(c[1:], 1):
        parts.append(bits[prev:p])
        gap = 64 * k + (k - (p + shift)) % 8
        parts.append(g.integers(0, 2, size=gap, dtype=np.uint8))
        shift += gap
        prev = p
    parts.append(bits[prev:])
    return np.packbits(np.concatenate(parts)).tobytes()


def _plant_block(k, seed, crc_flip=0):
    """A synthetic block whose Huffman data holds a block magic pattern (tests/bz2synth.py), in a BZh9 stream with a good
    block behind it; its stored CRC xor crc_flip."""
    used = list(range(1, 254))
    lens = [8] * (len(used) + 2)
    lens[2] = 7
    eob = len(used) + 1
    g = T.rng(seed)
    syms = [2] * k + W.decode_bits("{:048b}".format(W.BLOCK_MAGIC), lens, avoid={0, 1, eob})
    syms += [int(x) for x in g.integers(2, eob, size=30)] + [eob]
    b = W.block(syms, used, 3, lens=[lens, lens])
    if crc_flip:
        b.bits = b.bits.copy()
        b.crc ^= crc_flip
        b.bits[48:80] = W.bits_of(b.crc, 32)
    return W.File(W.Member([b, W.from_content(T.ascii_random(3000, seed))])).data


def _obsolete():
    z = three()
    return flip(z, M.candidates(z)[2] + 80)   # the randomised bit behind the block CRC


def _no_intact():
    g = T.rng(5)
    junk = bytearray(g.integers(0, 256, size=4000, dtype=np.uint8).tobytes())
    junk[1000:1006] = W.BLOCK_MAGIC.to_bytes(6, "big")
    junk[2500:2506] = W.BLOCK_MAGIC.to_bytes(6, "big")
    return bytes(junk)


def _check_all_intact(rows):
    assert rows and all(s == M.INTACT for s in statuses(rows)), statuses(rows)


def _members(levels, seed):
    return b"".join(bz2.compress(T.texty(150000 + 20000 * i, seed + i), lv) for i, lv in enumerate(levels))


@functools.lru_cache(maxsize=None)
def cases():
    cs = []

    def add(name, data, check):
        cs.append(Case(name, data, check))

    def huff_data_error(rows):
        assert statuses(rows) == [M.INTACT, M.DATA_ERROR, M.INTACT, M.INTACT], statuses(rows)
    add("huffman_flip_data_error", _huffman_flip(M.DATA_ERROR, 11), huff_data_error)

    def huff_bad_crc(rows):
        assert statuses(rows) == [M.INTACT, M.BAD_CRC, M.INTACT, M.INTACT], statuses(rows)
    add("huffman_flip_bad_crc", _huffman_flip(M.BAD_CRC, 12), huff_bad_crc)

    z = three()
    c = M.candidates(z)
    add("stored_crc_flip", flip(z, c[2] + 60), lambda rows: statuses(rows) == [M.INTACT, M.INTACT, M.BAD_CRC, M.INTACT] or _fail(rows))

    def magic_damaged(rows):
        # block 2's magic is gone: blocks 1, 3 and 4 (the block in front of the damage too) are intact
        assert [r.bitpos for r in rows] == [c[0], c[1], c[3]] and all(r.status == M.INTACT for r in rows), rows
    add("block_magic_damaged", flip(z, c[2] + 20), magic_damaged)

    eos = W.magic_positions(z)[1][0]
    add("eos_magic_damaged", flip(z, eos + 10), _check_all_intact)
    add("first_header_damaged", b"\0\0\0\0" + z[4:], _check_all_intact)

    def truncated(rows):
        assert statuses(rows) == [M.INTACT] * 3 + [M.DATA_ERROR], statuses(rows)
    add("truncated_last_block", z[:(c[3] + (len(z) * 8 - c[3]) // 2) // 8], truncated)

    def zero_span(rows):
        assert c[2] not in [r.bitpos for r in rows] and rows[1].status != M.INTACT and rows[0].status == M.INTACT, rows
    zs = bytearray(z)
    zs[c[2] // 8 - 200:c[2] // 8 + 200] = bytes(400)
    add("zeroed_span_across_edge", bytes(zs), zero_span)

    z9 = bz2.compress(T.texty(900000, 3), 1)   # nine blocks or more
    shifted = _insert_bits(z9, 4)

    def shifted_check(rows):
        _check_all_intact(rows)
        assert len(rows) >= 9 and {r.bitpos % 8 for r in rows[1:]} == set(range(8)), [r.bitpos % 8 for r in rows]
    add("garbage_between_blocks", shifted, shifted_check)

    ms = _members([9, 9, 9], 20)
    mc = [p for p in M.candidates(ms)]
    hdr = ms.index(b"BZh9", 10)
    add("multistream_member_header_damaged", ms[:hdr] + b"XXXX" + ms[hdr + 4:], lambda rows: len(rows) == len(mc) and _check_all_intact(rows) is None)
    add("multistream_levels_1_9", _members([1, 9, 1], 30), _check_all_intact)

    def planted_inside(rows):
        assert statuses(rows) == [M.INTACT, M.INSIDE, M.INTACT], statuses(rows)
    add("planted_inside_intact", _plant_block(40, 7), planted_inside)

    def planted_bad(rows):
        assert rows[0].status == M.BAD_CRC and rows[1].status != M.INSIDE and rows[-1].status == M.INTACT, statuses(rows)
    add("planted_inside_bad_crc", _plant_block(40, 8, 0x80000001), planted_bad)

    big = bz2.compress(T.ascii_random(400000, 6), 9)

    def big_check(rows):
        assert statuses(rows) == [M.INTACT] and rows[0].size > 100000, rows
    add("bzh1_block_over_100k", big[:3] + b"1" + big[4:], big_check)

    def obsolete(rows):
        assert statuses(rows) == [M.INTACT, M.INTACT, M.OBSOLETE, M.INTACT], statuses(rows)
    add("randomised_bit", _obsolete(), obsolete)

    def none_intact(rows):
        assert len(rows) == 2 and M.INTACT not in statuses(rows), rows
    add("no_intact_block", _no_intact(), none_intact)

    def no_rows(rows):
        assert rows == [], rows
    add("empty_input", b"", no_rows)
    add("not_bzip2", T.ascii_random(5000, 9), no_rows)
    add("undamaged_l1", three(), _check_all_intact)
    add("undamaged_l9", bz2.compress(T.texty(1200000, 2), 9), _check_all_intact)
    add("undamaged_compressjs", O.bzip2_compress(T.texty(250000, 4) + b"abcd" * 3 + b"zzzz", 1), _check_all_intact)
    return tuple(cs)


def _fail(rows):
    raise AssertionError(statuses(rows))


@functools.lru_cache(maxsize=None)
def by_name():
    return {c.name: c for c in cases()}
