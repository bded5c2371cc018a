"""Streams that the two bzip2 decoder flavors read differently (include/b2bz.h, b2_bzip2_decompress_flavor R1-R5),
built with the writer of tests/bz2synth.py, and a plain model of the libbz2 flavor on top of the writer's expectations.

A randomised block (R1) is written as `from_content(B ^ mask, rand=1, crc=crc32(rle1_decode(B)))`: its column is the
BWT of the masked bytes, so a decoder that does not derandomise gets other bytes and fails the CRC.  Every case names
its conditions and computes them from the writer's report, as tests/synth_corpus.py does.

`model(file, multistream)` gives what the libbz2 flavor returns: ("ok", bytes) or ("err", code, prefix).
"""
import functools
import hashlib
import os
import re
import struct

import numpy as np

from tests import bz2synth as W
from tests import synth_corpus as SC
from tests import util as T

EOF_ERR = -3
RNUMS_SHA256 = "fa6f7d5596f6084ee582060b76239c49c1bf8567f7ea556e2d83971c75e26951"
DECODE_CU = os.path.join(T.ROOT, "compressjs_b200", "csrc", "decode.cu")


@functools.lru_cache(maxsize=None)
def rnums():
    """libbz2's BZ2_rNums as the CUDA source holds it, checked against its SHA-256."""
    src = open(DECODE_CU).read()
    body = re.search(r"RNUMS\[512\] = \{(.*?)\};", src, re.S).group(1)
    t = [int(x) for x in body.replace("\n", " ").split(",")]
    assert len(t) == 512 and hashlib.sha256(struct.pack("<512i", *t)).hexdigest() == RNUMS_SHA256
    return t


@functools.lru_cache(maxsize=None)
def flips():
    """Positions below 900 000 that libbz2 XORs with 1 in a randomised block."""
    out, togo, t = [], 0, 0
    r = rnums()
    for i in range(900000):
        if togo == 0:
            togo, t = r[t], (t + 1) % 512
        togo -= 1
        if togo == 1:
            out.append(i)
    return np.array(out, np.int64)


def mask(n):
    m = np.zeros(n, np.uint8)
    f = flips()
    m[f[f < n]] = 1
    return m


def rand_block(P):
    """A randomised block whose bytes before RLE1 decoding are P once derandomised."""
    P = np.frombuffer(bytes(P), np.uint8)
    out, _, _ = W.model_rle1(P)
    b = W.from_content((P ^ mask(P.size)).tobytes(), rand=1, crc=W.crc32(out))
    b.P = P
    return b


# ---- the model -------------------------------------------------------------------------------------------------
def block_verdict(b):
    """(code, bytes) of one block in the libbz2 flavor: code 0 ok, else the error; bytes: what goes out (a block that
    fails only its CRC delivers its bytes)."""
    failed = list(b.failed)
    if failed and failed[0] == "randomised block":
        failed = failed[1:]
        if failed:
            return W.DATA_ERROR, b""
    elif b.err is not None:
        return b.err, b""
    if len(b.lens) in b.sel_mtf:   # R2
        return W.DATA_ERROR, b""
    B = np.asarray(b.report["B"], np.uint8)
    P = B ^ mask(B.size) if b.bits[80] else B
    out, _, pending = W.model_rle1(P)
    if pending:                    # R3
        return W.DATA_ERROR, b""
    out = out.tobytes()
    return (0 if W.crc32(out) == b.crc else W.DATA_ERROR), out


def _groups_agree(bits, pos):
    """R4 at bit pos: the input's whole bytes from pos on agree with the start of a block or end-of-stream magic."""
    k = min((bits.size - pos) // 8, 6) if bits.size > pos else 0
    got = bits[pos:pos + 8 * k]
    return any(np.array_equal(got, W.bits_of(m, 48)[:8 * k]) for m in (W.BLOCK_MAGIC, W.EOS_MAGIC))


def model(f, multistream=True, cut=None, tail=b""):
    """The libbz2 flavor on File f's bytes, cut to `cut` bytes, with `tail` behind: ("ok", bytes) or
    ("err", code, prefix)."""
    data = (f.data + tail)[:cut]
    bits = np.unpackbits(np.frombuffer(data, np.uint8))
    nb = bits.size
    out = []
    off = 0
    for mi, m in enumerate(f.members):
        if mi:
            rest = data[off:]
            if not rest:
                break
            want = b"BZh"
            head = rest[:4]
            if not all(head[k] == want[k] if k < 3 else 0x31 <= head[k] <= 0x39 for k in range(len(head))):
                break
            if len(head) < 4:
                return ("err", EOF_ERR, b"".join(out))
        if nb < off * 8 + 32:
            return ("err", W.NOT_BZIP, b"")
        if not 1 <= m.level_byte - 0x30 <= 9:
            return ("err", W.NOT_BZIP, b"".join(out))
        for p, b in zip(m.block_pos, m.blocks):
            p += off * 8
            if p + 80 > nb and _groups_agree(bits, p):
                return ("err", EOF_ERR, b"".join(out))
            if p + b.bits.size > nb:   # cut inside the block
                return ("err", W.DATA_ERROR, b"".join(out))
            code, o = block_verdict(b)
            if code:
                return ("err", code, b"".join(out) + o)
            out.append(o)
        e = off * 8 + m.eos_pos
        if e + 80 > nb and _groups_agree(bits, e):
            return ("err", EOF_ERR, b"".join(out))
        if not m.crc_ok:
            return ("err", W.DATA_ERROR, b"".join(out))
        off += len(m.data)
        if not multistream:
            break
    tail_after = data[off:]
    if multistream and off == len(f.data) and tail_after:
        head = tail_after[:4]
        if all(head[k] == b"BZh"[k] if k < 3 else 0x31 <= head[k] <= 0x39 for k in range(len(head))):
            if len(head) < 4:
                return ("err", EOF_ERR, b"".join(out))
            return ("err", EOF_ERR if len(tail_after) == 4 else W.NOT_BZIP, b"".join(out))
    return ("ok", b"".join(out))


# ---- cases -----------------------------------------------------------------------------------------------------
class Case:
    """f: a bz2synth File; cut: keep this many bytes; tail: bytes written behind; cond: the conditions it names."""

    def __init__(self, f, cond, cut=None, tail=b""):
        self.f, self.cond, self.cut, self.tail = f, cond, cut, tail

    @property
    def data(self):
        return (self.f.data + self.tail)[:self.cut]

    def expect(self, multistream=True):
        return model(self.f, multistream, self.cut, self.tail)


CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


@functools.lru_cache(maxsize=None)
def build(name):
    return CASES[name]()


def one(*blocks, **kw):
    return W.File(W.Member(list(blocks), 9, **kw))


def _literals(n, seed):
    """Bytes without two equal neighbours, from 'A'..'Z'."""
    a = T.rng(seed).integers(65, 91, size=n, dtype=np.uint8)
    for i in range(1, n):
        if a[i] == a[i - 1]:
            a[i] = 65 + (a[i] - 64) % 26
    return a


def _rle_ok(P):
    return not W.rle1_classes(np.asarray(P, np.uint8))[1]


# R1
@case
def rand_short():
    b = rand_block(T.ascii_random(600, 1))
    return Case(one(b), dict(no_flip=b.P.size <= flips()[0], rand=True))


@case
def rand_count_flips():
    P = _literals(3000, 2)
    f = flips()[flips() < 3000]
    for x in f:
        P[x - 4:x] = ord("q")
        P[x] = 7
        P[x + 1] = ord("r")
    cls = W.rle1_classes(P)[0]
    b = rand_block(P)
    return Case(one(b), dict(count_flipped=bool(all(cls[f])), flips=len(f) >= 2))


@case
def rand_make_break_run4():
    P = _literals(3000, 3)
    f = flips()[flips() < 3000]
    P[f[0] - 3:f[0] + 1] = ord("m")         # derandomised: a run of four (its count byte behind)
    P[f[0] + 1] = 2
    P[f[1] - 3:f[1]] = ord("k")             # stored: a run of four; derandomised: three and another byte
    P[f[1]] = ord("k") ^ 1
    stored = P ^ mask(P.size)
    c_p, c_s = W.rle1_classes(P)[0], W.rle1_classes(stored)[0]
    b = rand_block(P)
    return Case(one(b), dict(made=bool(c_p[f[0] + 1] and not c_s[f[0] + 1]), broken=bool(c_s[f[1] + 1] and not c_p[f[1] + 1])))


@case
def rand_flip_last_byte():
    n = int(flips()[1]) + 1
    b = rand_block(_literals(n, 4))
    return Case(one(b), dict(last_flipped=int(flips()[1]) == n - 1))


@case
def rand_granule_tile():
    """Count bytes flipped at both ends of 8-byte classify granules, and a run of four across a 2048-byte tile seam that
    the flip on its fourth byte makes.  No flip below 900 000 lies at 2047, 0 or 1 mod 2048 (so none is a tile's first
    or last byte); the one at 645 122 (2 mod 2048) is the only flip whose run of four can straddle a seam."""
    n = 650000
    P = _literals(n, 5)
    f = flips()[flips() < n - 2]
    at = [int(x) for x in f if x % 8 in (0, 7)][:8]
    for x in at:
        P[x - 4:x] = ord("z")
        P[x] = 3
        P[x + 1] = ord("y")
    seam = [int(x) for x in f if min(x % 2048, 2048 - x % 2048) <= 3]
    x = seam[0]
    P[x - 3:x + 1] = ord("s")                 # derandomised: a run of four across the seam, its count byte behind
    P[x + 1] = 4
    stored = P ^ mask(n)
    c_p, c_s = W.rle1_classes(P)[0], W.rle1_classes(stored)[0]
    b = rand_block(P)
    return Case(one(b), dict(granule=any(x % 8 == 0 for x in at) and any(x % 8 == 7 for x in at), counts=bool(all(c_p[at])),
                             no_flip_on_tile_edge=not any(v % 2048 in (0, 1, 2047) for v in flips().tolist()),
                             seam_run=seam == [645122] and (x - 3) // 2048 != x // 2048,
                             seam_run_made=bool(c_p[x + 1] and not c_s[x + 1])))


@case
def rand_wraps():
    b = rand_block(T.ascii_random(300000, 6))
    return Case(one(b), dict(wraps=b.P.size > 278212))


@case
def rand_full_block():
    P = np.frombuffer(T.ascii_random(900000, 7), np.uint8)
    b = rand_block(P)
    return Case(one(b), dict(full=b.P.size == 900000, flips=int((flips() < 900000).sum()) == 1655))


@case
def rand_mixed_members():
    r1, r2 = rand_block(T.ascii_random(5000, 8)), rand_block(T.ascii_random(7000, 9))
    p1, p2 = W.from_content(T.ascii_random(4000, 10)), W.from_content(T.ascii_random(3000, 11))
    f = W.File([W.Member([r1, p1], 9), W.Member([p2, r2], 5)])
    return Case(f, dict(members=len(f.members) == 2, rand=[bool(b.bits[80]) for b in (r1, p1, p2, r2)] == [True, False, False, True]))


@case
def rand_bad_crc():
    P = np.frombuffer(T.ascii_random(5000, 12), np.uint8)
    stored = P ^ mask(P.size)
    b = W.from_content(stored.tobytes(), rand=1, crc=W.crc32(W.model_rle1(stored)[0]))   # the CRC of the masked bytes
    good = W.from_content(T.ascii_random(2000, 13))
    return Case(one(good, b), dict(crc_masked=b.crc != W.crc32(W.model_rle1(P)[0])))


@case
def rand_run4_at_end():
    P = _literals(2000, 14)
    P[-4:] = ord("w")
    b = rand_block(P)
    return Case(one(W.from_content(T.ascii_random(1000, 15)), b), dict(run4=bool(W.rle1_classes(P)[1]), rand=True))


# R2
@case
def sel_eq_groupcount():
    f = SC.build("sel_mtf_eq_groupcount").file
    return Case(f, dict(eq=len(f.members[0].blocks[0].lens) in f.members[0].blocks[0].sel_mtf))


@case
def sel_groupcount_minus_1():
    L = T.texty(6000, 21)
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    lens = [W.uniform_lengths(ns)] * 6
    need = -(-len(syms) // 50)
    b = W.block(syms, used, 222, lens=lens, sel_mtf=[5] + [0] * (need - 1), L=L)
    return Case(one(b), dict(max_ones=max(b.sel_mtf) == 5 and len(b.lens) == 6))


# R3
def _tail_run(k, count=None):
    P = _literals(3000, 16 + k)
    P = np.r_[P, np.full(k, ord("v"), np.uint8)] if k else P
    if count is not None:
        P = np.r_[P, np.uint8(count)]
    return P


@case
def run3_at_end():
    P = _tail_run(3)
    return Case(one(W.from_content(P.tobytes())), dict(run3=_rle_ok(P)))


@case
def run4_at_end():
    P = _tail_run(4)
    return Case(one(W.from_content(P.tobytes())), dict(run4=not _rle_ok(P)))


@case
def run4_count_at_end():
    P = _tail_run(4, 5)
    b = W.from_content(P.tobytes())
    return Case(one(b), dict(counted=_rle_ok(P) and b.report["last_is_count"]))


# R4: cuts of a two-block member
def _two_blocks():
    return one(W.from_content(T.ascii_random(3000, 30)), W.from_content(T.ascii_random(2500, 31)))


def _cut(name_cond, cut_bytes_fn):
    def make():
        f = _two_blocks()
        cut, cond = cut_bytes_fn(f)
        return Case(f, cond, cut=cut)
    return make


def _add(name, fn):
    CASES[name] = fn


def _at(cut, p):
    """Where a cut of `cut` bytes leaves the 80 bits (magic + CRC) at bit p."""
    return dict(no_whole_byte=cut * 8 - p < 8, in_magic=p + 8 <= cut * 8 < p + 48, in_crc=p + 48 <= cut * 8 < p + 80,
                complete=cut * 8 >= p + 80)


def _cut_at(p_of, k, where):
    def make(f):
        p = p_of(f)
        cut = (p + 7) // 8 + k
        return cut, {where: _at(cut, p)[where]}
    return make


_add("cut_header_only", _cut("", lambda f: (4, dict(header_only=f.block_starts[0] == 32))))
_add("cut_behind_block", _cut("", _cut_at(lambda f: f.block_starts[1], 0, "no_whole_byte")))
_add("cut_inside_block", _cut("", lambda f: ((f.block_starts[1] + f.members[0].blocks[1].bits.size) // 8 - 20,
                                             dict(inside=f.block_starts[1] + 80 <= ((f.block_starts[1] + f.members[0].blocks[1].bits.size) // 8 - 20) * 8))))
for _k in range(1, 11):
    _w = "in_magic" if _k <= 5 else "in_crc" if _k <= 9 else "complete"
    _add("cut_block_magic_%d" % _k, _cut("", _cut_at(lambda f: f.block_starts[1], _k, _w)))
    _add("cut_eos_%d" % _k, _cut("", _cut_at(lambda f: f.members[0].eos_pos, _k, _w)))


# R5: tails behind a complete member
TAILS = {"empty": b"", "nul": b"\0", "nuls": b"\0" * 64, "x": b"x", "bzh0": b"BZh0", "bzhX": b"BZhX", "B": b"B",
         "BZ": b"BZ", "BZh": b"BZh", "BZh9": b"BZh9", "BZh9_junk": b"BZh9junk", "mib_nuls": b"\0" * (1 << 20)}
HEADER_START = {"B", "BZ", "BZh", "BZh9", "BZh9_junk"}   # the tails whose first bytes (up to four) agree with "BZh1".."BZh9"


def header_start(t):
    return bool(t) and all(t[k] == b"BZh"[k] if k < 3 else 0x31 <= t[k] <= 0x39 for k in range(min(4, len(t))))


for _n, _t in TAILS.items():
    _add("tail_" + _n, lambda n=_n, t=_t: Case(one(W.from_content(T.ascii_random(2000, 40))),
                                              dict(header_start_as_named=header_start(t) == (n in HEADER_START)), tail=t))


# Past the first 64 KiB window: four blocks of about 30 KB each.  Under B2_DEC_WINDOW=65536 a stream's end is not known
# when the chain first reaches these positions.
def _late():
    return one(*[W.from_content(T.ascii_random(36000, 60 + i)) for i in range(4)])


_add("late_cut_behind_block", lambda: (lambda f: Case(f, dict(past_64k=f.block_starts[3] > 8 * 65536,
                                                           **_cut_at(lambda g: g.block_starts[3], 0, "no_whole_byte")(f)[1]),
                                                      cut=(f.block_starts[3] + 7) // 8))(_late()))
_add("late_cut_in_magic", lambda: (lambda f: Case(f, dict(past_64k=f.block_starts[3] > 8 * 65536,
                                                       **_cut_at(lambda g: g.block_starts[3], 3, "in_magic")(f)[1]),
                                                  cut=(f.block_starts[3] + 7) // 8 + 3))(_late()))
_add("late_tail_BZ", lambda: (lambda f: Case(f, dict(past_64k=len(f.data) > 65536 * 1.5, header_start=header_start(b"BZ")),
                                             tail=b"BZ"))(_late()))
_add("late_tail_nuls", lambda: (lambda f: Case(f, dict(past_64k=len(f.data) > 65536 * 1.5, header_start=not header_start(b"\0" * 9)),
                                               tail=b"\0" * 9))(_late()))


@case
def two_members_then_garbage():
    f = W.File([W.Member([W.from_content(T.ascii_random(2000, 41))], 9), W.Member([W.from_content(T.ascii_random(900, 42))], 3)])
    return Case(f, dict(members=len(f.members) == 2, garbage=not header_start(b"signature")), tail=b"signature: not bzip2\n")
