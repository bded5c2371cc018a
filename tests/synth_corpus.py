"""The synthetic bzip2 corpus: hand-built streams that reach the corners of the format (tests/bz2synth.py writes them).

Every case carries `cond`, the conditions it names, each computed from the writer's report, so a test can assert that
the case really reached them.  `libbz2` marks streams in libbz2's language (libbz2 rejects a `j == groupCount`
selector and a block that ends in an uncounted run of four); `hdec` marks the cases whose point is the
Huffman stage, which the GPU test runs at all three CTA widths of the Huffman decode kernel.
"""
import functools

import numpy as np

from tests import bz2synth as W
from tests import util as T

CASES = {}


class Case:
    def __init__(self, file, cond, libbz2=True, hdec=False, level=9):
        self.file, self.cond, self.libbz2, self.hdec, self.level = file, cond, libbz2, hdec, level


def case(fn):
    CASES[fn.__name__] = fn
    return fn


@functools.lru_cache(maxsize=None)
def build(name):
    return CASES[name]()


def fails_only(b, *checks):
    """b is rejected by exactly these checks of the decoder (in decode order), and its CRC is that of the bytes it
    decodes to without them: a decoder that skips one of them returns bytes instead of the error."""
    return b.err == W.DATA_ERROR and b.failed == list(checks) and b.would_be is not None and b.crc == W.crc32(b.would_be)


def one(blk, level=9, **kw):
    return W.File(W.Member([blk], level, **kw))


def rand_bytes(n, seed, lo=0, hi=256):
    return T.rng(seed).integers(lo, hi, size=n, dtype=np.uint8).tobytes()


def freq_order(symbols, nsym, reverse=False):
    """Symbols ordered by falling frequency (ties by symbol); reverse: rarest first."""
    f = np.bincount(np.array(symbols), minlength=nsym)
    order = sorted(range(nsym), key=lambda s: (-f[s], s))
    return order[::-1] if reverse else order


# ---- codes and windows --------------------------------------------------------------------------------------------
def _maxlen(M):
    L, orig = T.ascii_random(6000, 100 + M), 1234
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    order = freq_order(syms, ns)
    lens = [W.chain_lengths(ns, M, order), W.chain_lengths(ns, M, order[::-1][:1] + order[:-1])]
    b = W.block(syms, used, orig, lens=lens, tables=[i % 2 for i in range(-(-len(syms) // 50))], L=L)
    return Case(one(b), dict(max_code_len=b.max_code_len == M, min_len_1=min(lens[0]) == 1,
                             min_len_used=any(lens[0][s] == 1 for s in syms)), hdec=True)


@case
def maxlen18():
    return _maxlen(18)


@case
def maxlen19():
    return _maxlen(19)


@case
def maxlen20():
    return _maxlen(20)


@case
def delta_swing():
    L = T.texty(5000, 7)
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    lens = [W.chain_lengths(ns, 20, freq_order(syms, ns)), W.uniform_lengths(ns)]
    paths = [[[20, 1]] * ns, [[1, 20, 1, 20]] * ns]
    b = W.block(syms, used, 17, lens=lens, paths=paths, tables=[0, 1] * 100)
    return Case(one(b), dict(range=b.delta_range == [(1, 20)] * 2, swings=min(b.delta_swings) >= ns), hdec=True)


def _hole_lens(ns):
    l = W.uniform_lengths(ns)
    assert sum(2.0 ** -x for x in l) < 1
    return l


@case
def incomplete_unhit():
    L = T.ascii_random(4000, 5)
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    b = W.block(syms, used, 99, lens=[_hole_lens(ns)] * 3, tables=[0, 1, 2] * 40)
    return Case(one(b), dict(incomplete=sum(2.0 ** -x for x in b.lens[0]) < 1, ok=b.err is None), hdec=True)


@case
def incomplete_hit():
    L = T.ascii_random(4000, 6)
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    lens = [_hole_lens(ns)] * 2
    # the top word of a uniform code with holes is unassigned; the symbols, EOB included, go on behind it
    b = W.block(syms, used, 99, lens=lens, hole_at=len(syms) // 2)
    return Case(one(b), dict(hole=b.hole == (0, lens[0][0]) and 2 ** lens[0][0] > ns,
                             only=fails_only(b, "code hole")), hdec=True)


def _wide_tables():
    """19 used bytes (21 symbols): table A gives MTF index 1 (symbol 2) a 1-bit code, table B a 20-bit code."""
    used = list(range(97, 116))
    ns = len(used) + 2
    eob = ns - 1
    rest = [s for s in range(ns) if s not in (2, eob)]
    A = W.chain_lengths(ns, 20, [2, eob] + rest)
    B = W.chain_lengths(ns, 20, rest + [2, eob])
    assert A[2] == 1 and B[2] == 20 and B[eob] == 20
    return used, [A, B], eob


@case
def fifty_20bit():
    used, lens, eob = _wide_tables()
    syms = [2] * (50 * 6) + [eob]
    b = W.block(syms, used, 5, lens=lens, tables=[1] * 7)
    return Case(one(b), dict(g1000=int(b.group_bits.max()) == 1000, max20=b.max_code_len == 20), hdec=True)


@case
def alternating_1_20():
    used, lens, eob = _wide_tables()
    syms = [2] * (50 * 12) + [eob]
    b = W.block(syms, used, 7, lens=lens, tables=[0, 1] * 6 + [0])
    gb = b.group_bits.tolist()
    return Case(one(b), dict(alt=any(gb[i] == 50 and gb[i + 1] == 1000 for i in range(len(gb) - 1))), hdec=True)


def _eob_case(nsym_before, extra_sel):
    L = T.ascii_random(3000, nsym_before)
    syms, used = W.mtf_symbols(L)
    body = [s for s in syms[:-1]]
    while len(body) < nsym_before:
        body.append(2)
    body = body[:nsym_before]
    eob = len(used) + 1
    syms = body + [eob]
    need = -(-len(syms) // 50)
    b = W.block(syms, used, 3, nsel=need + extra_sel, tables=[0, 1] * need)
    return b, len(syms) - 1, need + extra_sel


@case
def eob_group_pos0():
    b, e, ns = _eob_case(50 * 40, 0)
    return Case(one(b), dict(pos0=e % 50 == 0), hdec=True)


@case
def eob_group_pos49():
    b, e, ns = _eob_case(50 * 40 + 49, 1)
    return Case(one(b), dict(pos49=e % 50 == 49, not_last=e // 50 < ns - 1), hdec=True)


@case
def eob_last_selector_50th():
    b, e, ns = _eob_case(50 * 40 + 49, 0)
    return Case(one(b), dict(pos49=e % 50 == 49, last=e // 50 == ns - 1), hdec=True)


# ---- selectors ----------------------------------------------------------------------------------------------------
@case
def six_tables_one_used():
    L = T.texty(8000, 3)
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    lens = [W.uniform_lengths(ns)] + [W.chain_lengths(ns, 15 + g, freq_order(syms, ns)) for g in range(5)]
    b = W.block(syms, used, 4000, lens=lens, tables=[0])
    return Case(one(b), dict(six=len(b.lens) == 6, one_used=set(b.tables) == {0}), hdec=True)


def _nsel(extra=None, total=None):
    L = T.ascii_random(2500, 8)
    syms, used = W.mtf_symbols(L)
    need = -(-len(syms) // 50)
    nsel = total if total else need + extra
    b = W.block(syms, used, 11, nsel=nsel, tables=[0, 1] * need)
    return b, need, nsel


@case
def nsel_need():
    b, need, ns = _nsel(0)
    return Case(one(b), dict(nsel=ns == need), hdec=True)


@case
def nsel_need_plus1():
    b, need, ns = _nsel(1)
    return Case(one(b), dict(nsel=ns == need + 1), hdec=True)


@case
def nsel_32767():
    b, need, ns = _nsel(total=32767)
    return Case(one(b), dict(nsel=ns == 32767 and need < 100), hdec=True)


@case
def sel_mtf_eq_groupcount():
    """Six tables, table 0 differs from the other five; the first selector's MTF index is 6 == groupCount."""
    L = T.texty(6000, 21)
    syms, used = W.mtf_symbols(L)
    ns = len(used) + 2
    other = W.chain_lengths(ns, 17, freq_order(syms, ns))
    lens = [W.uniform_lengths(ns)] + [other] * 5
    need = -(-len(syms) // 50)
    mtf = [6] + [0] * 9 + [6] + [1, 0] * need
    b = W.block(syms, used, 222, lens=lens, sel_mtf=mtf[:need], L=L)
    return Case(one(b), dict(quirk=6 in b.sel_mtf, first_table0=b.tables[0] == 0, later_table5=b.tables[10] == 5,
                             t0_differs=lens[0] != lens[5]), libbz2=False, hdec=True)


@case
def selectors_exhausted():
    L = T.ascii_random(2500, 9)
    syms, used = W.mtf_symbols(L)
    need = -(-len(syms) // 50)
    ns = len(used) + 2
    lens = [W.uniform_lengths(ns), W.chain_lengths(ns, 12, freq_order(syms, ns))]
    b = W.block(syms, used, 11, lens=lens, tables=[0, 1] * need, nsel=need - 1)
    return Case(one(b), dict(short=b.eob_index // 50 >= b.nsel, tables_differ=lens[0] != lens[1],
                             only=fails_only(b, "selectors exhausted")), hdec=True)


# ---- alphabet and runs --------------------------------------------------------------------------------------------
@case
def symtotal_1():
    b = W.from_column(b"A" * 3001, 17)
    return Case(one(b), dict(st1=len(b.used) == 1))


@case
def symtotal_256():
    L = rand_bytes(20000, 4)
    b = W.from_column(L, 777)
    return Case(one(b), dict(st256=len(b.used) == 256))


@case
def sparse_map():
    g = T.rng(12)
    used = sorted(set([16 * k + int(g.integers(0, 16)) for k in range(0, 16, 3)] + [0, 255]))
    L = bytes(g.choice(used, size=5000).astype(np.uint8))
    b = W.from_column(L, 2)
    hi = {u >> 4 for u in b.used}
    return Case(one(b), dict(sparse=len(hi) < 16 and len(b.used) < 16))


@case
def run_before_first_literal():
    L = b"\x05" * 40 + rand_bytes(3000, 13, 6, 256)
    b = W.from_column(L, 1500, used=sorted(set(L)))
    return Case(one(b), dict(first_is_run=b.symbols[0] <= 1 and b.used[0] == 5))


@case
def run_straddles_unmtf_chunk():
    used = list(range(65, 91))
    eob = len(used) + 1
    d1 = W.run_digits(1000)
    d2 = W.run_digits(300000)
    syms = [2, 3] * 2046 + [2] + d1 + [3, 2] * ((8192 - 4095 - len(d1)) // 2 - 4)
    syms = syms + [2] * (8192 - 9 - len(syms)) + d2 + [3, 4, 5] + [eob]
    b = W.block(syms, used, 10, lens=[W.uniform_lengths(eob + 1)] * 2)
    run_at = [i for i in range(1, len(syms)) if syms[i] <= 1 and syms[i - 1] > 1]
    straddle = [i for i in run_at if any(i < k * 4096 < i + 10 for k in (1, 2))]
    return Case(one(b), dict(straddle=len(straddle) >= 2, digits18=len(d2) == 18))


def _run_block(nlit, run, level, tail=(2,)):
    """nlit literals, one run of `run` copies, the tail symbols, EOB (two used bytes: EOB is symbol 3)."""
    used = [ord("x"), ord("y")]
    syms = [2] * nlit + W.run_digits(run) + list(tail) + [3]
    return W.block(syms, used, 0, level=level, lens=[W.uniform_lengths(4)] * 2), len(W.run_digits(run))


@case
def run_fills_dbuf():
    b, _ = _run_block(1000, 100000 - 1000, 1, tail=())
    return Case(one(b, 1), dict(exact=b.report["n"] == 100000, ok=b.err is None), level=1)


@case
def run_past_dbuf():
    b, _ = _run_block(1000, 100000 - 1000 + 1, 1, tail=())
    return Case(one(b, 1), dict(only=fails_only(b, "run past dbufSize"), n=b.report["n"] == 100001), level=1)


def _digits_case(run, level):
    # the run is the last thing before EOB: where it is too long, the run bound is the only check that fails
    return _run_block(7, run, level, tail=())


@case
def run18_l9():
    b, d = _digits_case(300000, 9)
    return Case(one(b), dict(digits=d == 18, ok=b.err is None))


@case
def run19_l9():
    b, d = _digits_case(600000, 9)
    return Case(one(b), dict(digits=d == 19, ok=b.err is None))


@case
def run18_l1():
    b, d = _digits_case(300000, 1)
    return Case(one(b, 1), dict(digits=d == 18, only=fails_only(b, "run past dbufSize")), level=1)


@case
def run19_l1():
    b, d = _digits_case(600000, 1)
    return Case(one(b, 1), dict(digits=d == 19, only=fails_only(b, "run past dbufSize")), level=1)


@case
def run20_l9():
    b, d = _digits_case(2 ** 20 - 1, 9)
    return Case(one(b), dict(digits=d == 20, only=fails_only(b, "run past dbufSize")))


@case
def run21_l9():
    b, d = _digits_case(2 ** 21 + 5, 9)
    return Case(one(b), dict(digits=d == 21, only=fails_only(b, "run past dbufSize")))


# ---- block limits -------------------------------------------------------------------------------------------------
@case
def n_equals_1():
    b = W.from_column(b"Q", 0)
    return Case(one(b), dict(n1=b.report["n"] == 1))


def _full(level, extra):
    n = 100000 * level + extra
    return W.from_column(rand_bytes(n, level * 10 + extra, 32, 127), n // 3, level=level), n


@case
def n_dbuf_l1():
    b, n = _full(1, 0)
    return Case(one(b, 1), dict(n=b.report["n"] == 100000), level=1)


@case
def n_dbuf_plus1_l1():
    b, n = _full(1, 1)
    return Case(one(b, 1), dict(only=fails_only(b, b.failed[0]) and b.failed[0].endswith("past dbufSize"),
                                n=b.report["n"] == n), level=1)


@case
def n_dbuf_l9():
    b, n = _full(9, 0)
    return Case(one(b), dict(n=b.report["n"] == 900000))


@case
def n_dbuf_plus1_l9():
    b, n = _full(9, 1)
    return Case(one(b), dict(only=fails_only(b, b.failed[0]) and b.failed[0].endswith("past dbufSize"),
                             n=b.report["n"] == n))


def _orig(o):
    L = rand_bytes(5000, 77, 97, 123)
    syms, used = W.mtf_symbols(L)
    return W.block(syms, used, o)


@case
def orig_0():
    b = _orig(0)
    return Case(one(b), dict(ok=b.err is None))


@case
def orig_n_minus_1():
    b = _orig(4999)
    return Case(one(b), dict(ok=b.err is None))


@case
def orig_n():
    b = _orig(5000)
    return Case(one(b), dict(only=fails_only(b, "origPtr >= block length")))


@case
def orig_past_dbuf():
    b = _orig(900001)
    return Case(one(b), dict(only=fails_only(b, "origPtr > dbufSize", "origPtr >= block length")))


# ---- inverse BWT --------------------------------------------------------------------------------------------------
@case
def random_column():
    L = rand_bytes(60000, 31, 0, 40)
    b = W.from_column(L, 12345)
    return Case(one(b), dict(not_bwt=b.report["cycle"] < 60000))


@case
def short_cycle():
    L = np.frombuffer(rand_bytes(30000, 32, 0, 8), np.uint8)
    Tv = np.argsort(L, kind="stable")
    best = None
    for o in range(0, 30000, 7):
        r0 = int(Tv[o])
        row, c = int(Tv[r0]), 1
        while row != r0 and c < 500:
            row, c = int(Tv[row]), c + 1
        if c < 500:
            best = o
            break
    b = W.from_column(L.tobytes(), best)
    return Case(one(b), dict(short=b.report["cycle"] < 500))


def _visits(k, want_visits):
    """(X^k)'s column: every byte of a 54-byte column repeated k times, so the T-vector is k parallel cycles; the start
    row picks a cycle with no multiple of 128 in it, so the GPU walk is cut only at the start row, k times."""
    c = 54
    X = rand_bytes(c, 5, 97, 123)
    from oracle import oracle as O
    Lx, _ = O.bwt_cyclic(X)
    L = np.repeat(np.frombuffer(Lx, np.uint8), k)
    Tv = np.argsort(L, kind="stable")
    for t in range(1, k):
        rows = np.arange(c) * k + t
        if not np.any(rows % 128 == 0):
            break
    orig = int(np.flatnonzero(Tv == t)[0])
    b = W.from_column(L.tobytes(), orig)
    return Case(one(b), dict(visits=b.report["visits"] == want_visits, n=b.report["n"] == c * k))


@case
def visits_16383():
    return _visits(16383, 16383)


@case
def visits_16384():
    return _visits(16384, 16384)


@case
def visits_16385():
    return _visits(16385, 16385)


@case
def long_walks():
    b = W.from_content(T.texty(200000, 44))
    return Case(one(b), dict(walk=b.report["max_visit"] > W.IB_CAP))


# ---- RLE1 decode --------------------------------------------------------------------------------------------------
@case
def rle_runs_5_to_12():
    B = b"".join(bytes([65 + r]) * r + b"-" for r in range(5, 13)) * 20
    b = W.from_content(B)
    return Case(one(b), dict(eq=set(range(5, 13)) <= b.report["eq_count_runs"]))


@case
def rle_count_0_255():
    g = T.rng(55)
    parts = []
    for i in range(6000):
        f = int(g.integers(1, 9))
        filler = bytes(range(100, 100 + f))
        parts.append(filler + b"zzzz" + (b"\x00" if i % 2 else b"\xff"))
    B = b"".join(parts)
    b = W.from_content(B)
    r = b.report
    return Case(one(b), dict(mod8_0=r["count0_mod8"] == set(range(8)), mod8_255=r["count255_mod8"] == set(range(8)),
                             tile_edge={0, 255} <= r["count_at_tile_edge"]))


@case
def rle_count_last():
    B = T.ascii_random(5000, 3) + b"bbbb\x07"
    b = W.from_content(B)
    return Case(one(b), dict(last=b.report["last_is_count"]))


@case
def rle_run4_at_end():
    B = T.ascii_random(5000, 4).replace(b"bbbb", b"bcbc") + b"bbbb"
    b = W.from_content(B)
    return Case(one(b), dict(run4=b.report["trailing_run4"]), libbz2=False)


def max_expansion_block():
    """A full level-9 block of `aaaa\\xff` runs: (aaaa\\xff)^180000, whose column is \\xff * k + a * 4k."""
    k = 180000
    L = b"\xff" * k + b"a" * (4 * k)
    return W.from_column(L, 0)


@case
def rle_max_expansion():
    b = max_expansion_block()
    return Case(one(b), dict(stage=b.report["max_tile_out"] > 6144, ratio=len(b.out) == 259 * 180000))


# ---- magics and phases --------------------------------------------------------------------------------------------
def _plant_tables():
    """253 used bytes (255 symbols): symbol 2 has the one 7-bit code, all others 8 bits -- a complete code in which a
    magic pattern reads as six literals."""
    used = list(range(1, 254))
    ns = len(used) + 2
    lens = [8] * ns
    lens[2] = 7
    return used, [lens, lens], ns - 1


def _planted_block(k, seed, magics):
    used, lens, eob = _plant_tables()
    g = T.rng(seed)
    syms = [2] * k
    for m in magics:
        syms += W.decode_bits("{:048b}".format(m), lens[0], avoid={0, 1, eob})
        syms += [int(x) for x in g.integers(2, eob, size=5)]
    syms += [int(x) for x in g.integers(2, eob, size=30)] + [eob]
    return W.block(syms, used, 3, lens=lens)


def _phase_stream(magic):
    """Eight blocks, each with one planted `magic` pattern, at the 8 bit phases."""
    blocks, pos = [], 32
    for ph in range(8):
        for k in range(16):
            b = _planted_block(k, ph * 100 + k, [magic])
            bits = np.packbits(b.bits).tobytes()
            offs = [p for p in W.magic_positions(bits)[0 if magic == W.BLOCK_MAGIC else 1] if p > 0]
            if offs and (pos + offs[0]) % 8 == ph:
                break
        blocks.append(b)
        pos += b.bits.size
    f = one_of(blocks)
    planted = f.planted_block if magic == W.BLOCK_MAGIC else f.planted_eos
    return Case(f, dict(phases={p % 8 for p in planted} == set(range(8))), hdec=True)


def one_of(blocks, level=9):
    return W.File(W.Member(blocks, level))


@case
def planted_block_magic():
    return _phase_stream(W.BLOCK_MAGIC)


@case
def planted_eos_magic():
    return _phase_stream(W.EOS_MAGIC)


@case
def block_starts_mod32():
    blocks, pos = [], 32
    for i in range(32):
        L = rand_bytes(int(T.rng(i).integers(3, 40)), i, 97, 110)
        base = W.from_column(L, 1)
        need = len(base.sel_mtf)
        extra = (1 - base.bits.size) % 32
        b = W.from_column(L, 1, nsel=need + extra)
        assert b.bits.size % 32 == 1
        blocks.append(b)
    f = one_of(blocks)
    return Case(f, dict(res32={p % 32 for p in f.block_starts} == set(range(32))))


@case
def sharded_planted():
    """Block 0 holds a planted block magic, block 1 follows: the candidates are [block 0, planted, block 1], so at
    world sizes 2 and 3 the planted one lies in rank 1's share while its block lies in rank 0's."""
    b0 = _planted_block(3, 1, [W.BLOCK_MAGIC])
    b1 = W.from_column(T.ascii_random(3000, 2), 9)
    f = one_of([b0, b1])
    idx = f.candidates.index(f.planted_block[0]) if f.planted_block else -1
    return Case(f, dict(planted=len(f.planted_block) == 1 and len(f.candidates) == 3,
                        rank1_w2=idx >= 3 * 1 // 2, rank1_w3=idx >= 3 * 1 // 3 and idx < 3 * 2 // 3))


def multistream_file():
    """Two members, level 1 then level 9, whose blocks are synthetic."""
    a = W.from_column(rand_bytes(7000, 61, 97, 110), 5, level=1)
    b = max_expansion_block()
    return W.File([W.Member([a], 1), W.Member([b, W.from_column(rand_bytes(3000, 62, 120, 123), 4)], 9)])


def relevelled():
    """Blocks rejected only by a dbufSize bound of a level below 9, behind a level-9 header instead: (name, file,
    bytes the block decodes to without the bound)."""
    out = []
    for name in sorted(CASES):
        c = build(name)
        for b in c.file.members[0].blocks:
            if b.err is not None and b.level < 9 and all(f.endswith("past dbufSize") for f in b.failed):
                out.append((name, W.File(W.Member([b], 9)), b.would_be))
    return out
