"""Designed blocks for the libbz2 flavor's Huffman table search (csrc/huff.cu k_huffman_libbz2; sendMTFValues and
BZ2_hbMakeCodeLengths of libbz2): the 17-bit rescale in every round and table, the initial partition's odd-nPart step,
its running out of alphabet, ties between tables and in the heap, the largest group cost, and the selector counts and
symbol positions at the 256-group tile seam of the kernel.

Blocks are designed by their MTF ranks with the column designs of tests/mtfhuff_cases.py.  A design with no zero rank
has no zero run, so rank r is zero-run symbol r + 1 and the symbol frequencies are the rank counts.  Every case states
its claims as predicates over the libbz2 model's report of the blocks it ended up with (tests/libbz2_model.py encode:
per block the symbols and the table search's report); tests/test_libbz2_table_cases.py asserts them.

Two frequency shapes make the heap builder deep:
- a Fibonacci chain: each merged node is one of the two smallest until the root, so the depth grows by one per term;
- a pinned block: every group holds mostly one background symbol, so every group costs least under the same table and
  the other tables are never selected (rebuilt from all-1 weights, flat).  One table then holds the whole chain in
  every round, and the rescale survives into the written tables.  Where the groups are shuffled instead, the groups
  spread over several tables and each table holds a thinner chain.
"""
import functools
from dataclasses import dataclass, field

import numpy as np

from tests import libbz2_model as M
from tests import mtfhuff_cases as MC
from tests import util as U

GROUP = 50
TILE_GROUPS = MC.TILE_GROUPS


def fib(n, a=1, b=1):
    f = [a, b]
    while len(f) < n:
        f.append(f[-1] + f[-2])
    return f[:n]


# ---- designs: each returns the ranks of one block ------------------------------------------------------------------
def _pinned(chain, bg, seed, alpha=None, prefix=False, tail=()):
    """Groups of `bg` rank-1 symbols (the background) and 50 - bg symbols of a chain: chain[i] copies of rank i + 2,
    shuffled.  `prefix`: every rank of the alphabet once first (all `alpha` bytes used).  `tail`: ranks put last."""
    alpha = alpha or len(chain) + 2
    g = U.rng(seed)
    ch = np.repeat(np.arange(2, len(chain) + 2, dtype=np.int32), chain)
    g.shuffle(ch)
    k = GROUP - bg
    ng = -(-ch.size // k)
    grid = np.ones((ng, GROUP), np.int32)
    flat = np.ones(ng * k, np.int32)
    flat[:ch.size] = ch
    grid[:, :k] = flat.reshape(ng, k)
    for row in grid:
        g.shuffle(row)
    d = MC.Design(alpha, seed)
    if prefix:
        d.put(list(range(alpha - 1, 0, -1)), protect=False)
    d.put(grid.ravel(), protect=False)
    if len(tail):
        d.put(np.asarray(tail, np.int32))
    return d


def _shuffled(counts, seed, alpha=None):
    """counts[i] copies of rank i + 1, in a seeded order."""
    r = np.repeat(np.arange(1, len(counts) + 1, dtype=np.int32), counts)
    U.rng(seed).shuffle(r)
    return MC.Design(alpha or len(counts) + 1, seed).put(r, protect=False)


def _same_groups(alpha, ngroups, seed):
    """Every group a permutation of ranks 1..50: the groups cost the same under every table, and the table they all
    select holds 50 used symbols of one frequency."""
    g = U.rng(seed)
    rows = [g.permutation(np.arange(1, GROUP + 1, dtype=np.int32)) for _ in range(ngroups)]
    return MC.Design(alpha, seed).put(np.concatenate(rows), protect=False)


def _runa_heavy(n, seed):
    """Ranks [r, 0]: every zero run has length 1 and is one RUNA, half of the symbols."""
    g = U.rng(seed)
    r = np.zeros(n, np.int32)
    r[0::2] = np.minimum(g.geometric(0.2, size=(n + 1) // 2), 29)
    return MC.Design(30, seed).put(r, protect=False)


def _uniform(alpha, n, seed):
    return MC.Design(alpha, seed).uniform(n)


def _seam256(m_want, seed):
    """Alphabet 256, uniform ranks, rank 255 (symbol 256) planted at symbols 12 798..12 800: the last group of the
    kernel's first 256-group tile and the first group of the second (the end of block, symbol 257, ends one of them
    when m is 12 800 or 12 801).  m is tuned to m_want."""
    seam = TILE_GROUPS * GROUP

    def make(n, s):
        d = MC.Design(256, s)
        d.put(list(range(255, 0, -1)))
        if n >= seam:
            d.uniform(seam - 2 - d.n)
            d.put([255, 255] + ([255] if n >= seam + 2 else []))
        d.uniform(n - d.n)
        return d

    def tuned():
        for s in range(seed, seed + 8):     # the cycle merge can keep m off by one for a seed: take the next
            try:
                return MC._tune(lambda n: make(n, s), m_want)
            except AssertionError:
                pass
        raise AssertionError("no seed reaches m = %d" % m_want)
    return tuned


def _six_kinds(n, seed):
    """A full level-9 block of six kinds of groups in random order: a thinned Fibonacci chain (deep enough to rescale),
    uniform ranks and four geometric spreads, all 256 bytes used."""
    d = MC.Design(256, seed)
    d.put(list(range(255, 0, -1)), protect=False)
    chain = np.repeat(np.arange(1, 28, dtype=np.int32), fib(27)[::-1])
    d.g.shuffle(chain)
    used = 0
    ps = [0.5, 0.2, 0.08, 0.03]
    while d.n < n:
        k = min(int(d.g.integers(1, 6)) * GROUP, n - d.n)
        c = int(d.g.integers(0, 6))
        if c == 0 and used + k <= chain.size:
            d.put(chain[used:used + k], protect=False)
            used += k
        elif c == 1:
            d.uniform(k)
        else:
            d.fill(k, p=ps[min(c - 2, 3)])
    return d


# ---- the cases -----------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    make: object           # seed -> Design, or seed -> raw bytes, or () -> [(ranks, used, protect)] (tuned)
    levels: tuple
    claims: list = field(default_factory=list)   # (what, predicate(Info))
    seed: int = 0          # the first seed that reaches every claim (found by search; see find_seed)


class Info:
    """The raw input of a case and the libbz2 model's blocks of it (M.encode), at the case's first level."""

    def __init__(self, case, seed=None):
        self.case = case
        self.seed = case.seed if seed is None else seed
        self.raw = raw(case.name) if seed is None else build(case, seed)
        self.stream, self.blocks = M.encode(self.raw, case.levels[0])

    def rounds(self, b=0):
        return self.blocks[b]["report"]["rounds"]

    def init(self, b=0):
        return self.blocks[b]["report"]["init"]

    def freq(self, b=0):
        blk = self.blocks[b]
        return np.bincount(blk["syms"], minlength=blk["alpha"] + 2)

    def holds(self):
        return [what for what, f in self.case.claims if not f(self)]


def build(case, seed):
    d = case.make(seed) if case.make.__code__.co_argcount else case.make()
    if isinstance(d, (bytes, bytearray)):
        return bytes(d)
    if isinstance(d, MC.Design):
        d = [(d.ranks(), MC.used_bytes(d.alpha, seed), d.protect())]
    ranks, used, prot = d[0]
    return MC.build_block(ranks, used, 9, False, None, prot).raw.tobytes()


@functools.lru_cache(maxsize=None)
def raw(name):
    c = case(name)
    return build(c, c.seed)


def find_seed(case, tries=40):
    """The first seed from case.seed on at which every claim holds (used to pick the seeds below)."""
    for s in range(case.seed, case.seed + tries):
        if not Info(case, s).holds():
            return s
    raise AssertionError("%s: no seed reaches every claim" % case.name)


# ---- predicates ----------------------------------------------------------------------------------------------------
def _tables(ci, rounds=range(4), b=0):
    return [(r, t, x) for r in rounds for t, x in enumerate(ci.rounds(b)[r]["tables"])]


def rescale_in(rounds, tables=None, max_len=None, alpha=None):
    def f(ci):
        if alpha is not None and ci.blocks[0]["alpha"] != alpha:
            return False
        return any(x["rescales"] >= 1 and (tables is None or t in tables) and (max_len is None or x["max_len"] == max_len)
                   for r, t, x in _tables(ci, rounds))
    return f


def no_rescale_in(rounds):
    return lambda ci: not any(x["rescales"] for r, t, x in _tables(ci, rounds))


def _six_tables(ci):
    return ci.blocks[0]["ngroups"] == 6


def odd_moved(*parts):
    return lambda ci: _six_tables(ci) and set(parts) <= set(ci.init()["odd_moved"])


def odd_single(ci):
    return bool(ci.init()["odd_single"])


def exhausted_flat_written(ci):
    """A table of all 15s (its part ran out of alphabet) that no group selects in any round: every build of it is from
    all-1 weights, and the written one no selector names."""
    rng = ci.init()["ranges"]
    return ci.init()["exhausted"] and any(rng[t][0] > rng[t][1] and all(ci.rounds()[r]["tables"][t]["selected"] == 0
                                                                        for r in range(4)) for t in range(len(rng)))


def over_tfreq(ci):
    """The first part is symbol 0 (RUNA) alone, whose frequency exceeds tFreq."""
    blk = ci.blocks[0]
    gs, ge, tf = ci.init()["ranges"][blk["ngroups"] - 1]
    return gs == ge == 0 and int(ci.freq()[0]) > tf


def ties_in(r):
    return lambda ci: ci.rounds()[r]["ties"] > 0


def equal_heap(count):
    return lambda ci: any(x["equal_used"] >= count and x["heap_tie"] for r, t, x in _tables(ci))


def max_cost(cost):
    return lambda ci: any(rd["max_cost"] == cost for rd in ci.rounds())


def nsel_is(k):
    return lambda ci: ci.blocks[0]["nsel"] == k


def m_mod(r):
    return lambda ci: ci.blocks[0]["m"] % GROUP == r


def hi_symbol_at_seam(ci):
    """Symbol 256 or 257 in group 255 and, when the block has it, in group 256 (either side of the first tile seam)."""
    s = np.asarray(ci.blocks[0]["syms"])
    grp = np.flatnonzero(s >= 256) // GROUP
    return {TILE_GROUPS - 1, min(TILE_GROUPS, ci.blocks[0]["nsel"] - 1)} <= set(grp.tolist())


def full_l9(ci):
    blk = ci.blocks[0]
    return blk["nsel"] >= 17900 and len(set(blk["sel"])) == 6 and rescale_in(range(4))(ci)


def rescale_with_zeros(ci):
    """A table of A = 258 (alphabet 256) with symbols of frequency 0 (weight 1) rescales."""
    return ci.blocks[0]["alpha"] == 256 and any(x["rescales"] and x["zeros"] for _, _, x in _tables(ci))


@functools.lru_cache(maxsize=1)
def cases():
    # rescale_written and group_850 start from all 256 bytes; the built blocks keep 128 of them (their alphabet is claimed
    # nowhere: l9_six_kinds holds the alphabet-256 rescale)
    cs = [
        Case("rescale_written", lambda s: _pinned(fib(20, 5, 14), 25, s, alpha=256, prefix=True), (9,),
             [("a table of round 4 rescales once and its longest code is 17", rescale_in([3], max_len=17)),
              ("the rescale is in a table other than table 0", rescale_in([3], tables=range(1, 6))),
              ("a table no group selects is rebuilt flat and written", lambda ci: any(x["selected"] == 0 for _, _, x in _tables(ci, [3])))]),
        Case("rescale_early_only", lambda s: _shuffled(fib(28)[::-1], s), (9,),
             [("a table of round 1, 2 or 3 rescales", rescale_in(range(3))),
              ("no table of round 4 rescales", no_rescale_in([3])),
              ("groups tie between tables in round 1 and in round 4", lambda ci: ties_in(0)(ci) and ties_in(3)(ci))]),
        Case("odd_step_moves", lambda s: _uniform(40, 3200, s), (1,),
             [("six tables; the odd step moves a bound at nPart 5 and 3", odd_moved(5, 3))]),
        Case("odd_step_single", lambda s: _shuffled(fib(18)[::-1], s), (1,),
             [("the odd step is due on a single-symbol part and skipped", odd_single)]),
        Case("exhausted_alpha2", lambda s: _letters(2, 3000, s), (1,),
             [("the partition runs out of alphabet: an all-15 table never selected, rebuilt flat, written",
               exhausted_flat_written)]),
        Case("exhausted_alpha3", lambda s: _letters(3, 4000, s), (1,),
             [("the partition runs out of alphabet: an all-15 table never selected, rebuilt flat, written",
               exhausted_flat_written)]),
        Case("runa_over_tfreq", lambda s: _runa_heavy(6000, s), (1,),
             [("the first part is RUNA alone, over tFreq", over_tfreq)]),
        Case("same_groups", lambda s: _same_groups(51, 60, s), (1,),
             [("groups tie between tables in round 1", ties_in(0)),
              ("groups tie between tables in round 4", ties_in(3))]),
        Case("group_850", lambda s: _pinned(fib(20, 5, 14), 25, s, alpha=256, prefix=True, tail=np.arange(200, 250)), (9,),
             [("a group costs 50 x 17 = 850 bits under a table", max_cost(850)),
              ("48+ used symbols of one frequency in a table, and the heap ties", equal_heap(48))]),
    ]
    for nsel, m in ((255, 12749), (256, 12800), (257, 12801), (511, 25549), (512, 25600)):
        claims = [("nsel = %d" % nsel, nsel_is(nsel)), ("m = %d (mod 50)" % (m % GROUP), m_mod(m % GROUP))]
        if nsel in (256, 257):
            claims.append(("symbol 256 or 257 on both sides of the 256-group tile seam", hi_symbol_at_seam))
        cs.append(Case("nsel_%d" % nsel, _seam256(m, 901 + nsel), (9,), claims))
    cs.append(Case("l9_six_kinds", lambda s: _six_kinds(899981 - 2000, s), (9,),
                   [("nsel >= 17 900, all six tables selected, a rescale", full_l9),
                    ("alphabet 256: a table with symbols of frequency 0 rescales", rescale_with_zeros)]))
    return cs


def _letters(k, n, seed):
    """Random bytes of k letters, no run longer than 3 (no RLE1 count byte): A = k + 2 symbols for six tables."""
    g = U.rng(seed)
    out, last, run = bytearray(), None, 0
    while len(out) < n:
        c = int(g.integers(0, k))
        if c == last and run == 3:
            c = (c + 1) % k
        run = run + 1 if c == last else 1
        last = c
        out.append(97 + c)
    return bytes(out)


def case(name):
    return next(c for c in cases() if c.name == name)


@functools.lru_cache(maxsize=None)
def info(name):
    return Info(case(name))


def corpus():
    """(name, raw, level) of every case at each of its levels."""
    return [(c.name, raw(c.name), lv) for c in cases() for lv in c.levels]


def whole():
    """Every case's input, joined: one file of several level-9 blocks."""
    return b"".join(raw(c.name) for c in cases())


# ---- reference trace -----------------------------------------------------------------------------------------------
def _byte_at_every_bit(bits):
    v = np.zeros(bits.size - 7, np.uint8)
    for k in range(8):
        v |= bits[k:bits.size - 7 + k] << (7 - k)
    return v


def _find(v, pattern):
    ok = np.ones(v.size - 8 * (len(pattern) - 1), bool)
    for k, byte in enumerate(pattern):
        ok &= v[8 * k:8 * k + ok.size] == byte
    return np.flatnonzero(ok)


def block_edges(z):
    """Bit positions of every block magic of the bzip2 stream z, and of its end-of-stream magic last."""
    v = _byte_at_every_bit(np.unpackbits(np.frombuffer(z, np.uint8)))
    starts = _find(v, b"\x31\x41\x59\x26\x53\x59")
    end = _find(v, b"\x17\x72\x45\x38\x50\x90")
    return np.concatenate((starts, end[-1:])).tolist()


def block_bit_lens(z):
    """Bits from each block's magic to the end of its symbols in the bzip2 stream z (a block ends where the next magic
    starts)."""
    return np.diff(block_edges(z)).tolist()


def reference_trace(data, level, z):
    """Per block the TRACE_FIELDS of the libbz2 flavor: n, pidx, m, alpha, ngroups and nsel of the oracle's blocks
    (the two flavors cut these inputs alike: the tests assert it), the CRC, and bit_len from libbz2's stream z."""
    from oracle import oracle as O
    _, tr = O.bzip2_compress(data, level, trace=True)
    rows = np.array([[getattr(t, f) for f in M.TRACE_FIELDS] for t in tr], dtype=np.int64).reshape(-1, len(M.TRACE_FIELDS))
    lens = block_bit_lens(z)
    assert len(lens) == len(rows), "libbz2 wrote %d blocks, the oracle %d" % (len(lens), len(rows))
    rows[:, M.TRACE_FIELDS.index("bit_len")] = lens
    return rows
