"""Case corpus for the encoder's move-to-front + zero-run coder (csrc/mtf.cu) and Huffman table search (csrc/huff.cu),
built from the stage's own point of view.

The input of both stages is a pure function of the block's BWT column L, so every case designs L (as an MTF rank
sequence over the sorted used-byte list) and then finds an input that makes the encoder produce exactly that column:

1. the designed ranks run through the inverse MTF give a column L;
2. a column is the cyclic BWT of some block only when its LF permutation is one cycle.  Swapping two adjacent,
   different bytes of L composes LF with the transposition of their rows, which merges the two cycles when the rows
   lie in different ones; a union-find over the cycle labels picks the swaps (positions the design marks as protected
   are avoided while others will do).  Fixed points inside a run that covers its own byte's F bucket are not next to
   a different byte, but every pass swaps the run's edge byte, which moves the next one to the edge for the pass
   after, so repeated passes reach them without rotating the run;
3. the block T is the inverse BWT of L, rotated to start on a run start so that the encoder's RLE1 stage reads it
   back unchanged; a T that no rotation makes a valid RLE1 output (a run of four followed by a count the encoder
   would not write) has its long runs broken and its column recomputed;
4. the raw input is T with its RLE1 count bytes expanded; blocks of a multi-block case are full (blockSize RLE1
   bytes), so that the encoder cuts where the design says.

Perturbations are expected, so every case states what it reaches as predicates over the column it ended up with and
over the oracle's compress_block_stages output (symbols, selectors, code lengths, trace); the CPU test asserts them.
`search` is a plain model of the Huffman table search (lib/Bzip2.js:685-733) that also reports the ties the search
met, with the oracle's length-limited allocator for the code lengths.
"""
import functools
import heapq
from dataclasses import dataclass, field

import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

from oracle import oracle as O
from tests import bz2synth as S
from tests import util as U

CHUNK = 4096          # zero-run coder chunk (k_mtf_ranks, k_rle2)
WINDOW = 32           # bytes one warp ranks per step
GROUP = 50
TILE_GROUPS = 256     # groups per staged tile of k_huffman; also its thread count
MAX_LEN = 20


def block_size(level):
    return level * 100000 - 19


# ---- the stage's own model ---------------------------------------------------------------------------------------
BRING_MIN, BRING_MAX = -1, -2   # design ranks that bring the smallest / largest used byte to the front


def unmtf(ranks, used):
    """Column whose MTF ranks over the sorted used-byte list are `ranks`."""
    lst = list(used)
    out = bytearray(len(ranks))
    for i, r in enumerate(ranks.tolist() if isinstance(ranks, np.ndarray) else ranks):
        if r < 0:
            r = lst.index(used[0] if r == BRING_MIN else used[-1])
        if r:
            lst.insert(0, lst.pop(r))
        out[i] = lst[0]
    return np.frombuffer(bytes(out), np.uint8).copy()


def mtf_ranks(L):
    """MTF rank of every byte of L over its sorted used-byte list."""
    used = sorted(set(np.asarray(L).tolist()))
    lst = list(used)
    out = np.empty(len(L), np.int32)
    for i, b in enumerate(np.asarray(L).tolist()):
        if lst[0] == b:
            out[i] = 0
            continue
        j = lst.index(b)
        del lst[j]
        lst.insert(0, b)
        out[i] = j
    return out


def zero_runs(ranks):
    """(start, length) of every maximal run of zero ranks."""
    z = np.concatenate(([0], (np.asarray(ranks) == 0).astype(np.int8), [0]))
    d = np.diff(z)
    s, e = np.flatnonzero(d == 1), np.flatnonzero(d == -1)
    return s, e - s


def lf(L):
    order = np.argsort(L, kind="stable")
    out = np.empty(L.size, np.int64)
    out[order] = np.arange(L.size)
    return out


def cycles(L):
    n = L.size
    g = csr_matrix((np.ones(n, np.int8), (np.arange(n), lf(L))), shape=(n, n))
    return connected_components(g, directed=True, connection="strong")


def merge_cycles(L, protect=None):
    """One-cycle column close to L.  Returns (column, adjacent swaps)."""
    L = L.copy()
    swaps = 0
    while True:
        k, lab = cycles(L)
        if k == 1:
            return L, swaps
        parent = list(range(k))

        def find(a):
            while parent[a] != a:
                parent[a] = parent[parent[a]]
                a = parent[a]
            return a

        diff = (L[:-1] != L[1:]) & (lab[:-1] != lab[1:])
        did = 0
        tries = [diff & ~protect[:-1] & ~protect[1:], diff] if protect is not None else [diff]
        for cand in tries:
            last = -2
            for i in np.flatnonzero(cand).tolist():
                if i <= last + 1:
                    continue
                a, b = find(int(lab[i])), find(int(lab[i + 1]))
                if a == b:
                    continue
                L[i], L[i + 1] = L[i + 1], L[i]
                parent[a] = b
                last = i
                did += 1
            if did:
                break
        swaps += did
        if not did:
            raise AssertionError("no swap of adjacent different bytes merges the remaining %d cycles" % k)


def _rle1_valid(T, full, level):
    """Whether the encoder's RLE1 stage reads T's raw input back as exactly T (one block, full or last)."""
    raw, _, pending = S.model_rle1(T)
    if pending and not full:
        return None
    starts, lens, _, blocks = O.rle1_split(raw.tobytes(), level)
    if len(lens) != 1 or int(lens[0]) != T.size or not np.array_equal(blocks[0][:T.size], T):
        return None
    return raw


def _break_runs(T, used):
    """T with every 4th byte of a run replaced, so that it has no run of four."""
    T = T.copy()
    n = T.size
    st = np.flatnonzero(np.r_[True, T[1:] != T[:-1]])
    ln = np.diff(np.r_[st, n])
    for s, l in zip(st.tolist(), ln.tolist()):
        for q in range(s + 3, s + l, 4):
            x = T[q]
            nxt = T[q + 1] if q + 1 < n else T[0]
            T[q] = next(u for u in used if u != x and u != nxt)
    return T


@dataclass
class Built:
    L: np.ndarray          # the column the encoder sees
    T: np.ndarray          # the block (RLE1 output)
    raw: np.ndarray        # raw bytes of the block
    pidx: int
    swaps: int = 0
    rle1_repair: bool = False


def build_block(ranks, used, level, full, prev_last=None, protect=None):
    """Column -> block -> raw input.  `used` is the sorted used-byte list the ranks index."""
    L, swaps = merge_cycles(unmtf(ranks, used), protect)
    repaired = False
    for attempt in range(2):
        T0 = S.model_ibwt(L, 0)[0]
        n = T0.size
        starts = np.flatnonzero(T0 != np.roll(T0, 1)) if n > 1 else np.zeros(1, np.int64)
        for s in starts.tolist()[:64]:
            T = np.roll(T0, -s)
            if prev_last is not None and T[0] == prev_last:
                continue
            raw = _rle1_valid(T, full, level)
            if raw is not None:
                Lc, pidx = O.bwt_cyclic(T.tobytes())
                assert Lc == L.tobytes()
                return Built(L, T, raw, pidx, swaps, repaired)
        T0 = _break_runs(T0, sorted(set(T0.tolist())))
        L = np.frombuffer(O.bwt_cyclic(T0.tobytes())[0], np.uint8).copy()
        repaired = True
    raise AssertionError("no rotation of the block is a valid RLE1 output")


# ---- Huffman search model ------------------------------------------------------------------------------------------
def code_lengths(freq):
    """shuff_build: sort (freq << 9 | sym), length-limited lengths by the oracle's allocator."""
    keys = sorted((int(f) << 9) | s for s, f in enumerate(freq))
    srt = O.huffman_code_lengths([k >> 9 for k in keys], MAX_LEN)
    out = [0] * len(freq)
    for k, l in zip(keys, srt):
        out[k & 511] = l
    return out


def huffman_depth(freq):
    """Depth of an unconstrained Huffman code on the non-zero frequencies."""
    h = [(int(f), i, 0) for i, f in enumerate(freq) if f]
    if len(h) < 2:
        return 1
    heapq.heapify(h)
    k = len(h)
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        heapq.heappush(h, (a[0] + b[0], k, max(a[2], b[2]) + 1))
        k += 1
    return h[0][2]


def target_tables(m):
    return 6 if m >= 2400 else 5 if m >= 1200 else 4 if m >= 600 else 3 if m >= 200 else 2


def search(sym, A):
    """The table search of one block: (selectors, tables, rounds, final).  Every assign pass (each round, and the
    final one) reports the groups tied between two tables and the largest cost of a group under any table (the 10-bit
    cost fields of huff.cu hold up to 50 x 20 = 1000); every round also reports its most-used table, whether two
    tables tied for most used, and the split: the threshold cost, how many of the table's groups sit on it, how many
    of those stay (keep_eq), and across how many 256-thread ranges they lie."""
    sym = np.asarray(sym, np.int64)
    m = sym.size
    nsel = (m + GROUP - 1) // GROUP
    G = np.zeros((nsel, A), np.int64)
    np.add.at(G, (np.arange(m) // GROUP, sym), 1)
    tables = [code_lengths(G.sum(0)), code_lengths([1] * A)]
    per = (nsel + TILE_GROUPS - 1) // TILE_GROUPS
    rounds = []
    sel = np.zeros(nsel, np.int64)
    while True:
        cost = G @ np.array(tables, np.int64).T
        sel = np.argmin(cost, axis=1)
        best = cost[np.arange(nsel), sel]
        table_ties = int(((cost == best[:, None]).sum(1) > 1).sum())
        if len(tables) >= target_tables(m):
            return sel, tables, rounds, dict(table_ties=table_ties, max_cost=int(cost.max()))
        gcount = np.bincount(sel, minlength=len(tables))
        which = int(np.argmax(gcount))
        idx = np.flatnonzero(sel == which)
        c = cost[idx, which]
        order = np.argsort(c, kind="stable")
        half = idx.size >> 1
        cstar = int(c[order[half]])
        below = int((c < cstar).sum())
        on = idx[c == cstar]
        rounds.append(dict(ng=len(tables), which=which, most_tie=int((gcount == gcount[which]).sum()) > 1,
                           table_ties=table_ties, max_cost=int(cost.max()), cstar=cstar, eq=int(on.size), keep_eq=half - below,
                           eq_threads=len(set((on // per).tolist()))))
        sel[idx[order[half:]]] = len(tables)
        F = np.zeros((len(tables) + 1, A), np.int64)
        np.add.at(F, sel, G)
        tables = [code_lengths(F[t]) for t in range(len(tables) + 1)]


# ---- rank designs --------------------------------------------------------------------------------------------------
class Design:
    """A rank sequence built piece by piece, with the positions a feature needs marked as protected.  It follows the
    MTF list (as indices into the used-byte list), so that filler can avoid a byte."""

    def __init__(self, alpha, seed):
        self.alpha = alpha
        self.g = U.rng(seed)
        self.parts, self.prot, self.n = [], [], 0
        self.lst = list(range(alpha))

    def put(self, ranks, protect=True):
        r = np.asarray(ranks, np.int32)
        assert r.size == 0 or (r.min() >= BRING_MAX and r.max() < self.alpha), "rank out of range"
        lst = self.lst
        for x in r[r != 0].tolist():
            j = x if x > 0 else lst.index(0 if x == BRING_MIN else self.alpha - 1)
            lst.insert(0, lst.pop(j))
        self.parts.append(r)
        self.prot.append(np.full(r.size, protect))
        self.n += r.size
        return self

    def fill(self, k, hi=None, p=0.25, zeros=False, avoid=()):
        """k filler ranks: 1 + geometric(p), capped at hi (default alpha - 1); no zero ranks unless `zeros`.  Ranks
        that would pick a used-byte index in `avoid` are moved off it."""
        if k <= 0:
            return self
        hi = min(hi or self.alpha - 1, self.alpha - 1)
        r = np.minimum(self.g.geometric(p, size=k), hi).astype(np.int32)
        if zeros:
            r -= 1
            r[r < 0] = 0
        if avoid:
            lst, out = self.lst, []
            for x in r.tolist():
                while x and lst[x] in avoid:
                    x = x + 1 if x < hi else 1
                if x == 0 and lst[0] in avoid:
                    x = 1
                    while lst[x] in avoid:
                        x += 1
                out.append(x)
                if x:
                    lst.insert(0, lst.pop(x))
            self.parts.append(np.array(out, np.int32))
            self.prot.append(np.zeros(k, bool))
            self.n += k
            return self
        return self.put(r, protect=False)

    def uniform(self, k, lo=1, hi=None):
        hi = min(hi or self.alpha - 1, self.alpha - 1)
        return self.put(self.g.integers(lo, hi + 1, size=k).astype(np.int32), protect=False)

    def fill_to(self, pos, **kw):
        return self.fill(pos - self.n, **kw)

    def zero_run(self, length, start=None, end=None, head=1, **kw):
        """A byte brought to the front by rank `head` and `length` zero ranks behind it, the zeros starting at `start`
        or ending (last zero) at `end`; filler up to there.  A long run of byte x is kept out of x's own F bucket
        (head BRING_MIN near the end of the block, BRING_MAX near its start, and no x in the filler that the bucket
        covers): a run inside its bucket makes LF step through it a few rows at a time, and the block T then holds
        long runs of x that are no RLE1 output."""
        first = start if start is not None else end - length + 1
        self.fill_to(first - 1, **kw)
        return self.put([head] + [0] * length)

    def ranks(self):
        return np.concatenate(self.parts) if self.parts else np.zeros(0, np.int32)

    def protect(self):
        return np.concatenate(self.prot) if self.prot else np.zeros(0, bool)


def used_bytes(alpha, seed=0):
    """A sorted used-byte list of `alpha` values, avoiding 252..255 when it can (so that no byte of a block is a count
    byte the encoder would not write)."""
    if alpha >= 253:
        return list(range(256 - alpha, 256)) if alpha < 256 else list(range(256))
    g = U.rng(seed + 7)
    return sorted(g.choice(252, size=alpha, replace=False).tolist())


# ---- cases ---------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    designs: object        # () -> [(ranks, used, protect)] per block, or raw bytes for a case built from content
    levels: tuple
    claims: list = field(default_factory=list)   # (what, predicate(info)) with info a CaseInfo


class CaseInfo:
    """What the encoder sees for one case: per block the column, block, oracle stages, ranks and the search model."""

    def __init__(self, case):
        self.case = case
        d = case.designs()
        level = case.levels[0]
        self.built = []
        if isinstance(d, (bytes, bytearray)):
            self.raw = bytes(d)
            _, lens, _, blocks = O.rle1_split(self.raw, level)
            for k, ln in enumerate(lens.tolist()):
                T = blocks[k][:ln].copy()
                L, pidx = O.bwt_cyclic(T.tobytes())
                self.built.append(Built(np.frombuffer(L, np.uint8).copy(), T, None, pidx))
        else:
            prev = None
            for k, item in enumerate(d):
                b = item if isinstance(item, Built) else build_block(*item[:2], level, k + 1 < len(d), prev, item[2])
                self.built.append(b)
                prev = b.raw[-1]
            self.raw = b"".join(b.raw.tobytes() for b in self.built)
        self.blocks = []
        for b in self.built:
            st = O.compress_block_stages(b.T.tobytes())
            st["L"], st["ranks"] = b.L, mtf_ranks(b.L) if b.L.size else np.zeros(0, np.int32)
            st["n"], st["m"] = int(b.T.size), int(st["trace"].m)
            self.blocks.append(st)

    @functools.cached_property
    def searches(self):
        return [search(st["sym"], int(st["trace"].alpha) + 2) for st in self.blocks]

    def any_block(self, f):
        return any(f(st) for st in self.blocks)


# ---- predicates ----------------------------------------------------------------------------------------------------
def _has_run(length, where):
    """A zero run of `length` that starts ("start"), ends ("end") or both ("both") on a chunk seam."""
    def f(ci):
        for st in ci.blocks:
            s, l = zero_runs(st["ranks"])
            e = s + l
            ok = (l == length) & {"start": s % CHUNK == 0, "end": e % CHUNK == 0,
                                  "both": (s % CHUNK == 0) & (e % CHUNK == 0)}[where]
            if ok.any():
                return True
        return False
    return f


def _all_zero_chunk(st):
    r = st["ranks"]
    nc = r.size // CHUNK
    return nc > 0 and bool((r[:nc * CHUNK].reshape(nc, CHUNK) == 0).all(1).any())


def _z_lead(st):
    """A run that comes into a chunk from the one before and ends inside it."""
    s, l = zero_runs(st["ranks"])
    e = s + l
    return bool(((s % CHUNK != 0) & (s // CHUNK < e // CHUNK) & (e % CHUNK != 0) & (e < st["n"])).any())


def _ends_in_run(st):
    return st["n"] > 1 and st["ranks"][-1] == 0


def _rank_at(rank, where):
    """A byte used at MTF rank `rank` at chunk offset 0 / 4095 or window lane 0 / 31 (away from chunk edges), for the
    first time in its chunk: k_mtf_ranks ranks it by the live keys of the chunk start (key 255 - rank)."""
    def f(st):
        L = st["L"]
        p = np.flatnonzero(st["ranks"] == rank)
        o = p % CHUNK
        sel = {"chunk0": o == 0, "chunk4095": o == CHUNK - 1,
               "lane0": (p % WINDOW == 0) & (o != 0), "lane31": (p % WINDOW == WINDOW - 1) & (o != CHUNK - 1)}[where]
        return any(not (L[q - q % CHUNK:q] == L[q]).any() for q in p[sel].tolist())
    return f


def _seam_reuse(gap):
    """A byte used at chunk offset 4095 - gap and again at offset 0 of the next chunk, nothing of it in between."""
    def f(st):
        L = st["L"]
        for c in range(CHUNK, L.size, CHUNK):
            a = c - 1 - gap
            if a >= 0 and L[a] == L[c] and not (L[a + 1:c] == L[c]).any():
                return True
        return False
    return f


def _far_back(chunks):
    """A byte whose previous use lies `chunks` or more chunks back."""
    def f(st):
        L = st["L"]
        last = {}
        for p in range(0, L.size):
            b = int(L[p])
            q = last.get(b)
            if q is not None and p // CHUNK - q // CHUNK >= chunks:
                return True
            last[b] = p
        return False
    return f


def _window_repeat(between):
    """A byte at lanes i and i + between + 1 of one window with `between` distinct other bytes in between."""
    def f(st):
        L = st["L"]
        for w in range(0, L.size - WINDOW + 1, WINDOW):
            x = L[w:w + WINDOW]
            for i in range(0, WINDOW - between - 1):
                j = i + between + 1
                mid = x[i + 1:j]
                if x[i] == x[j] and not (mid == x[i]).any() and np.unique(mid).size == between:
                    return True
        return False
    return f


def _sym256_last_group(st):
    nsel = int(st["trace"].nsel)
    p = np.flatnonzero(st["sym"] == 256)
    return st["m"] % GROUP != 0 and bool((p >= GROUP * (nsel - 1)).any())


def _limit_binds(st):
    A = int(st["trace"].alpha) + 2
    return huffman_depth(np.bincount(st["sym"], minlength=A)) > MAX_LEN and int(st["lens"].max()) == MAX_LEN


def _thread_runs(st, distinct):
    sel = st["sel"]
    per = (sel.size + TILE_GROUPS - 1) // TILE_GROUPS
    return sum(np.unique(sel[t * per:(t + 1) * per]).size >= distinct for t in range(TILE_GROUPS))


def each(f):
    return lambda ci: ci.any_block(f)


def on_block(k, f):
    return lambda ci: f(ci.blocks[k])


def _search_round(ci, f):
    return any(f(r) for sr in ci.searches for r in sr[2])


def _max_cost(ci, cost):
    """Some group costs `cost` under some table in some assign pass of the search."""
    return any(r["max_cost"] == cost for sr in ci.searches for r in sr[2] + [sr[3]])


def _equal_freqs(count):
    """`count` or more used symbols (MTF ranks 1..alpha-1, EOB) share one non-zero frequency."""
    def f(st):
        A = int(st["trace"].alpha) + 2
        h = np.bincount(st["sym"], minlength=A)[2:]
        return int(np.bincount(h[h > 0]).max()) >= count
    return f


# ---- designs -------------------------------------------------------------------------------------------------------
def _mixed(alpha, n, seed, zeros=True):
    d = Design(alpha, seed)
    while d.n < n:
        d.fill(min(int(d.g.integers(20, 400)), n - d.n), p=float(d.g.choice([0.6, 0.3, 0.1])), zeros=zeros)
    return d


def _plants(d, n, rank_hi, zeros=True, nchunks=None):
    """Filler of ranks below rank_hi, with, in turn at every chunk: first uses at ranks 127, 128 and 255 at chunk
    offset 0 (every other chunk), lane 31 of a window, lane 0 of a window and chunk offset 4095; a byte used at offset 4095 (or 4094)
    and again at offset 0 of the next chunk; windows where a byte comes back after 1, 15 and 30 other bytes."""
    ranks = [r for r in (127, 128, 255) if r < d.alpha]
    d.put(list(range(1, d.alpha)), protect=False)    # every byte once, in list order: the alphabet stays whole
    c = 1
    while (c + 2) * CHUNK <= n and (nchunks is None or c <= nchunks):
        base = c * CHUNK
        r = ranks[c % len(ranks)]
        if c % 2 == 1:
            d.fill_to(base, hi=rank_hi, zeros=zeros, p=0.02)
            d.put([r])
        d.fill_to(base + 5 * WINDOW + 31, hi=rank_hi, zeros=zeros, p=0.02)
        d.put([r])
        d.fill_to(base + 9 * WINDOW, hi=rank_hi, zeros=zeros, p=0.02)
        d.put([r])
        k = (1, 15, 30)[c % 3]
        d.fill_to(base + 20 * WINDOW + 31 - (k + 1), hi=rank_hi, zeros=zeros, p=0.02)
        d.put([40] * (k + 1) + [k])
        d.fill_to(base + CHUNK - 2, hi=rank_hi, zeros=zeros, p=0.02)
        if c % 4 == 1:
            d.put([r, 1, 1])          # x at 4094, y at 4095, x at offset 0 of the next chunk (rank 1)
        elif c % 4 == 3:
            d.put([1, r, 0])          # x at 4095, x again at offset 0 (rank 0)
        c += 1
    return d


def _tune(make, m_want):
    """Ranks of a no-zero design whose block has m symbols: the design length is moved until the built block has."""
    n, seen = m_want - 1, set()
    for _ in range(40):
        while n in seen:
            n += 1
        seen.add(n)
        d = make(n)
        b = build_block(d.ranks(), used_bytes(d.alpha, d.alpha), 9, False, None, d.protect())
        m = int(O.compress_block_stages(b.T.tobytes())["trace"].m)
        if m == m_want:
            return [(d.ranks(), used_bytes(d.alpha, d.alpha), d.protect())]
        n += m_want - m
    raise AssertionError("could not reach m = %d" % m_want)


def _eob(alpha, r):
    """No zero ranks, every byte used: m = n + 1 moved until the end of block sits at residue r of its group."""
    def make(n):
        d = Design(alpha, 300 + alpha + r)
        d.put(list(range(alpha - 1, 0, -1)))
        return d.uniform(n - d.n)
    return lambda: _tune(make, 6000 + (r + 1) % GROUP)


def _rank255_last():
    def make(n):
        d = Design(256, 5)
        d.put(list(range(255, 0, -1)))
        d.uniform(n - 7 - d.n)
        return d.put([255]).uniform(6)
    return _tune(make, 3021)


def _m_case(m):
    """No zero ranks (m = n + 1 up to the swaps of the cycle merge), ranks 1..29 with designed Zipf frequencies
    (rank j about n / (j H_29) times, rank 1 taking the rest) in a seeded order."""
    def make(n):
        w = 1.0 / np.arange(1, 30)
        c = np.floor(n * w / w.sum()).astype(np.int64)
        c[0] += n - c.sum()
        ranks = np.repeat(np.arange(1, 30, dtype=np.int32), c)
        U.rng(m).shuffle(ranks)
        return Design(30, m).put(ranks, protect=False)
    return lambda: _tune(make, m)


def _fib(level):
    """Fibonacci frequencies from (3, 3) over ranks 1..25: the unconstrained Huffman depth is 24, so the limit of 20
    binds.  No zero ranks: RUNA and RUNB have frequency 0."""
    g = U.rng(61)
    f = [3, 3]
    while len(f) < 25:
        f.append(f[-1] + f[-2])
    ranks = np.repeat(np.arange(1, 26, dtype=np.int32), f)
    g.shuffle(ranks)
    d = Design(26, 61).put(ranks, protect=False)
    return [(d.ranks(), used_bytes(26, 61), d.protect())]


def _group_1000(seed):
    """A group of fifty 20-bit codes: 64 ranks used once each (65 symbols of frequency 1 with the end of block)
    beside a backbone of ranks 1..14 with frequencies 65 F(k) (Fibonacci).  Fifty of the rare ranks, in ascending
    order (each picks a byte no other rare rank picks), fill one aligned group.  Once the split has moved the groups
    of the backbone to tables of their own, the tables built from them give the rare symbols (frequency 0 there) the
    deepest codes, 20 bits, and the rare group costs 50 x 20 = 1000 bits under them in the later assign passes."""
    g = U.rng(81 + seed)
    f = [1, 1]
    while len(f) < 14:
        f.append(f[-1] + f[-2])
    ranks = np.repeat(np.arange(1, 15, dtype=np.int32), 65 * np.array(f))
    g.shuffle(ranks)
    k = ranks.size // 2 // GROUP * GROUP
    d = Design(79, 81)
    d.put(ranks[:k], protect=False)
    d.put(np.arange(15, 65, dtype=np.int32))
    d.put(ranks[k:], protect=False)
    d.put(np.arange(65, 79, dtype=np.int32))
    d.put(ranks[:GROUP * 3], protect=False)
    return d.ranks(), used_bytes(79, 81 + seed), d.protect()


def _six_tables(n, seed, plants):
    """Groups from six different rank distributions in random order (all six tables in use, with long recency
    histories in every thread's run of selectors), and the rank plants of `_plants`."""
    d = Design(256, seed)
    if plants:
        _plants(d, n, 60, zeros=False, nchunks=40)
    ps = [0.7, 0.4, 0.2, 0.08, 0.03]
    while d.n < n:
        k = min(int(d.g.integers(1, 6)) * GROUP, n - d.n)
        c = int(d.g.integers(0, 6))
        if c == 5:
            d.uniform(k)
        else:
            d.fill(k, p=ps[c])
    return d


def _most_tie(seed):
    """Groups of two kinds, skewed ranks and uniform ranks, as many of each: the global and the flat table tie for
    most used in the first round."""
    d = Design(40, seed)
    for k in range(8):
        d.fill(GROUP, p=0.6)
        d.uniform(GROUP)
    return [(d.ranks(), used_bytes(40, seed), d.protect())]


def _zero_runs(specs, n, seed, alpha=40):
    """Zero runs (length, where) in order, each on its own chunk seam: runs in the first half of the block are of the
    largest used byte, in the second half of the smallest, and the near-uniform filler holds neither, so that no run
    lies in its own byte's F bucket and T has few runs of four."""
    d = Design(alpha, seed)
    kw = dict(p=0.02, avoid=(0, alpha - 1))
    d.fill(CHUNK // 2, **kw)
    for length, where in specs:
        head = BRING_MAX if d.n < n // 2 else BRING_MIN
        if where == "end":
            seam = (d.n + length + 2 + CHUNK - 1) // CHUNK * CHUNK
            d.zero_run(length, end=seam - 1, head=head, **kw)
        else:
            d.zero_run(length, start=(d.n + CHUNK + 2) // CHUNK * CHUNK, head=head, **kw)
    d.fill_to(n - 800, **kw)
    return d


SMALL_RUNS = [(2 ** k + o, ("start", "end")[(k + o) % 2] if (2 ** k + o) % CHUNK else "both")
              for k in range(1, 13) for o in (-2, -1, 0, 1) if 2 ** k + o > 0]
BIG_RUNS = [(2 ** k + o, "both" if o == 0 else ("start", "end")[(k + o) % 2]) for k in range(13, 20) for o in (-2, -1, 0, 1)]


def _small_runs():
    def make(seed):
        d = _zero_runs(SMALL_RUNS, 2 * len(SMALL_RUNS) * CHUNK, 71 + 100 * seed)
        seam = (d.n + CHUNK + 200) // CHUNK * CHUNK
        d.zero_run(300, start=seam - 100, head=BRING_MIN, p=0.02, avoid=(0, 39))   # comes into a chunk (z_lead)
        d.fill(3000, p=0.02, avoid=(0, 39))
        d.put([BRING_MIN] + [0] * 777)     # the block ends inside a run
        return d.ranks(), used_bytes(40, 71 + 100 * seed), d.protect()
    return [_retry(make, 9, False)]


def _big_runs(k, level=9):
    """Runs of 2^k - 2 .. 2^k + 1 zeros, as many to a full block as fit."""
    BS = block_size(level)
    runs = [(l, w) for l, w in BIG_RUNS if l in range(2 ** k - 2, 2 ** k + 2)]
    per = max(1, (BS - 3 * CHUNK) // (2 ** k + 2 * CHUNK))
    blocks = []
    for i in range(0, len(runs), per):
        d = _zero_runs(runs[i:i + per], BS, 300 + k * 8 + i) if per > 1 else None
        if d is None:    # one run per block: the smallest byte, ending on the block's last chunk seam or starting
            l, w = runs[i]   # so that it ends on or in front of it
            d = Design(40, 300 + k * 8 + i)
            last_seam = (BS - 1500) // CHUNK * CHUNK
            kw = dict(p=0.02, avoid=(0,))
            if w == "end":
                d.zero_run(l, end=last_seam - 1, head=BRING_MIN, **kw)
            else:
                d.zero_run(l, start=(last_seam - l) // CHUNK * CHUNK, head=BRING_MIN, **kw)
        d.fill_to(BS, p=0.02, avoid=(0,))
        blocks.append((d.ranks(), used_bytes(40, 300 + k * 8 + i), d.protect()))
    return blocks


def _big_runs_block(k):
    """2^13 and 2^14: all four runs in one full block, with a design that needs no RLE1 repair."""
    runs = [(l, w) for l, w in BIG_RUNS if l in range(2 ** k - 2, 2 ** k + 2)]

    def make(seed):
        d = _zero_runs(runs, block_size(9), 300 + k * 8 + 100 * seed)
        d.fill_to(block_size(9), p=0.02, avoid=(0, 39))
        return d.ranks(), used_bytes(40, 300 + k * 8 + 100 * seed), d.protect()
    return [_retry(make, 9, False)]


def _retry(make, level, full, tries=8):
    """Build make(seed) for seeds 0, 1, ... until the block needs no RLE1 repair (the repair moves the whole column)."""
    for seed in range(tries):
        ranks, used, prot = make(seed)
        b = build_block(ranks, used, level, full, None, prot)
        if not b.rle1_repair:
            break
    return b


def _small(n, alpha, seed):
    d = _mixed(alpha, n, seed)
    return [(d.ranks(), used_bytes(alpha, seed), d.protect())]


@functools.lru_cache(maxsize=1)
def cases():
    cs = []
    for r in (0, 1, 31, 32, 33):
        n = 3 * CHUNK + r
        cs.append(Case("len_4096k_plus_%d" % r, (lambda n=n: _small(n, 64, n)), (1, 9),
                       [("n = %d (mod 4096)" % r, on_block(0, lambda st, r=r: st["n"] % CHUNK == r))]))
    for n, alpha in ((17, 8), (CHUNK, 64)):
        cs.append(Case("len_%d" % n, (lambda n=n, a=alpha: _small(n, a, n)), (1,),
                       [("n = %d" % n, on_block(0, lambda st, n=n: st["n"] == n))]))
    plant_claims = [("first use at rank %d at %s" % (r, w), each(_rank_at(r, w)))
                    for r in (127, 128, 255) for w in ("chunk0", "chunk4095", "lane0", "lane31")]
    plant_claims += [("a byte used at chunk offset %d and again at offset 0 of the next chunk" % (4095 - gap), each(_seam_reuse(gap)))
                     for gap in (0, 1)]
    plant_claims += [("a byte whose previous use is 8+ chunks back", each(_far_back(8)))]
    plant_claims += [("a byte back in its window after %d distinct bytes" % k, each(_window_repeat(k))) for k in (1, 15, 30)]
    def plants_l1(seed):
        d = _plants(Design(256, 11 + 100 * seed), block_size(1), 60, zeros=False).fill_to(block_size(1), hi=60, p=0.02)
        return d.ranks(), list(range(256)), None
    cs.append(Case("blocksize_l1", lambda: [_retry(plants_l1, 1, True)] + _small(5000, 256, 12), (1,),
                   [("first block n = blockSize", on_block(0, lambda st: st["n"] == block_size(1)))] + plant_claims))
    six = [("n = blockSize, nsel near 18000", on_block(0, lambda st: st["n"] == block_size(9) and int(st["trace"].nsel) >= 17900)),
           ("all six tables in use", on_block(0, lambda st: int(st["trace"].ngroups) == 6 and np.unique(st["sel"]).size == 6)),
           ("200+ of the 256 thread runs of the selector MTF use 4+ tables", on_block(0, lambda st: _thread_runs(st, 4) >= 200)),
           ("many groups tie at the split threshold across thread ranges, keep_eq splits them",
            lambda ci: _search_round(ci, lambda r: r["eq"] >= 64 and r["eq_threads"] >= 16 and 0 < r["keep_eq"] < r["eq"])),
           ("groups cost the same under two tables", lambda ci: any(sr[3]["table_ties"] > 0 for sr in ci.searches))]
    def six_l9(seed):
        return _six_tables(block_size(9), 13 + 100 * seed, True).ranks(), list(range(256)), None
    cs.append(Case("blocksize_l9_six_tables", lambda: [_retry(six_l9, 9, False)], (9,),
                   six + plant_claims))
    cs.append(Case("zero_runs_small", _small_runs, (9,),
                   [("zero run of %d %s on a chunk seam" % (l, w), _has_run(l, w)) for l, w in SMALL_RUNS] +
                   [("a run comes into a chunk and ends inside it (z_lead)", each(_z_lead)),
                    ("the block ends inside a run", each(_ends_in_run)),
                    ("a run covers a whole chunk", each(_all_zero_chunk))]))
    for k in range(13, 20):
        runs = [(l, w) for l, w in BIG_RUNS if l in range(2 ** k - 2, 2 ** k + 2)]
        cs.append(Case("zero_runs_2^%d" % k, (lambda k=k: _big_runs_block(k) if k < 15 else _big_runs(k)), (9,),
                       [("zero run of %d %s on a chunk seam" % (l, w), _has_run(l, w)) for l, w in runs] +
                       [("first blocks at blockSize", lambda ci: all(st["n"] == block_size(9) for st in ci.blocks[:-1])),
                        ("a run covers whole chunks", each(_all_zero_chunk))]))
    # The longest zero run a block can have beside one other symbol: T = "aaaa" + count 'b', L = "baaaa", ranks
    # [1, 1, 0, 0, 0].  A run over all of L but its first byte needs L[1:] == L[0], i.e. a block of one byte value; with
    # two, the second byte's first use has a non-zero rank too.  A longer block of two byte values with one long run of
    # L is no RLE1 output (its block T would hold a run of five or more).
    cs.append(Case("alphabet_2_run_behind_two_bytes", lambda: b"a" * 102, (1, 9),
                   [("alphabet of 2, ranks 1, 1, 0, 0, 0", on_block(0, lambda st: int(st["trace"].alpha) == 2 and
                                                                    st["ranks"].tolist() == [1, 1, 0, 0, 0])),
                    ("the block ends inside a run", on_block(0, _ends_in_run))]))
    for n in (1, 3):
        cs.append(Case("alphabet_1_n%d" % n, (lambda n=n: b"q" * n), (1,),
                       [("alphabet of 1", on_block(0, lambda st: int(st["trace"].alpha) == 1))]))
    for alpha in (255, 256):
        for r in (0, 1, 49):
            cs.append(Case("alphabet_%d_eob_at_%d" % (alpha, r), _eob(alpha, r), (1, 9),
                           [("alphabet %d" % alpha, on_block(0, lambda st, a=alpha: int(st["trace"].alpha) == a)),
                            ("end of block at group residue %d" % r,
                             on_block(0, lambda st, r=r, a=alpha: (st["m"] - 1) % GROUP == r and int(st["sym"][-1]) == a + 1))]))
    cs.append(Case("rank255_in_last_group", _rank255_last, (9,),
                   [("symbol 256 in the last, partial group", on_block(0, _sym256_last_group))]))
    for m in (199, 200, 201, 599, 600, 1199, 1200, 2399, 2400, 2401):
        cs.append(Case("m_%d" % m, _m_case(m), (9,),
                       [("m = %d" % m, on_block(0, lambda st, m=m: st["m"] == m)),
                        ("%d tables" % target_tables(m), on_block(0, lambda st, m=m: int(st["trace"].ngroups) == target_tables(m)))]))
    for nsel in (256, 257, 511):
        cs.append(Case("nsel_%d" % nsel, _m_case(50 * nsel - (0 if nsel % 2 == 0 else 49)), (9,),
                       [("nsel = %d" % nsel, on_block(0, lambda st, k=nsel: int(st["trace"].nsel) == k))]))
    cs.append(Case("fibonacci_limit20", lambda: _fib(9), (9,),
                   [("global depth > 20 and the limit binds", on_block(0, _limit_binds)),
                    ("symbols of frequency 0", on_block(0, lambda st: (np.bincount(st["sym"], minlength=int(st["trace"].alpha) + 2) == 0).any())),
                    ("groups cost the same under two tables", lambda ci: ci.searches[0][3]["table_ties"] > 0)]))
    cs.append(Case("group_of_1000_bits", lambda: [_retry(_group_1000, 9, False)], (1, 9),
                   [("a group costs 1000 bits under a table", lambda ci: _max_cost(ci, 1000)),
                    ("48+ used symbols of equal frequency", on_block(0, _equal_freqs(48))),
                    ("the limit of 20 bits is reached", on_block(0, lambda st: int(st["lens"].max()) == MAX_LEN))]))
    cs.append(Case("most_used_tie", lambda: _most_tie(5), (9,),   # seed 5: found by search, the two kinds tie
                   [("two tables tie for most used", lambda ci: _search_round(ci, lambda r: r["most_tie"]))]))
    return cs


def case(name):
    return next(c for c in cases() if c.name == name)


@functools.lru_cache(maxsize=None)
def info(name):
    return CaseInfo(case(name))
