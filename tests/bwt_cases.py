"""Forward-BWT case corpus and a CPU model of how bwt_forward_batch (csrc/bwt.cu) finishes each batch.

A batch of blocks ends in one of four ways: the MSD scatter + shared-memory bucket sort with 5-byte ties ordered by
k_resolve_direct (bwt_msd.cu), the 4-byte LSD sort + k_emit_detect + k_resolve_direct, the rank-based prefix-doubling
rounds, or the 8-byte ("wide") initial sort followed by the rounds.  Which one runs depends on the data, so an input
exercises one path only.  The cases below are built from fixed seeds to sit on the thresholds of each path, and
`predict` restates the selection rules in numpy so that a test can say which path every batch must take.  The
library reports the path through b2_stats (bwt_msd_done, bwt_direct_done, bwt_rounds_batches, bwt_wide_batches and
the fallback bits).

The rules mirrored (bwt.cu unless noted):
- k_text_score: score = mean over the batch's blocks (empty ones included) of n * (sum p_c^2)^4.  The first batch of
  a call runs in the mode of its own score, every later batch in the mode of the batch before it (score > 0.5:
  wide); B2_BWT_PREFIX8 forces the mode.
- bwt_msd.cu k_msd_prep: a (block, first byte) bucket larger than MB_CAP = 10238 gives up (bit 1).
- bwt_msd.cu k_msd_bucket: records ordered by key = (k * S) >> 32 of their symbols 1..4 (dense ranks r, base a = the
  block's alphabet, S = floor((2^64 - 1) / a^4), or 2^32 when a^4 >= 2^32); a cell (key >> 18) of more than
  MB_MAXCELL = 512 records gives up (bit 2).
- bwt_forward_batch: a tie list (members of groups equal on h0 bytes) longer than n_total / 8 gives up (bit 4).
- k_resolve_direct: a group of more than RD_MAXGROUP = 16 members (bit 8), or two rotations equal on h0 + 64 bytes
  (bit 16).  h0 = 5 on the MSD path, 4 on the LSD path.  Insertion sort compares every pair that ends up adjacent,
  so the depth is the longest common prefix of neighbours in the sorted order, taken here from the oracle.
"""
import functools
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle as O
from tests import util as T

MB_CAP, MB_MAXCELL, CELL_SHIFT = 10238, 512, 18
RD_MAXGROUP, RD_DEPTH = 16, 64
RR_TILE = 2048
WHY_BUCKET, WHY_CELL, WHY_TIES, WHY_GROUP, WHY_DEPTH = 1, 2, 4, 8, 16
LCP_CAP = 80  # > 5 + RD_DEPTH: deeper common prefixes only need to be known as "too deep"


def cyclic_order(blk):
    """Rotation order of the block (what the oracle's bwt_cyclic sorts): suffixes of the doubled block below n."""
    n = len(blk)
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    sa = np.asarray(O.suffixsort(blk + blk), dtype=np.int64)
    return sa[sa < n]


def _lcp(t, n, x, y):
    """Longest common prefix (capped at LCP_CAP) of the rotations x[i], y[i] of block t."""
    out = np.empty(x.size, dtype=np.int64)
    d = np.arange(LCP_CAP, dtype=np.int64)
    for s in range(0, x.size, 1 << 15):
        xs, ys = x[s:s + (1 << 15), None], y[s:s + (1 << 15), None]
        ne = t[(xs + d) % n] != t[(ys + d) % n]
        out[s:s + xs.shape[0]] = np.where(ne.any(axis=1), ne.argmax(axis=1), LCP_CAP)
    return out


@dataclass
class Ties:
    """Groups of rotations equal on their first h0 bytes, in sorted order."""
    members: int = 0      # length of the tie list
    max_group: int = 0
    depth: int = 0        # deepest common prefix of neighbours inside a group of <= RD_MAXGROUP members
    rot0_group: int = 1   # size of the group rotation 0 is in (1: none)
    straddles: bool = False  # a group crosses a RR_TILE row boundary


def _ties(t, n, key, sa):
    ks = key[sa]
    brk = np.flatnonzero(ks[1:] != ks[:-1]) + 1
    starts = np.concatenate(([0], brk))
    sizes = np.diff(np.concatenate((starts, [n])))
    res = Ties()
    multi = sizes > 1
    if not multi.any():
        return res
    res.members = int(sizes[multi].sum())
    res.max_group = int(sizes.max())
    ends = starts + sizes - 1
    res.straddles = bool(((starts // RR_TILE) != (ends // RR_TILE))[multi].any())
    row0 = int(np.flatnonzero(sa == 0)[0])
    res.rot0_group = int(sizes[np.searchsorted(starts, row0, side="right") - 1])
    small = multi & (sizes <= RD_MAXGROUP)
    if small.any():
        grp = np.repeat(np.arange(sizes.size), sizes)
        j = np.flatnonzero(small[grp[:-1]] & (grp[:-1] == grp[1:]))
        res.depth = int(_lcp(t, n, sa[j], sa[j + 1]).max())
    return res


@dataclass
class BlockModel:
    n: int
    score: float = 0.0
    alphabet: int = 0
    bucket_max: int = 0
    cell_max: int = 0
    rot0_cell: int = 0       # records in the cell of rotation 0
    t5: Ties = field(default_factory=Ties)
    t4: Ties = field(default_factory=Ties)


def msd_keys(t, a, lut):
    """bwt_msd.cu k_msd_prep / k_msd_scatter: the scaled base-a key of symbols 1..4 of every rotation."""
    n = t.size
    i = np.arange(n, dtype=np.int64)
    r = [lut[t[(i + j) % n]].astype(np.uint64) for j in (1, 2, 3, 4)]
    a = np.uint64(a)
    k = ((r[0] * a + r[1]) * a * a + r[2] * a + r[3])
    a4 = int(a) ** 4
    S = 1 << 32 if a4 >= 1 << 32 else (2 ** 64 - 1) // a4
    s_hi, s_lo = np.uint64(S >> 32), np.uint64(S & 0xffffffff)
    return (k * s_hi + ((k * s_lo) >> np.uint64(32))) & np.uint64(0xffffffff)


def model_block(blk, sa=None):
    n = len(blk)
    m = BlockModel(n)
    if n == 0:
        return m
    t = np.frombuffer(blk, dtype=np.uint8)
    hist = np.bincount(t, minlength=256)
    p = hist / n
    m.score = float(n * float(p @ p) ** 4)
    m.alphabet = int((hist > 0).sum())
    m.bucket_max = int(hist.max())
    lut = (np.cumsum(hist > 0) - 1).astype(np.int64)
    key = msd_keys(t, m.alphabet, lut)
    cell = (t.astype(np.int64) << 14) | (key >> np.uint64(CELL_SHIFT)).astype(np.int64)
    cc = np.bincount(cell, minlength=256 << 14)
    m.cell_max = int(cc.max())
    m.rot0_cell = int(cc[cell[0]])
    sa = cyclic_order(blk) if sa is None else sa
    i = np.arange(n, dtype=np.int64)
    k4 = np.zeros(n, dtype=np.int64)
    for j in range(4):
        k4 = (k4 << 8) | t[(i + j) % n]
    k5 = (k4 << 8) | t[(i + 4) % n]
    m.t5 = _ties(t, n, k5, sa)
    m.t4 = _ties(t, n, k4, sa)
    return m


@dataclass
class Counters:
    """What b2_stats reports for one call (the bwt_* fields and msd_launches)."""
    msd_launches: int = 0
    bwt_msd_done: int = 0
    bwt_direct_done: int = 0
    bwt_rounds_batches: int = 0
    bwt_wide_batches: int = 0
    bwt_msd_fallback_why: int = 0
    bwt_direct_fallback_why: int = 0
    batches: list = field(default_factory=list)  # per batch: (wide, finish, msd why, direct why, score)

    FIELDS = ("msd_launches", "bwt_msd_done", "bwt_direct_done", "bwt_rounds_batches", "bwt_wide_batches",
              "bwt_msd_fallback_why", "bwt_direct_fallback_why")

    def as_tuple(self):
        return tuple(getattr(self, f) for f in self.FIELDS)


def _direct_why(ties, n_total, h0):
    if sum(t.members for t in ties) > n_total // 8:
        return WHY_TIES
    why = WHY_GROUP if any(t.max_group > RD_MAXGROUP for t in ties) else 0
    return why | (WHY_DEPTH if any(t.depth >= h0 + RD_DEPTH for t in ties) else 0)


def predict(models, batch, msd=True, prefix8=None):
    """Counters of one b2_bwt_cyclic_batch call over blocks with these models, `batch` blocks per batch."""
    c = Counters()
    wide_next = None  # mode of the next batch, once a batch of this call has run
    for k0 in range(0, len(models), batch):
        ms = models[k0:k0 + batch]
        n_total = sum(m.n for m in ms)
        if n_total == 0:
            continue
        score = sum(m.score for m in ms) / len(ms)
        wide = bool(prefix8) if prefix8 is not None else (score > 0.5 if wide_next is None else wide_next)
        wide_next = score > 0.5
        mwhy = dwhy = 0
        if wide:
            c.bwt_wide_batches += 1
            finish = "rounds"
        else:
            finish = None
            if msd:
                c.msd_launches += 1
                if max(m.bucket_max for m in ms) > MB_CAP:
                    mwhy = WHY_BUCKET
                elif max(m.cell_max for m in ms) > MB_MAXCELL:
                    mwhy = WHY_CELL
                else:
                    mwhy = _direct_why([m.t5 for m in ms], n_total, 5)
                finish = None if mwhy else "msd"
            if finish is None:
                dwhy = _direct_why([m.t4 for m in ms], n_total, 4)
                finish = None if dwhy else "direct"
            finish = finish or "rounds"
        c.bwt_msd_fallback_why |= mwhy
        c.bwt_direct_fallback_why |= dwhy
        c.bwt_msd_done += finish == "msd"
        c.bwt_direct_done += finish == "direct"
        c.bwt_rounds_batches += finish == "rounds"
        c.batches.append((wide, finish, mwhy, dwhy, score))
    return c


# ---- the corpus ---------------------------------------------------------------------------------------------------
ASCII = np.frombuffer(bytes(range(32, 126)) + b"\n", dtype=np.uint8)  # T.ascii_random's 95 symbols


def ascii_arr(n, seed):
    return np.frombuffer(T.ascii_random(n, seed), dtype=np.uint8).copy()


def _rand_ascii(g, k):
    return ASCII[g.integers(0, ASCII.size, size=k)]


def bucket_block(target, seed, n=900000, byte=ord("A")):
    """A 900k ASCII block whose bucket of `byte` holds exactly `target` records."""
    a = ascii_arr(n, seed)
    g = T.rng(seed)
    have = int((a == byte).sum())
    pos = g.permutation(np.flatnonzero(a != byte))[:target - have]
    a[pos] = byte
    return a.tobytes()


def planted_cell_block(size, seed, n=100000, at0=True):
    """An ASCII block whose rotation 0 (at0) or some rotation sits in a cell of exactly `size` records: the 4-gram
    'QRST' between two symbols that each cycle through the other 94, `size` times (one cell of the 'Q' bucket: the keys that follow
    differ in their last symbol only, so 5-byte tie groups stay at ceil(size / 94) members).  The 'Q' bucket holds the
    plants only; the seed search finds a cell that no key boundary splits."""
    rest = ASCII[ASCII != ord("Q")]
    for s in range(seed, seed + 200):
        g = T.rng(s)
        a = ascii_arr(n, s)
        a[a == ord("Q")] = ord("q")  # the 'Q' bucket holds the plants only
        slots = g.choice(n // 8 - 1, size=size, replace=False) * 8 + 8
        if at0:
            slots[0] = 0
        for k, p in enumerate(slots):
            a[p:p + 4] = np.frombuffer(b"QRST", dtype=np.uint8)
            a[p + 4] = rest[k % rest.size]
            a[p - 1] = rest[3 * k % rest.size]
        b = a.tobytes()
        m = model_block(b)
        if (m.rot0_cell == size) if at0 else (m.cell_max == size):
            return b
    raise AssertionError("no seed gives a cell of %d" % size)


def singleton_rot0_block(seed, n=100000):
    for s in range(seed, seed + 200):
        b = T.ascii_random(n, s)
        if model_block(b).rot0_cell == 1:
            return b
    raise AssertionError("no seed")


def plant_repeat(a, g, length, copies, pos=None):
    """Write one random ASCII string of `length` bytes at `copies` places, so that the rotations starting there share
    exactly `length` bytes: the bytes before and after the copies all differ."""
    n = a.size
    s = _rand_ascii(g, length)
    pos = pos if pos is not None else np.sort(g.choice(n // (length + 4) - 2, size=copies, replace=False) + 1) * (length + 4)
    for k, p in enumerate(pos):
        a[p:p + length] = s
        a[p - 1] = ASCII[k % ASCII.size]
        a[p + length] = ASCII[(k + 7) % ASCII.size]
    return a


def repeat_block(length, copies, seed, n=100000, base=None):
    a = ascii_arr(n, seed) if base is None else np.frombuffer(base, dtype=np.uint8).copy()
    return plant_repeat(a, T.rng(seed + 1), length, copies).tobytes()


def tie_list_block(n_over, seed, n=100000):
    """An ASCII block with a 5-byte tie list of exactly n // 8 + n_over members: pairs of random 5-grams followed by
    random bytes, topped up by a third copy of one 5-gram."""
    target = n // 8 + n_over
    for s in range(seed, seed + 50):
        g = T.rng(s)
        a = ascii_arr(n, s)
        slots = iter(g.permutation(n // 8 - 2) * 8 + 8)
        gram = None

        def plant(k, fresh=True):
            nonlocal gram
            gram = _rand_ascii(g, 5) if fresh else gram
            for _ in range(k):
                p = next(slots)
                a[p:p + 5] = gram
        for _ in range(100):
            d = target - model_block(a.tobytes()).t5.members
            if d == 0:
                return a.tobytes()
            if d < 0:
                break
            if d == 1:
                plant(1, fresh=False)  # a third copy of the last pair adds 1
            for _ in range(max(d * 9 // 20, 1) if d > 1 else 0):
                plant(2)  # a fresh pair adds 2, a little more when it meets a neighbour: approach from below
    raise AssertionError("no seed gives a tie list of %d" % target)


def alphabet_block(a_size, n, seed):
    """Uniform random bytes over `a_size` symbols, 0x00 and 0xff among them."""
    g = T.rng(seed)
    mid = g.permutation(np.arange(1, 255))[:max(a_size - 2, 0)]
    syms = np.concatenate(([0, 255][:min(a_size, 2)], mid)).astype(np.uint8)
    assert np.unique(syms).size == a_size
    d = syms[g.integers(0, a_size, size=n)]
    d[:a_size] = syms  # every symbol in use
    return d.tobytes()


def periodic(p, n, seed, near=False):
    g = T.rng(seed)
    unit = _rand_ascii(g, p) if p > 3 else np.frombuffer(b"abc"[:p], dtype=np.uint8)
    a = np.resize(unit, n)
    if near:
        a[int(g.integers(0, n))] ^= 1
    return a.tobytes()


@dataclass
class Case:
    name: str
    blocks: list
    claims: list = field(default_factory=list)  # (description, predicate over the case's Model)
    compress: bool = False  # also compare a level-9 Bzip2.compressFile of the joined blocks with the oracle


class Model:
    """Block models of a case and its predicted counters under a configuration."""

    def __init__(self, case, sas=None):
        self.case = case
        self.blocks = [model_block(b, None if sas is None else sas[k]) for k, b in enumerate(case.blocks)]

    def predict(self, batch=264, msd=True, prefix8=None):
        return predict(self.blocks, batch, msd, prefix8)

    def margin_ok(self, batch):
        """The kernel sums the score in float32: every batch stays >= 10 % away from the 0.5 threshold."""
        return all(abs(s - 0.5) >= 0.05 for *_, s in self.predict(batch).batches)


def _finish(model, *want, **cfg):
    return [b[1] for b in model.predict(**cfg).batches] == list(want)


def _wrong_modes(model, batch):
    bs = model.predict(batch).batches
    return len(bs) > 2 and all(w != (s > 0.5) for w, _, _, _, s in bs[1:])


@functools.lru_cache(maxsize=1)
def cases():
    """The corpus (built once per process)."""
    C = []
    # -- (block, first byte) buckets at MB_CAP - 1, MB_CAP, MB_CAP + 1 (the last one ends in the LSD direct finish) --
    for tgt in (MB_CAP - 1, MB_CAP, MB_CAP + 1):
        claims = [("bucket of %d" % tgt, lambda m, t=tgt: m.blocks[0].bucket_max == t)]
        if tgt <= MB_CAP:
            claims.append(("MSD finish", lambda m: _finish(m, "msd")))
        else:
            claims += [("LSD direct finish by default", lambda m: _finish(m, "direct")),
                       ("MSD gave up on the bucket", lambda m: m.predict().bwt_msd_fallback_why == WHY_BUCKET),
                       ("a 4-byte tie group straddles a RR_TILE row boundary", lambda m: m.blocks[0].t4.straddles)]
        C.append(Case("bucket_%d" % tgt, [bucket_block(tgt, 11 + tgt)], claims, compress=tgt > MB_CAP))
    # -- interpolation cells at MB_MAXCELL and MB_MAXCELL + 1, made with a planted 4-gram --
    C.append(Case("cell_512", [planted_cell_block(512, 500, n=300000, at0=False)],
                  [("cell of 512", lambda m: m.blocks[0].cell_max == 512), ("MSD finish", lambda m: _finish(m, "msd"))]))
    C.append(Case("cell_513", [planted_cell_block(513, 600, n=300000, at0=False)],
                  [("cell of 513", lambda m: m.blocks[0].cell_max == 513),
                   ("MSD gave up on the cell", lambda m: m.predict().bwt_msd_fallback_why == WHY_CELL)]))
    # -- rotation 0 in every kind of cell (singleton, small_cell<2/3/4>, big_cell) and in a resolved tie group --
    sizes = (2, 3, 4, 5, 32, 33, 512)
    rot0 = [singleton_rot0_block(700)] + [planted_cell_block(k, 710 + k) for k in sizes]
    tie0 = plant_repeat(ascii_arr(100000, 790), T.rng(791), 9, 2, pos=[0, 50000]).tobytes()
    C.append(Case("rot0_cells", rot0 + [tie0], [
        ("rotation 0 in cells of 1, 2, 3, 4, 5, 32, 33, 512", lambda m: [b.rot0_cell for b in m.blocks[:8]] == [1, *sizes]),
        ("rotation 0 in a 5-byte tie group", lambda m: m.blocks[8].t5.rot0_group == 2),
        ("MSD finish", lambda m: _finish(m, "msd"))]))
    # -- tie groups of RD_MAXGROUP and RD_MAXGROUP + 1 with short common prefixes, on both resolvers --
    big = bucket_block(MB_CAP + 60, 900)  # the MSD path gives up on the bucket: the LSD direct finish by default
    for g in (16, 17):
        C.append(Case("group5_%d" % g, [repeat_block(6, g, 910 + g)], [
            ("5-byte group of %d" % g, lambda m, g=g: m.blocks[0].t5.max_group == g and m.blocks[0].t5.depth < 69),
            ("MSD finish" if g == 16 else "MSD gave up on the group",
             (lambda m: _finish(m, "msd")) if g == 16 else (lambda m: m.predict().bwt_msd_fallback_why == WHY_GROUP))]))
        C.append(Case("group4_%d" % g, [repeat_block(5, g, 920 + g, base=big)], [
            ("4-byte group of %d" % g, lambda m, g=g: m.blocks[0].t4.max_group == g and m.blocks[0].t4.depth < 68),
            ("LSD direct finish" if g == 16 else "LSD direct gave up on the group",
             (lambda m: _finish(m, "direct")) if g == 16 else (lambda m: m.predict().bwt_direct_fallback_why == WHY_GROUP))]))
    # -- the resolvers' depth limit: equal on 5 + 64 bytes (MSD) and 4 + 64 bytes (LSD) --
    for d in (68, 69):
        C.append(Case("depth5_%d" % d, [repeat_block(d, 2, 930 + d)], [
            ("MSD tie depth %d" % d, lambda m, d=d: m.blocks[0].t5.depth == d),
            ("MSD finish" if d == 68 else "MSD gave up on the depth",
             (lambda m: _finish(m, "msd")) if d == 68 else (lambda m: m.predict().bwt_msd_fallback_why == WHY_DEPTH))]))
    for d in (67, 68):
        C.append(Case("depth4_%d" % d, [repeat_block(d, 2, 940 + d, base=big)], [
            ("LSD tie depth %d" % d, lambda m, d=d: m.blocks[0].t4.depth == d),
            ("LSD direct finish" if d == 67 else "LSD direct gave up on the depth",
             (lambda m: _finish(m, "direct")) if d == 67 else (lambda m: m.predict().bwt_direct_fallback_why == WHY_DEPTH))]))
    # -- the tie list at n / 8 and n / 8 + 1 --
    for over in (0, 1):
        C.append(Case("tielist_%s" % ("at" if over == 0 else "over"), [tie_list_block(over, 950 + over)], [
            ("5-byte tie list of n/8%s" % ("" if over == 0 else " + 1"), lambda m, o=over: m.blocks[0].t5.members == 100000 // 8 + o),
            ("MSD finish" if over == 0 else "MSD gave up on the tie list",
             (lambda m: _finish(m, "msd")) if over == 0 else (lambda m: m.predict().bwt_msd_fallback_why == WHY_TIES))]))
    # -- alphabets on the MSD path: 2, 3, 4, 255, 256 symbols (0x00 and 0xff in use) in a low-score batch; one symbol --
    filler = [T.ascii_random(3000, 1000 + k) for k in range(180)]
    alpha = [alphabet_block(2, 64, 1), alphabet_block(3, 200, 2), alphabet_block(4, 600, 3),
             alphabet_block(255, 200000, 4), alphabet_block(256, 200000, 5)]
    C.append(Case("alphabets", alpha + filler, [
        ("alphabets 2, 3, 4, 255, 256", lambda m: [b.alphabet for b in m.blocks[:5]] == [2, 3, 4, 255, 256]),
        ("MSD finish", lambda m: _finish(m, "msd"))], compress=True))
    C.append(Case("one_symbol", [b"\xff" * 40] + filler[:120], [
        ("one symbol", lambda m: m.blocks[0].alphabet == 1),
        ("the MSD path runs, gives up on the group", lambda m: m.predict().msd_launches == 1 and m.predict().bwt_msd_fallback_why == WHY_GROUP)]))
    # -- periodic blocks whose period divides n, and the same with one byte changed --
    for p, n in ((1, 900000), (2, 900000), (3, 900000), (67, 67 * 3000), (68, 68 * 3000), (69, 69 * 3000),
                 (4096, 4096 * 219), (300000, 900000)):
        C.append(Case("periodic_%d" % p, [periodic(p, n, p), periodic(p, n, p, near=True)],
                      [("period %d divides %d" % (p, n), lambda m, p=p, n=n: n % p == 0 and m.blocks[0].n == n)]))
    # -- block lengths 0..5, 900000 and every tile edge +-1 --
    lens = [0, 1, 2, 3, 4, 5, 900000] + [e + d for e in (2048, 4096, 16384) for d in (-1, 0, 1)]
    C.append(Case("lengths", [T.ascii_random(k, 1100 + k) for k in lens], [("MSD finish", lambda m: _finish(m, "msd"))]))
    for blk in (b"ab", b"abc", b"abcd", b"abcde"):
        C.append(Case("single_%d" % len(blk), [blk], [("MSD finish", lambda m: _finish(m, "msd"))]))
    # -- every batch in the wrong mode for its data, at 1 and 3 blocks per batch --
    kinds = {"A": lambda s: T.ascii_random(200000, s), "T": lambda s: T.texty(200000, s), "R": lambda s: T.runs(200000, s),
             "U": lambda s: b"z" * 200000}
    order = "ATAUATRUA"
    C.append(Case("handover_1", [kinds[k](1200 + i) for i, k in enumerate(order)],
                  [("batches 1.. in the wrong mode at 1 block per batch", lambda m: _wrong_modes(m, 1))], compress=True))
    C.append(Case("handover_3", [kinds[k](1300 + i) for i, k in enumerate(order) for _ in range(3)],
                  [("batches 1.. in the wrong mode at 3 blocks per batch", lambda m: _wrong_modes(m, 3))]))
    return tuple(C)


# the configurations of tests/test_gpu_bwt_paths.py: environment, and the model's (batch, msd, prefix8)
CONFIGS = {
    "default": ({}, dict()),
    "msd_first": ({"B2_BWT_PREFIX8": "0"}, dict(prefix8=False)),
    "lsd": ({"B2_BWT_MSD": "0", "B2_BWT_PREFIX8": "0"}, dict(msd=False, prefix8=False)),
    "wide": ({"B2_BWT_PREFIX8": "1"}, dict(prefix8=True)),
    "batch1": ({"B2_BWT_BATCH": "1"}, dict(batch=1)),
    "batch3": ({"B2_BWT_BATCH": "3"}, dict(batch=3)),
}
