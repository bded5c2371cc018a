"""RLE1 block-cut case corpus and a numpy model of the encoder's RLE1 stage (csrc/rle1.cu).

The stage restates readBlock (lib/Bzip2.js:636-667), a byte-serial state machine whose run state resets at every block
boundary, as parallel pieces: per-4-KiB-tile summaries (a fast path for aligned tiles without four equal bytes, looking
three bytes back), a scan of the tile summaries (one CTA up to 8192 tiles, a multi-CTA group scan of 2048 tiles per
group above that or with $B2_RLE_SCAN_GROUPS), the block walk (a speculative parallel walk from W = k * blockSize when a
file has 16 blocks or more, one CTA otherwise or when the segments do not chain up), the emit and the CRC pieces.  A
round trip cannot see a block cut in the wrong place, so the cases below are built to sit on the seams of those pieces,
and `Model` restates each piece in numpy so that a test can say what every case reaches:

- w(i), W(x): RLE1 bytes of raw byte i / of raw[0, x) under maximal-run phases (phases restart every 255 bytes);
- the tile summaries and plain (fast-path) flags for a given buffer alignment, and the scan state of every tile and
  group (mirrors rs_make / rs_combine, compressjs_b200/sharded.py);
- the sequential cut (what k_rle_blocks computes with one CTA), which must equal the oracle's rle1_split;
- whether the speculative walk with P = min(64, blocks / 8) segments chains up, and so the path counters of b2_stats
  (rle_group_scans, rle_walk_parallel, rle_walk_serial) for a plan.
"""
import functools
from dataclasses import dataclass, field

import numpy as np

from compressjs_b200.sharded import rs_combine
from tests import util as T

TILE = 4096
RG_TILES = 2048                    # tiles per group of the multi-CTA scan
GROUP = TILE * RG_TILES            # 8 MiB
ONE_CTA_TILES = 4 * RG_TILES       # the single-CTA scan handles up to 8192 tiles (32 MiB)
_W_OF_PHASE = np.zeros(255, dtype=np.uint8)
_W_OF_PHASE[:3] = 1
_W_OF_PHASE[3] = 2


def block_size(level):
    return level * 100000 - 19


def outfresh(c):
    q, r = divmod(int(c), 255)
    return 5 * q + (r if r <= 3 else 5)


def cneed(target):
    """Smallest c with outfresh(c) >= target (target >= 1)."""
    q = (target - 1) // 5
    rem = target - 5 * q
    return 255 * q + (rem if rem <= 3 else 4)


def rs_make(allsame, fc, lc, trail, ln):
    return (1 << 63) | (int(allsame) << 62) | (int(fc) << 24) | (int(lc) << 16) | ((int(trail) % 255) << 8) | (int(ln) % 255)


@dataclass
class Block:
    s: int        # first raw byte
    e: int        # one past the last raw byte
    b: int        # end of the re-phased run the block starts in (== s when it starts on a run start)
    n: int        # RLE1 bytes
    kind: str     # "fill_first_run" (the ofs >= BS branch), "last" (input ends first) or "full"
    end_phase: int  # run phase (1..255, block-local) of the last raw byte
    end: str      # "lit" (phase 1-3), "count0" (4th byte + count byte), "nocount" (4th byte, no room for the count)


class View:
    """Maximal-phase RLE1 arithmetic over a buffer (a whole file, or a share + halo of one): W is absolute (the RLE1
    output of the whole input before each position), run ends are capped at the end of the buffer."""

    def __init__(self, a, W, rstarts):
        self.a, self.W, self.rstarts, self.n = a, W, rstarts, a.size

    def run_end(self, s):
        k = int(np.searchsorted(self.rstarts, s, side="right"))
        return int(self.rstarts[k]) if k < self.rstarts.size else self.n

    def run_start(self, x):
        return int(self.rstarts[int(np.searchsorted(self.rstarts, x, side="right")) - 1])

    def first_reaching(self, v):
        """Smallest x >= 1 with W[x] >= v."""
        return int(np.searchsorted(self.W[1:], v, side="left")) + 1

    def block(self, s, BS):
        """k_rle_blocks for the block that starts at s (one iteration of its walk)."""
        a, W, N = self.a, self.W, self.n
        midrun = s > 0 and a[s - 1] == a[s]
        b = min(self.run_end(s), N, s + cneed(BS)) if midrun else s
        ofs = outfresh(b - s)
        if ofs >= BS:
            e = s + cneed(BS)
            return self._fin(Block(s, e, e, BS, "fill_first_run", 0, ""), BS, ofs=None)
        Wb = int(W[b])
        V = Wb + (BS - ofs)
        if V > int(W[N]):
            return self._fin(Block(s, N, b, ofs + int(W[N]) - Wb, "last", 0, ""), BS, ofs)
        e = self.first_reaching(V)
        return self._fin(Block(s, e, b, min(ofs + int(W[e]) - Wb, BS), "full", 0, ""), BS, ofs)

    def _fin(self, blk, BS, ofs):
        x = blk.e - 1
        d = (x - blk.s) if x < blk.b else (x - self.run_start(x))
        blk.end_phase = d % 255 + 1
        if blk.end_phase != 4:
            blk.end = "lit"
        elif blk.kind == "fill_first_run":
            blk.end = "nocount" if outfresh(blk.e - blk.s) > BS else "count0"
        else:
            produced = ofs + int(self.W[blk.e]) - int(self.W[blk.b])
            blk.end = "nocount" if produced > blk.n else "count0"
        return blk

    def walk(self, s, BS, maxblocks):
        out = []
        while s < self.n and len(out) < maxblocks:
            blk = self.block(s, BS)
            out.append(blk)
            s = blk.e
        return out

    def spec_start(self, u):
        """Raw position where a speculative segment starts: behind the byte that completes u RLE1 bytes."""
        return 0 if u == 0 else self.first_reaching(u)


class Model:
    def __init__(self, data):
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        n = a.size
        self.a, self.n = a, n
        start = np.ones(n, dtype=bool)
        start[1:] = a[1:] != a[:-1]
        self.rstarts = np.flatnonzero(start)
        idx = np.arange(n, dtype=np.int64)
        rs = np.where(start, idx, 0)
        np.maximum.accumulate(rs, out=rs)
        idx -= rs
        del rs
        w = _W_OF_PHASE[idx % 255]
        del idx
        self.W = np.zeros(n + 1, dtype=np.int32 if n < (1 << 30) else np.int64)   # W(x) <= 5/4 x
        np.cumsum(w, out=self.W[1:])
        self.view = View(a, self.W, self.rstarts)

    # ---- A: tile summaries ------------------------------------------------------------------------------------------
    @functools.lru_cache(maxsize=4)
    def tiles(self, mis=0):
        """Per tile: (plain, fc, lc, lead, trail, allsame, rest, length) as k_rle_summary writes them for a buffer
        whose address is `mis` mod 16."""
        a, n = self.a, self.n
        eq = np.zeros(n, dtype=bool)        # eq[i]: a[i] == a[i-1] == a[i-2] == a[i-3]
        if n >= 4:
            eq[3:] = (a[3:] == a[2:-1]) & (a[3:] == a[1:-2]) & (a[3:] == a[:-3])
        if n:
            # the first tile looks back into bytes that do not exist: k_rle_summary makes them up from ~a[0] + k
            x0, pw = int(a[0]), 0
            for k in (1, 2, 3):
                pw |= (((~x0) & 255) + k) << (8 * (4 - k))
            pw &= 0xffffffff
            ext = np.array([(pw >> 8) & 255, (pw >> 16) & 255, (pw >> 24) & 255] + list(a[:3]), dtype=np.uint8)
            for i in range(min(3, n)):
                eq[i] = bool(ext[i + 3] == ext[i + 2] == ext[i + 1] == ext[i])
        out = []
        for t in range(0, (n + TILE - 1) // TILE):
            t0 = t * TILE
            ln = min(TILE, n - t0)
            fc, lc = int(a[t0]), int(a[t0 + ln - 1])
            plain = ln == TILE and (mis + t0) % 16 == 0 and not eq[t0:t0 + ln].any()
            if plain:
                lead = 1
                while lead < 4 and a[t0 + lead] == fc:
                    lead += 1
                trail = 1
                while trail < 4 and a[t0 + ln - 1 - trail] == lc:
                    trail += 1
                out.append((True, fc, lc, lead, trail, False, ln - lead, ln))
                continue
            k = int(np.searchsorted(self.rstarts, t0, side="right"))
            first = int(self.rstarts[k]) - t0 if k < self.rstarts.size else ln
            lead = min(first, ln)
            k2 = int(np.searchsorted(self.rstarts, t0 + ln, side="left")) - 1
            last = max(int(self.rstarts[k2]) - t0, 0) if k2 >= 0 else 0
            rest = int(self.W[t0 + ln] - self.W[t0 + lead])
            out.append((False, fc, lc, lead, ln - last, lead == ln, rest, ln))
        return out

    def tile_state(self, t, mis=0):
        plain, fc, lc, lead, trail, allsame, rest, ln = self.tiles(mis)[t]
        return rs_make(allsame, fc, lc, trail, ln)

    # ---- B: the scan ------------------------------------------------------------------------------------------------
    def scan(self, mis=0):
        """Carry (run length mod 255 entering the tile) and W(tile start) per tile, by combining the tile states as the
        scan kernels do, plus the aggregate state of every 2048-tile group."""
        st, carry, pref, groups = 0, [], [], []
        Wacc, gagg = 0, 0
        for t, (plain, fc, lc, lead, trail, allsame, rest, ln) in enumerate(self.tiles(mis)):
            if t % RG_TILES == 0:
                if t:
                    groups.append(gagg)
                gagg = 0
            c = ((st >> 8) & 255) if (st >> 63) and ((st >> 16) & 255) == fc else 0
            carry.append(c)
            pref.append(Wacc)
            Wacc += outfresh(c + lead) - outfresh(c) + rest
            ts = rs_make(allsame, fc, lc, trail, ln)
            st = rs_combine(st, ts)
            gagg = rs_combine(gagg, ts)
        if self.n:
            groups.append(gagg)
        return carry, pref + [Wacc], groups, st

    def carry_from_data(self):
        """The same carries, straight from the bytes: length (mod 255) of the run that enters each tile."""
        out = []
        for t0 in range(0, self.n, TILE):
            if t0 and self.a[t0 - 1] == self.a[t0]:
                out.append((t0 - self.view.run_start(t0 - 1)) % 255)
            else:
                out.append(0)
        return out

    def crossing_carries(self, edges):
        """Run lengths (mod 255) carried across the given edges by runs that go on behind them."""
        return {(e - self.view.run_start(e - 1)) % 255 for e in edges if 0 < e < self.n and self.a[e - 1] == self.a[e]}

    def ntiles(self):
        return (self.n + TILE - 1) // TILE

    def ngroups(self):
        return (self.ntiles() + RG_TILES - 1) // RG_TILES

    # ---- C: the block walk ------------------------------------------------------------------------------------------
    @functools.lru_cache(maxsize=16)
    def cut(self, level):
        return self.view.walk(0, block_size(level), self.maxblocks(level))

    def maxblocks(self, level):
        BS = block_size(level)
        return self.n // (BS * 4 // 5) + 2

    def total_guess(self, level):
        BS = block_size(level)
        return (int(self.W[self.n]) + BS - 1) // BS

    @functools.lru_cache(maxsize=16)
    def parallel_walk(self, level):
        """None when the exact plan does not try the speculative walk; else (accepted, segment starts)."""
        BS = block_size(level)
        total, maxb = self.total_guess(level), self.maxblocks(level)
        P = min(64, total // 8)
        if not (P > 1 and total < maxb):
            return None
        blocks, cuts, starts = [], [], []
        for r in range(P):
            first, nxt = r * total // P, (r + 1) * total // P
            s = self.view.spec_start(first * BS)
            starts.append(s)
            seg = self.view.walk(s, BS, (maxb - first) if r == P - 1 else nxt - first)
            cuts.append(len(seg))
            blocks += seg
        ok = all(cuts[r] == (r + 1) * total // P - r * total // P for r in range(P - 1)) and cuts[P - 1] > 0
        if ok:
            blocks = blocks[:(P - 1) * total // P + cuts[P - 1]]
            ok = blocks[0].s == 0 and blocks[-1].e == self.n and all(x.e == y.s for x, y in zip(blocks, blocks[1:]))
        return ok, starts

    def libbz2(self, level):
        """libbz2 rejects a block that ends on a 4th byte without its count byte; every other cut is in its language."""
        return not any(b.end == "nocount" for b in self.cut(level))

    def counters(self, level, force_groups=False):
        """(rle_group_scans, rle_walk_parallel, rle_walk_serial) of one exact plan of the whole buffer."""
        if self.n == 0:
            return (0, 0, 0)
        g = int(self.ntiles() > ONE_CTA_TILES or force_groups)
        pw = self.parallel_walk(level)
        if pw is not None and pw[0]:
            return (g, 1, 0)
        return (g, 0, 1)

    # ---- sharded input ----------------------------------------------------------------------------------------------
    def share_summary(self, g0, g1):
        """b2_bzip2_share_summary of data[g0:g1]: (state, lead, RLE1 bytes when no run enters, length)."""
        n = g1 - g0
        if n == 0:
            return (0, 0, 0, 0)
        a = self.a
        lead = min(self.view.run_end(g0), g1) - g0
        trail = g1 - max(self.view.run_start(g1 - 1), g0)
        w = outfresh(lead) + int(self.W[g1] - self.W[g0 + lead])
        return (rs_make(lead == n, a[g0], a[g1 - 1], trail, n), lead, w, n)

    def range_plan(self, level, g0, hold, first, count, force_groups=False):
        """b2_bzip2_plan_share on data[g0:g0+hold] for blocks [first, first+count): (counters, blocks cut)."""
        BS = block_size(level)
        k0 = int(np.searchsorted(self.rstarts, g0, side="right"))
        k1 = int(np.searchsorted(self.rstarts, g0 + hold, side="left"))
        rst = np.concatenate([[0], self.rstarts[k0:k1] - g0]).astype(np.int64)
        v = View(self.a[g0:g0 + hold], self.W[g0:g0 + hold + 1], rst)
        ntiles = (hold + TILE - 1) // TILE
        g = int(ntiles > ONE_CTA_TILES or force_groups) if hold else 0
        maxb = min(hold // (BS * 4 // 5) + 2, count)
        if maxb == 0 or hold == 0:
            return (g, 0, 0), []
        P = min(64, maxb // 8)
        if P > 1:
            blocks, cuts = [], []
            for r in range(P):
                f, nx = first + r * maxb // P, first + (r + 1) * maxb // P
                u = f * BS
                if u > int(v.W[hold]):
                    cuts.append(0)
                    continue
                seg = v.walk(v.spec_start(u) if u else 0, BS, nx - f)
                cuts.append(len(seg))
                blocks += seg
            ok = all(cuts[r] == (r + 1) * maxb // P - r * maxb // P for r in range(P - 1)) and cuts[P - 1] > 0
            if ok:
                blocks = blocks[:(P - 1) * maxb // P + cuts[P - 1]]
                ok = all(x.e == y.s for x, y in zip(blocks, blocks[1:]))
            if ok:
                return (g, 1, 0), blocks
        u = first * BS
        if u > int(v.W[hold]):
            return (g, 0, 1), []
        return (g, 0, 1), v.walk(v.spec_start(u) if u else 0, BS, maxb)


# ---- corpus builders ---------------------------------------------------------------------------------------------------
class Builder:
    """Appends literals and runs while tracking the RLE1 bytes of the block being filled (readBlock semantics), so that
    a case can say on which run phase a block fills."""

    def __init__(self, level, seed):
        self.BS = block_size(level)
        self.g = T.rng(seed)
        self.buf = bytearray()
        self.cur = 0      # RLE1 bytes of the current block
        self.blocks = 1

    def _lit_bytes(self, k):
        # printable bytes (33..125), no two neighbours equal, the first one unlike the byte before
        prev = self.buf[-1] - 33 if self.buf and 33 <= self.buf[-1] <= 125 else int(self.g.integers(0, 93))
        v = 33 + (prev + np.cumsum(self.g.integers(1, 93, size=k, dtype=np.int64))) % 93
        return bytearray(v.astype(np.uint8).tobytes())

    def lit(self, k):
        while k > 0:
            room = self.BS - self.cur
            take = min(k, room)
            self.buf += self._lit_bytes(take)
            self.cur += take
            k -= take
            if self.cur == self.BS:
                self.cur = 0
                self.blocks += 1
        return self

    def fill_to(self, left):
        """Literals until `left` RLE1 bytes of the current block remain."""
        return self.lit((self.BS - self.cur - left) % self.BS)

    def run(self, ln, ch=None):
        if ch is None:
            ch = 0x5a if not self.buf or self.buf[-1] != 0x5a else 0x5b
        self.buf += bytes([ch]) * ln
        rest = ln
        while rest:
            room = self.BS - self.cur
            if outfresh(rest) < room:
                self.cur += outfresh(rest)
                break
            c = cneed(room)
            rest -= c
            self.cur = 0
            self.blocks += 1
        return self

    def bytes(self):
        return bytes(self.buf)


def _ascii_no_runs(n, seed):
    """Random printable bytes, no two neighbours equal (every tile takes the fast path when aligned)."""
    return Builder(9, seed)._lit_bytes(n)


def _plant(buf, pos, ln, ch):
    """Run of `ln` bytes `ch` at pos; the bytes around it are made to differ."""
    buf[pos:pos + ln] = bytes([ch]) * ln
    for q in (pos - 1, pos + ln):
        if 0 <= q < len(buf) and buf[q] == ch:
            buf[q] = ch ^ 0x40


RUN_LENGTHS = list(range(1, 7)) + list(range(254, 262)) + list(range(509, 517)) + list(range(764, 772))


def _edge_runs(seed):
    """One tile per (run length, offset, start/end): a run that starts or ends at tile edge + offset (-4..+4), and in
    the middle of the same tile one that starts or ends at a 16-byte thread-chunk edge + offset."""
    g = T.rng(seed)
    plans = [(ln, o, se) for ln in RUN_LENGTHS for o in range(-4, 5) for se in (0, 1)]
    buf = bytearray(_ascii_no_runs(TILE * (len(plans) + 2), seed))
    for k, (ln, o, se) in enumerate(plans):
        t0 = TILE * (k + 1)
        ch = int(g.integers(0, 256))
        _plant(buf, t0 + o if se == 0 else t0 + o - ln, ln, ch)
        c0 = t0 + 2048 + 16 * int(g.integers(-2, 3))
        _plant(buf, c0 + o if se == 0 else c0 + o - ln, ln, ch ^ 0x81)
    return bytes(buf)


def _lookback(seed):
    """Runs of four (and of three) across the start of an aligned tile, split 1+3, 2+2 and 3+1, in otherwise run-free
    tiles: only the fast path's three-byte look-back sees the first three bytes."""
    buf = bytearray(_ascii_no_runs(TILE * 16, seed))
    k = 1
    for ln in (4, 3):
        for before in (1, 2, 3):
            t0 = TILE * k
            _plant(buf, t0 - before, ln, 0x41 + k)
            k += 2
    return bytes(buf)


def _long_runs_at_edges(nbytes, seed, edges, mods, cover=None, cross=None):
    """Disk-image-like bytes (zero runs up to 64 KiB with printable islands) with runs of many tiles planted across
    each edge: the run across edges[i] has 255 k + mods[i] bytes in front of the edge and 1-3000 behind it, so the scan
    carries a run of mods[i] (mod 255) into the tile or group that starts there.  cover: (start, end) of one run;
    cross: (start, end) of another."""
    g = T.rng(seed)
    buf = bytearray(nbytes)
    pos = 0
    while pos < nbytes:
        z = int(g.integers(1, 1 << 16))
        pos += z
        isl = int(g.integers(64, 2048))
        if pos < nbytes:
            buf[pos:pos + isl] = _ascii_no_runs(isl, int(g.integers(1 << 30)))[:max(0, nbytes - pos)]
        pos += isl
    del buf[nbytes:]
    for i, (edge, m) in enumerate(zip(edges, mods)):
        ln = 255 * int(g.integers(20, 60)) + m
        _plant(buf, edge - ln, ln + int(g.integers(1, 3000)), 0x10 + i)
    if cover:
        _plant(buf, cover[0], cover[1] - cover[0], 0xee)
    if cross:
        _plant(buf, cross[0], cross[1] - cross[0], 0xdd)
    return bytes(buf)


def _disk_image(nbytes, seed):
    """Zero runs of random length up to 2^20 with printable and text islands, and a run planted across every group edge
    with 255 k + (0, 1, 3, 4, ...) bytes in front of it."""
    g = T.rng(seed)
    buf = bytearray(nbytes)
    pos = 0
    while pos < nbytes:
        pos += int(g.integers(1, 1 << 20))
        if g.random() < 0.5:
            isl = _ascii_no_runs(int(g.integers(256, 16384)), int(g.integers(1 << 30)))
        else:
            isl = T.texty(int(g.integers(256, 16384)), int(g.integers(1 << 30)))
        isl = isl[:max(0, nbytes - pos)]
        buf[pos:pos + len(isl)] = isl
        pos += len(isl)
    for i, e in enumerate(range(GROUP, nbytes, GROUP)):
        a = 255 * int(g.integers(1, 1100)) + (0, 1, 3, 4)[i % 4]
        _plant(buf, e - a, a + int(g.integers(1, 300000)), 0x80 + i)
    return bytes(buf)


def _phases(level, seed, last):
    """Blocks that fill on run phases 1, 2, 3, on a 4th byte with no room for its count byte, on a count byte (0), and
    on the first byte after a full 255-run (count 251); each fill leaves the rest of the run to the next block, which
    starts in the middle of it.  The file ends with a last block of `last` bytes."""
    b = Builder(level, seed)
    for left, ln in ((1, 700), (2, 700), (3, 700), (4, 700), (5, 700), (6, 900)):
        b.fill_to(left).run(ln).lit(37)
    b.fill_to(0).lit(last)
    return b.bytes()


def _slip(level, seed, nblocks, slip_blocks):
    """nblocks blocks of literals; blocks in slip_blocks fill inside a run (re-phasing it, so every later block
    boundary moves away from W = k * blockSize)."""
    b = Builder(level, seed)
    todo = set(slip_blocks)
    while b.blocks <= nblocks:
        if b.blocks in todo:
            todo.discard(b.blocks)
            b.fill_to(2).run(1000)
        b.lit(int(b.g.integers(20000, 40000)))
    return b.bytes()


@dataclass
class Case:
    name: str
    make: object
    levels: tuple
    claims: list = field(default_factory=list)   # (what, predicate(model, level)) -- checked at every level
    groups_hook: bool = False   # run with B2_RLE_SCAN_GROUPS too (8-40 MiB cases)
    skew: bool = False          # run b2_bzip2_compress_dev at pointer skews 0, 1, 255
    chunk: tuple = ()           # B2_H2D_CHUNK values for a pinned upload
    window: tuple = ()          # B2_STREAM_WINDOW values ("block:k" = the raw start of block k at the first level)
    shares: tuple = ()          # (world, halo) of simulated ranks, share edges moved into planted runs

    @functools.cached_property
    def data(self):
        return self.make()


def _ends(m, level):
    return {(b.end_phase, b.end) for b in m.cut(level)}


def _reaches(kind):
    return lambda m, lv: any(b.kind == kind for b in m.cut(lv))


def _walk(accepted):
    return lambda m, lv: m.parallel_walk(lv) is not None and m.parallel_walk(lv)[0] == accepted


def group_edges(m):
    return list(range(GROUP, m.n, GROUP))


def tile_edges(m):
    return [e for e in range(TILE, m.n, TILE) if e % GROUP]


def _shares_chain(m, lv):
    c = next(c for c in cases() if model(c.name) is m)
    return all(share_plan(c, lv, world, halo)[1] for world, halo in c.shares)


@functools.lru_cache(maxsize=1)
def cases():
    cs = []
    cs.append(Case("edge_runs", lambda: _edge_runs(11), (1, 9),
                   [("plain tiles next to run tiles", lambda m, lv: 0 < sum(t[0] for t in m.tiles()) < m.ntiles()),
                    ("runs entering tiles with carries 1..4 and 254", lambda m, lv: {1, 2, 3, 4, 254} <= set(m.scan()[0]))],
                   skew=True, window=("block:12",)))
    for ln in RUN_LENGTHS:
        for where in ("start", "end"):
            tail = _ascii_no_runs(3000 + ln, ln)
            run = bytes([tail[-1] ^ 0x40 if where == "end" else tail[0] ^ 0x40]) * ln
            data = (run + bytes(tail)) if where == "start" else (bytes(tail) + run)
            cs.append(Case("run%d_at_%s" % (ln, where), (lambda d=data: d), (1,),
                           [("one block", lambda m, lv: len(m.cut(lv)) == 1)]))
    cs.append(Case("lookback", lambda: _lookback(5), (1,),
                   [("runs of four across a tile edge turn the fast path off",
                     lambda m, lv: [t[0] for t in m.tiles()][1:12:2] == [False] * 3 + [True] * 3)], skew=True))
    for level in (1, 5, 9):
        for last in ((1, 2, 3, 4) if level == 1 else (2 if level == 5 else 4,)):
            cs.append(Case("phases_l%d_last%d" % (level, last), (lambda lv=level, la=last: _phases(lv, 21 + lv, la)), (level,),
                           [("blocks fill on phases 1-4, count bytes 0 and after 251",
                             lambda m, lv: {(1, "lit"), (2, "lit"), (3, "lit"), (4, "nocount"), (4, "count0")} <= _ends(m, lv)),
                            ("a block fills on the byte after a full 255-run",
                             lambda m, lv: any(b.end_phase == 1 and b.e - 1 >= b.b and b.e - 1 - m.view.run_start(b.e - 1) >= 255
                                               for b in m.cut(lv))),
                            ("last block of %d bytes" % last, lambda m, lv, la=last: m.cut(lv)[-1].n == la)],
                           chunk=(1 << 16, (1 << 16) + 1) if level == 1 and last == 1 else (),
                           window=("block:2",) if level == 9 else (), skew=level == 5))
    cs.append(Case("run12M", lambda: b"q" * 12000000 + _ascii_no_runs(300000, 7), (1, 9),
                   [("the ofs >= BS branch", lambda m, lv: lv != 1 or _reaches("fill_first_run")(m, lv))],
                   chunk=(1 << 20, (1 << 20) + 1), window=(6 << 20,), shares=((2, 2 << 20), (3, 2 << 20))))
    cs.append(Case("spec_holds", lambda: T.texty(30 * 99981, 17), (1,), [("speculative walk accepted", _walk(True))],
                   shares=((2, 1 << 20), (3, 1 << 20))))
    for where, slips in (("first", [2]), ("middle", [13]), ("last", [27])):
        cs.append(Case("slip_%s" % where, (lambda sl=slips: _slip(1, 31, 30, sl)), (1,),
                       [("speculative walk %s" % ("accepted" if where == "last" else "rejected"), _walk(where == "last"))],
                       shares=((3, 1 << 20),)))
    # halo: the whole rest of the input, so that every block that starts in a share can be finished and the ranks chain
    whole = 64 << 20
    cs.append(Case("group_edges_24M",
                   lambda: _long_runs_at_edges(24 << 20, 41, [GROUP, 2 * GROUP, GROUP + 77 * TILE, GROUP + 300 * TILE,
                                                              GROUP + 500 * TILE, GROUP + 900 * TILE, 2 * GROUP + 5 * TILE],
                                               [0, 1, 3, 0, 1, 4, 5]), (1, 9),
                   [("runs cross both group edges with carries 0 and 1", lambda m, lv: {0, 1} <= m.crossing_carries(group_edges(m))),
                    ("runs cross tile edges with carries 0, 1, 3, 4 and 5", lambda m, lv: {0, 1, 3, 4, 5} <= m.crossing_carries(tile_edges(m))),
                    ("simulated ranks chain up at level 9 (a phase slip moves the level-1 boundaries)",
                     lambda m, lv: lv != 9 or _shares_chain(m, lv))],
                   groups_hook=True, chunk=(1 << 20,), shares=((2, whole), (3, whole))))
    cs.append(Case("group_cover_28M",
                   lambda: _long_runs_at_edges(28 << 20, 43, [GROUP, GROUP - 20 * TILE, GROUP + 11 * TILE], [3, 4, 0],
                                               cover=(2 * GROUP - (255 * 30 + 4), 3 * GROUP + 1000)), (1, 9),
                   [("a group that is one run", lambda m, lv: any((s >> 62) & 1 for s in m.scan()[2])),
                    ("runs cross group edges with carries 3 and 4", lambda m, lv: {3, 4} <= m.crossing_carries(group_edges(m)))],
                   groups_hook=True))
    cs.append(Case("group_cross_20M",
                   lambda: _long_runs_at_edges(20 << 20, 45, [2 * GROUP + 9 * TILE], [1],
                                               cross=(GROUP - (255 * 40 + 5), 2 * GROUP + 5000)), (1,),
                   [("a run across two group edges", lambda m, lv: m.view.run_start(2 * GROUP) < GROUP < 2 * GROUP < m.view.run_end(2 * GROUP)),
                    ("it crosses the first with carry 5", lambda m, lv: 5 in m.crossing_carries([GROUP]))],
                   groups_hook=True))
    cs.append(Case("disk_image_40M", lambda: _disk_image(40 << 20, 47), (1, 9),
                   [("group scan without the hook", lambda m, lv: m.counters(lv)[0] == 1 and m.ngroups() >= 3),
                    ("runs cross group edges with carries 0, 1, 3 and 4", lambda m, lv: {0, 1, 3, 4} <= m.crossing_carries(group_edges(m))),
                    ("simulated ranks chain up at level 9 (a phase slip moves the level-1 boundaries)",
                     lambda m, lv: lv != 9 or _shares_chain(m, lv))],
                   groups_hook=True, shares=((2, whole), (3, whole))))
    return cs


def case(name):
    return next(c for c in cases() if c.name == name)


# Every model stays cached for the session: the block walks of the GPU test's checks come back to the same cases many
# times.  A model holds the input and W (4 bytes per input byte), under 1 GB for the whole corpus.
@functools.lru_cache(maxsize=None)
def model(name):
    return Model(case(name).data)


def window_bytes(c, spec):
    if isinstance(spec, int):
        return spec
    k = int(spec.split(":")[1])
    return model(c.name).cut(c.levels[0])[k].s


def window_counters(data, level, win, force_groups=False):
    """Counters of b2_bzip2_compress with a streaming window of `win` bytes (an unpinned input: one plan per window)."""
    n, pos, tot = len(data), 0, np.zeros(3, dtype=np.int64)
    while True:
        wlen = min(win, n - pos)
        last_window = pos + wlen == n
        m = Model(np.frombuffer(data, dtype=np.uint8)[pos:pos + wlen])
        tot += m.counters(level, force_groups)
        cut = m.cut(level)
        nfinal = len(cut) if last_window else len(cut) - 1
        if last_window or nfinal <= 0:
            break
        pos += cut[nfinal - 1].e
    return tuple(int(x) for x in tot)


def share_edges(c, world):
    """Share boundaries: equal shares, each edge moved into the longest run near it (within a quarter share)."""
    m = model(c.name)
    n = m.n
    edges = []
    for r in range(1, world):
        e = r * n // world
        if m.view.run_end(e) - m.view.run_start(e) < 600:
            reach = min(1 << 20, n // (4 * world))
            k0 = int(np.searchsorted(m.rstarts, e - reach))
            k1 = int(np.searchsorted(m.rstarts, e + reach))
            st = m.rstarts[k0:k1]
            en = np.append(m.rstarts[k0 + 1:k1 + 1], n)[:st.size]
            if st.size:
                j = int(np.argmax(en - st))
                if en[j] - st[j] >= 600:
                    e = int(st[j] + en[j]) // 2
        edges.append(e)
    return [0] + edges + [n]


def share_plan(c, level, world, halo, force_groups=False):
    """What the simulated ranks of one share job compute, by the model: per rank (g0, g1, hold, first, count, share
    summary, counters of the summary call, counters and blocks of the plan_share call), and whether their pieces
    chain up (sharded.spec_plan_ok), i.e. whether the assembled stream is used."""
    from compressjs_b200 import sharded as S
    m = model(c.name)
    edges = share_edges(c, world)
    summaries = [m.share_summary(edges[r], edges[r + 1]) for r in range(world)]
    plan, total, _ = S.share_plan_inputs(summaries, level)
    ranks, infos = [], []
    for r in range(world):
        g0, g1 = edges[r], edges[r + 1]
        hold = min(m.n, g1 + halo) - g0
        first, count = plan[r][2], plan[r][3]
        g = int((g1 - g0 + TILE - 1) // TILE > ONE_CTA_TILES or force_groups) if g1 > g0 else 0
        cnt, blocks = m.range_plan(level, g0, hold, first, count, force_groups)
        ranks.append(dict(g0=g0, g1=g1, hold=hold, first=first, count=count, summary=summaries[r], sum_counters=(g, 0, 0),
                          counters=cnt, blocks=blocks))
        infos.append((blocks[0].s + g0 if blocks else 0, blocks[-1].e + g0 if blocks else 0, first, count, len(blocks), total))
    return ranks, S.spec_plan_ok(infos, m.n)
