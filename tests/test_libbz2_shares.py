"""CPU tests of the libbz2 flavor's sharded block cut: a numpy model of the per-share cut table
(b2_bzip2_share_cut_table), built from the piece logic of tests/libbz2_model.cut, chained by
compressjs_b200.sharded.libbz2_share_chain, must give exactly libbz2_model.cut's blocks -- for every world size,
level, seam and drift, up to the largest drift a share can see.  A gloo test runs compress_shares(flavor="libbz2")
with the model standing in for the device calls."""
import bz2
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from compressjs_b200 import sharded as S
from tests import libbz2_model as M
from tests import util as T
from tests.test_libbz2_model import _libbz2_ok
from tests.test_sharded_host import _free_port, _py_share_summary


# ---- the model -------------------------------------------------------------------------------------------------
def pieces(data):
    """Every piece of `data` as libbz2_model.cut reads them (stretches of one byte value, at most 255 long, the
    255-chunks of the maximal runs): (raw starts, W starts, W total), W = RLE1 bytes in front (L < 4 -> L, else 5)."""
    a = np.frombuffer(data, dtype=np.uint8)
    n = len(a)
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), 0
    rs = np.flatnonzero(np.r_[True, a[1:] != a[:-1]])
    rl = np.diff(np.r_[rs, n])
    nch = (rl + 254) // 255
    first = np.repeat(np.cumsum(nch) - nch, nch)
    starts = np.repeat(rs, nch) + 255 * (np.arange(int(nch.sum())) - first)
    plen = np.diff(np.r_[starts, n])
    w = np.where(plen < 4, plen, 5)
    W = np.r_[0, np.cumsum(w)]
    return starts.astype(np.int64), W[:-1].astype(np.int64), int(W[-1])


def w_at(P, x):
    """W(x): RLE1 bytes in front of raw position x under the pieces P."""
    starts, Ws, _ = P
    i = int(np.searchsorted(starts, x, side="right")) - 1
    if i < 0:
        return 0
    c = x - int(starts[i])          # bytes of the piece in front of x: the first three emit 1, the fourth 2, the rest 0
    return int(Ws[i]) + (c if c <= 3 else 5)


def model_table(P, g0, hold, share_len, w_in, level, dmax):
    """Rows (k, blocks, exit drift, flags) of the share data[g0:g0+share_len] with the halo up to g0 + hold, as
    k_cut_table computes them from the piece starts of the buffer (bits) in W space."""
    starts, Ws, _ = P
    M_ = level * 100000 - 19
    sel = (starts >= g0) & (starts < g0 + hold)
    bits = np.sort(Ws[sel] - w_in)
    wbuf = w_at(P, g0 + hold) - w_in
    wshare = w_at(P, g0 + share_len) - w_in

    def next_piece(x):
        if x >= wbuf:
            return None
        i = int(np.searchsorted(bits, x))
        return int(bits[i]) if i < len(bits) and bits[i] <= x + 4 else None

    rows = []
    for d in range(dmax + 1):
        k = (w_in - d + M_ - 1) // M_ if w_in > d else 0
        s = k * M_ + d - w_in
        flags, cnt = 0, 0
        if s < wbuf and next_piece(s) != s:
            flags |= S.CUT_NOT_PIECE
        while s < wshare:
            cnt += 1
            nx = next_piece(s + M_)
            if cnt == 1 and nx == s + M_:
                flags |= S.CUT_STEP_EXACT
            if nx is None:
                flags |= S.CUT_BUF_END
                break
            s = nx
        ex = 0 if flags & S.CUT_BUF_END else w_in + s - (k + cnt) * M_
        rows.append((k, cnt, ex, flags))
    return rows


def model_walk(P, first, drift, count, level, limit_raw):
    """Raw starts of the blocks [first, first + count) from the entry W = first * M + drift (k_cut_chain)."""
    starts, Ws, wt = P
    M_ = level * 100000 - 19
    Ws = Ws[starts < limit_raw]
    out, s = [], first * M_ + drift
    for _ in range(count):
        i = int(np.searchsorted(Ws, s))
        assert i < len(Ws) and Ws[i] == s
        out.append(int(starts[i]))
        j = int(np.searchsorted(Ws, s + M_))
        s = int(Ws[j]) if j < len(Ws) and Ws[j] <= s + M_ + 4 else wt
    return out


def shares_from_bounds(data, bounds, halo):
    """Summaries, share plan inputs and buffers of contiguous shares [a, b) with halos of `halo` bytes."""
    n = len(data)
    summaries = [_py_share_summary(data[a:b]) for a, b in bounds]
    holds = [min(n, b + halo) - a for a, b in bounds]
    return summaries, holds


def chain_of(data, bounds, level, halo):
    """Model tables of every share, chained by sharded.libbz2_share_chain: (chain, P, W total)."""
    summaries, holds = shares_from_bounds(data, bounds, halo)
    ins, _, w_total = S.share_plan_inputs(summaries, level)
    P = pieces(data)
    tables, ends = [], []
    for r, (a, b) in enumerate(bounds):
        w_in = ins[r][1]
        assert w_in == w_at(P, a)
        tables.append(model_table(P, a, holds[r], b - a, w_in, level, S.share_drift_bound(w_in, level)) if b > a else None)
        ends.append(a + holds[r] == len(data))
    return S.libbz2_share_chain(ins, w_total, tables, level, ends), P, w_total


def check_chain(data, bounds, level, halo=10 ** 9, ref=None):
    ref = M.cut(data, level) if ref is None else ref
    ch, P, _ = chain_of(data, bounds, level, halo)
    assert ch is not None
    res, total = ch
    assert total == len(ref)
    got = []
    for r, (first, drift, count) in enumerate(res):
        a, b = bounds[r]
        blk = model_walk(P, first, drift, count, level, len(data))
        assert all(a <= s < b for s in blk), (r, blk, a, b)
        if count:
            assert first == len(got)
        got += blk
    assert got == [s for s, _, _ in ref]
    return res


def even_bounds(n, world):
    return [(r * n // world, (r + 1) * n // world) for r in range(world)]


def random_bounds(n, world, g):
    cuts = sorted(int(x) for x in g.integers(0, n + 1, size=world - 1))
    e = [0] + cuts + [n]
    return [(e[r], e[r + 1]) for r in range(world)]


def max_drift(n):
    """Alternating runs of exactly 4 bytes: every piece is 5 RLE1 bytes, and M = 1 (mod 5) at every level, so every cut
    drifts by exactly 4."""
    return (b"aaaabbbb" * (n // 8 + 1))[:n]


def runs_across(n, seed):
    """Long runs (up to 1200 bytes) between random bytes: runs straddle share seams and cross 255-chunks."""
    g = T.rng(seed)
    out = bytearray()
    while len(out) < n:
        out += bytes([int(g.integers(0, 4))]) * int(g.integers(1, 1200))
        out += g.integers(0, 256, size=int(g.integers(0, 50)), dtype=np.uint8).tobytes()
    return bytes(out[:n])


KINDS = {"ascii": T.ascii_random, "text": T.texty, "runs": runs_across, "maxdrift": lambda n, s: max_drift(n)}


# ---- model against the sequential cut ---------------------------------------------------------------------------------
def test_model_pieces_give_the_rle1_size_of_every_block():
    data = runs_across(700000, 3)
    P = pieces(data)
    for s, ln, blk in M.cut(data, 1):
        assert w_at(P, s + ln) - w_at(P, s) == len(blk)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_chain_level1_even_and_random_shares(kind, world):
    data = KINDS[kind](9 * 99981 + 4321, 50 + world)
    ref = M.cut(data, 1)
    check_chain(data, even_bounds(len(data), world), 1, ref=ref)
    g = T.rng(world * 7 + len(kind))
    for _ in range(2):
        check_chain(data, random_bounds(len(data), world, g), 1, ref=ref)


@pytest.mark.parametrize("kind", ["ascii", "maxdrift", "runs"])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_chain_level9(kind, world):
    data = KINDS[kind](4 * 899981 + 777, 60 + world)
    ref = M.cut(data, 9)
    check_chain(data, even_bounds(len(data), world), 9, ref=ref)
    check_chain(data, random_bounds(len(data), world, T.rng(world)), 9, ref=ref)


def test_max_drift_input_reaches_the_bound():
    """Every cut drifts by exactly 4: block k has drift 4 k, the bound the tables are sized for."""
    level = 1
    data = max_drift(30 * 99981)
    ref = M.cut(data, level)
    P = pieces(data)
    Mb = level * 100000 - 19
    assert [w_at(P, s) - k * Mb for k, (s, _, _) in enumerate(ref)] == [4 * k for k in range(len(ref))]
    res = check_chain(data, even_bounds(len(data), 8), level)
    for r, (first, drift, count) in enumerate(res):
        if count and r:
            a = even_bounds(len(data), 8)[r][0]
            assert drift == 4 * first and drift <= S.share_drift_bound(w_at(P, a), level)


@pytest.mark.parametrize("level", [1, 9])
@pytest.mark.parametrize("kind", ["ascii", "maxdrift", "text"])
def test_share_starting_0_to_4_bytes_after_a_block_start(kind, level):
    """The two-index edge: a share whose W start is within 4 of a block start, so that (k - 1) M + d and k M + d can
    both be consistent for the same drift d; each row names its block index."""
    n = (6 * 99981 if level == 1 else 3 * 899981) + 999
    data = KINDS[kind](n, 71)
    ref = M.cut(data, level)
    P = pieces(data)
    assert len(ref) >= 3
    for k in ((1, 2) if level == 1 else (2,)):
        s = ref[k][0]
        ws = w_at(P, s)
        seen = set()
        for j in range(6):
            # the first raw position whose W is at least j past the block start
            x = s
            while x < n and w_at(P, x) < ws + j:
                x += 1
            seen.add(w_at(P, x) - ws)
            check_chain(data, [(0, x), (x, n)], level, ref=ref)
            if level == 1:
                check_chain(data, [(0, x // 2), (x // 2, x), (x, min(n, x + 300000)), (min(n, x + 300000), n)], level, ref=ref)
        assert {0, 1, 2, 3, 4} & seen


@pytest.mark.parametrize("world", [3, 8])
def test_runs_straddling_every_seam(world):
    """Every seam falls inside a long run, at every phase of its 255-chunks."""
    level = 1
    base = bytearray(T.ascii_random(8 * 99981, 5))
    n = len(base)
    bounds = even_bounds(n, world)
    for phase in (1, 4, 5, 255, 256):
        data = bytearray(base)
        for (a, b) in bounds[1:]:
            data[a - phase: a + 700] = b"z" * (phase + 700)
        check_chain(bytes(data), bounds, level)


def test_short_and_empty_shares():
    level = 1
    data = T.texty(9 * 99981 + 55, 8)
    n = len(data)
    cases = [
        [(0, 0), (0, 5000), (5000, 5000), (5000, 80000), (80000, n)],          # empty and short shares
        [(0, n - 10), (n - 10, n - 3), (n - 3, n), (n, n)],                      # short shares at the end, empty last
        [(0, 1), (1, 2), (2, 50000), (50000, 50001), (50001, n)],
        [(0, n), (n, n), (n, n)],
    ]
    for bounds in cases:
        check_chain(data, bounds, level)
    check_chain(b"", [(0, 0), (0, 0)], level)
    check_chain(b"x", [(0, 0), (0, 1)], level)


def test_short_halo_is_reported():
    """A halo too short for a share's last block: the chain is refused (the caller falls back to the whole input);
    a halo that reaches the input's end always suffices (a block of these runs spans about 1.5 MB of raw input)."""
    level = 1
    data = runs_across(8 * 99981, 9)
    bounds = even_bounds(len(data), 4)
    ch, _, _ = chain_of(data, bounds, level, 20000)
    assert ch is None
    ch, _, _ = chain_of(data, bounds, level, len(data))
    assert ch is not None
    check_chain(data, bounds, level, len(data))


def test_chain_rejects_a_contradicting_row():
    ins = [(0, 0, 0, 0, 0), (0, 150000, 1, 0, 100000)]
    good = [[(0, 1, 3, 0)], [(1, 1, 0, S.CUT_BUF_END)] * 5]
    assert S.libbz2_share_chain(ins, 200000, good, 1, [False, True]) == ([(0, 0, 1), (1, 3, 1)], 2)
    bad = [[(0, 1, 3, 0)], [(1, 1, 0, S.CUT_BUF_END | S.CUT_NOT_PIECE)] * 5]
    assert S.libbz2_share_chain(ins, 200000, bad, 1, [False, True]) is None
    assert S.libbz2_share_chain(ins, 200000, good, 1, [False, False]) is None   # the last block needs more input
    arrays = [np.array(t, dtype=np.int32) for t in good]                            # as compress_shares gathers them
    assert S.libbz2_share_chain(ins, 200000, arrays, 1, [False, True]) == ([(0, 0, 1), (1, 3, 1)], 2)


# ---- compress_shares(flavor="libbz2") host logic with gloo, the model standing in for the device calls ------------------
class _ModelLib:
    """The device calls of compress_shares on CPU tensors, computed by the model.  A buffer is known by its data_ptr."""

    def __init__(self, data, level, bufs):
        self.data, self.level, self.bufs, self.P = data, level, bufs, pieces(data)
        self.cached = None

    def b2_bzip2_share_summary(self, ptr, n, out):
        g0, hold = self.bufs[ptr]
        for i, v in enumerate(_py_share_summary(self.data[g0:g0 + n])):
            out[i] = v
        return 0

    def b2_bzip2_share_cut_table(self, ptr, n, level, st_in, w_in, share_len, dmax, tab):
        g0, hold = self.bufs[ptr]
        for d, row in enumerate(model_table(self.P, g0, hold, share_len, w_in, level, dmax)):
            tab[4 * d: 4 * d + 4] = list(row)
        return 0

    def b2_bzip2_plan_share_flavor(self, ptr, n, level, st_in, w_in, first, count, drift, flavor, info):
        assert flavor == S.FLAVORS["libbz2"]
        g0, hold = self.bufs[ptr]
        cut = M.cut(self.data, level)
        blk = model_walk(self.P, first, drift, count, level, g0 + hold)
        assert blk == [s for s, _, _ in cut[first: first + count]]
        self.cached = (ptr, first, count)
        s = blk[0] - g0 if blk else 0
        e = cut[first + count - 1][0] + cut[first + count - 1][1] - g0 if blk else 0
        info[:6] = [s, e, first, count, len(blk), 0]
        return 0

    def b2_bzip2_plan_flavor(self, ptr, n, level, total, flavor):
        """The exact plan of the full-input fallback: the buffer must hold the whole input, gathered from the shares."""
        assert flavor == S.FLAVORS["libbz2"] and C.string_at(ptr, n) == self.data
        total._obj.value = len(M.cut(self.data, level))
        self.cached = (ptr, "exact")
        return 0

    def b2_bzip2_encode_range_dev_flavor(self, ptr, n, level, first, count, phase, out_ptr, cap, bits, crcs, flavor):
        assert self.cached in ((ptr, first, count), (ptr, "exact")) and flavor == S.FLAVORS["libbz2"]
        frag, nb, cr = _block_bits(self.data, level, first, count)
        C.memmove(out_ptr, frag, len(frag))
        bits._obj.value = nb
        for i, c in enumerate(cr):
            crcs[i] = c
        return 0


def _block_bits(data, level, first, count):
    """Blocks [first, first + count) of bz2.compress(data, level) as a fragment from bit 0: each block alone compresses
    to the same block bits, which sit between the 32-bit header and the 80-bit trailer."""
    bits, crcs = [], []
    for s, ln, _ in M.cut(data, level)[first: first + count]:
        raw = data[s: s + ln]
        crc = M.crc32(raw)
        z = np.unpackbits(np.frombuffer(bz2.compress(raw, level), dtype=np.uint8))
        tail = np.unpackbits(np.frombuffer((0x177245385090 << 32 | crc).to_bytes(10, "big"), dtype=np.uint8))
        end = next(len(z) - p for p in range(8) if (z[len(z) - p - 80: len(z) - p] == tail).all())
        bits.append(z[32: end - 80])
        crcs.append(crc)
    a = np.concatenate(bits) if bits else np.zeros(0, np.uint8)
    return np.packbits(a).tobytes() + bytes(8), len(a), crcs


def _worker(rank, world, port, level, kind, n, halo, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from compressjs_b200 import _native
    data = KINDS[kind](n, 31)
    g0, ln, hold = S.share_bounds(n, rank, world, halo)
    buf = torch.frombuffer(bytearray(data[g0:g0 + hold]) + bytearray(1), dtype=torch.uint8)[:hold]
    fake = _ModelLib(data, level, {buf.data_ptr(): (g0, hold)})
    real = _native.lib
    _native.lib = lambda: fake
    try:
        out = S.compress_shares(buf, ln, level, flavor="libbz2")
        fell_back = "fallback_full_input" in S.PHASES
    finally:
        _native.lib = real
    if rank == 0:
        q.put((bytes(out.numpy().tobytes()) == bz2.compress(data, level), fell_back))
    dist.destroy_process_group()


@pytest.mark.skipif(not _libbz2_ok(), reason="bz2 is not linked against libbz2 1.0.3 or later")
@pytest.mark.parametrize("world,kind,n,halo,fallback", [(2, "text", 450000, 150000, False), (3, "maxdrift", 520000, 150000, False),
                                                       (3, "runs", 99981, 150000, False), (3, "runs", 3000000, 20000, True)])
def test_compress_shares_libbz2_host_logic(world, kind, n, halo, fallback):
    """The chained path, and a halo shorter than a block of long runs (a block spans about 1.5 MB of them), where every
    rank gathers the whole input and takes the exact plan: libbz2's bytes either way."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, 1, kind, n, halo, q)) for r in range(world)]
    for p in procs:
        p.start()
    ok, fell_back = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
    assert ok and fell_back == fallback
