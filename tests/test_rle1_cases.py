"""The RLE1 case corpus (tests/rle1_cases.py) reaches every seam it claims, and its model cuts blocks exactly as the
oracle's readBlock does.  tests/test_gpu_rle1_seams.py then holds the GPU to the oracle and to the model's counters.
Also the oracle's own block arrays, which must hold the most blocks an input can have."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import rle1_cases as RC
from tests.test_sharded_host import _py_share_summary


def _names():
    return [c.name for c in RC.cases()]


def test_case_names_are_unique():
    assert len(_names()) == len(set(_names()))


@pytest.mark.parametrize("name", _names())
def test_case_reaches_its_claims_and_cuts_like_the_oracle(name):
    c = RC.case(name)
    m = RC.model(name)
    assert c.claims
    for level in c.levels:
        for what, ok in c.claims:
            assert ok(m, level), "%s level %d: %s" % (name, level, what)
        starts, lens, crcs, _ = O.rle1_split(c.data, level)
        cut = m.cut(level)
        got = [(b.s, b.e - b.s, b.n) for b in cut]
        exp = [(int(s), int(e) - int(s), int(l)) for s, e, l in zip(starts, list(starts[1:]) + [m.n], lens)]
        assert got == exp, "%s level %d: first differing block %s" % (
            name, level, next((k, g, x) for k, (g, x) in enumerate(zip(got + [None] * len(exp), exp + [None] * len(got))) if g != x))


@pytest.mark.parametrize("name", _names())
def test_scan_of_the_tile_summaries_gives_the_carries_and_W(name):
    """Combining the tile states (fast-path tiles with their capped leads and trails included) must give the run that
    enters every tile and W at every tile start, whatever the buffer alignment."""
    m = RC.model(name)
    exp_carry = m.carry_from_data()
    exp_W = [int(m.W[t0]) for t0 in range(0, m.n, RC.TILE)] + [int(m.W[m.n])]
    for mis in ((0, 1) if m.n < (4 << 20) else (0,)):
        carry, pref, groups, _ = m.scan(mis)
        assert carry == exp_carry, (name, mis)
        assert pref == exp_W, (name, mis)
        assert len(groups) == m.ngroups()
        if mis:
            assert not any(t[0] for t in m.tiles(mis)), "no fast path on a misaligned buffer"


def test_share_summary_model_matches_the_plain_restatement():
    for name in ("edge_runs", "lookback", "run509_at_start", "phases_l1_last1"):
        c = RC.case(name)
        m = RC.model(name)
        n = m.n
        for g0, g1 in ((0, n), (1, n - 1), (n // 3, 2 * n // 3), (0, 1), (n - 5, n)):
            assert m.share_summary(g0, g1) == _py_share_summary(c.data[g0:g1]), (name, g0, g1)
    # inside one long run
    data = b"xy" + b"q" * 3000 + b"z"
    m = RC.Model(data)
    for g0, g1 in ((2, 3002), (5, 600), (0, 3003), (2, 258)):
        assert m.share_summary(g0, g1) == _py_share_summary(data[g0:g1]), (g0, g1)


def test_corpus_reaches_every_path():
    """Across the corpus: the group scan with and without the hook on >= 3 groups, the accepted speculative walk and
    its serial fallback, the block that fills inside its re-phased first run, and every run phase of interest carried
    into a group."""
    groups_default = groups_hook = par = ser = 0
    fill_first = False
    group_carries = set()
    for c in RC.cases():
        m = RC.model(c.name)
        if c.groups_hook:
            group_carries |= m.crossing_carries(RC.group_edges(m))
        for lv in c.levels:
            g, p, s = m.counters(lv)
            if g and m.ngroups() >= 3:
                groups_default += 1
            if c.groups_hook and m.ngroups() >= 3:
                groups_hook += 1
            par += p
            if m.parallel_walk(lv) is not None and not p:
                ser += 1
            fill_first |= any(b.kind == "fill_first_run" for b in m.cut(lv))
    assert groups_default and groups_hook and par and ser and fill_first
    # runs of 0, 1, 3, 4 and 5 (mod 255) go on across a group edge in the cases that also run with the hook
    assert {0, 1, 3, 4, 5} <= group_carries


def test_share_edges_fall_inside_planted_runs():
    """Every case with simulated ranks cuts a share inside a run of 600 bytes or more (the run state and RLE1 output in
    front of the next share then carry that run), except the run-free texts."""
    for c in RC.cases():
        m = RC.model(c.name)
        inside = []
        for world, _ in c.shares:
            edges = RC.share_edges(c, world)
            assert all(a < b for a, b in zip(edges, edges[1:])), (c.name, world, edges)
            inside += [e for e in edges[1:-1] if m.view.run_end(e) - m.view.run_start(e) >= 600 and m.a[e - 1] == m.a[e]]
        assert inside or not c.shares or c.name.startswith(("spec_", "slip_")), c.name


def test_outfresh_and_cneed():
    for t in range(1, 3000):
        c = RC.cneed(t)
        assert RC.outfresh(c) >= t and (c == 1 or RC.outfresh(c - 1) < t)


@pytest.mark.parametrize("level", [1, 9])
def test_oracle_block_arrays_hold_runs_of_four(level):
    """Runs of exactly four give 5 RLE1 bytes per 4 raw bytes, so a block can hold as few as 4/5 of blockSize raw
    bytes: the oracle's block split, its traced compress and its multi-threaded compress must size their block arrays
    for that, and agree with the stream's own block table."""
    BS = level * 100000 - 19
    data = b"aaaabbbb" * (12 * (BS + 19) // 8)
    starts, lens, crcs, blocks = O.rle1_split(data, level)
    z, tr = O.bzip2_compress(data, level, trace=True)
    table = O.bzip2_table(z)
    assert len(starts) == len(tr) == len(table) > len(data) // BS + 2
    assert [t.raw_start for t in tr] == [int(s) for s in starts]
    assert [t.crc for t in tr] == [int(x) for x in crcs]
    assert O.bzip2_compress(data, level, threads=4) == z
    assert O.bzip2_decompress(z) == data
