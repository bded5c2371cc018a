"""The MTF / zero-run / Huffman case corpus (tests/mtfhuff_cases.py) reaches every seam it claims.

For every case: the encoder's RLE1 stage reads the raw input back as exactly the designed blocks, the oracle's BWT
of each block is the column the case ended up with, bz2synth's independent model of the MTF + zero-run stage gives
the oracle's symbols, the plain model of the table search gives the oracle's selectors and code lengths, and every
named predicate holds.  tests/test_gpu_mtfhuff_seams.py then holds the GPU to the oracle on the same inputs.
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests import bz2synth as S
from tests import mtfhuff_cases as MC


def _names():
    return [c.name for c in MC.cases()]


def test_case_names_are_unique():
    assert len(_names()) == len(set(_names()))


@pytest.mark.parametrize("name", _names())
def test_case_reaches_its_claims(name):
    c = MC.case(name)
    ci = MC.info(name)
    assert c.claims
    for level in c.levels:
        _, lens, _, blocks = O.rle1_split(ci.raw, level)
        assert [int(x) for x in lens] == [b.T.size for b in ci.built], (name, level)
        for k, b in enumerate(ci.built):
            assert np.array_equal(blocks[k][:b.T.size], b.T), (name, level, k)
    for k, (b, st) in enumerate(zip(ci.built, ci.blocks)):
        L, pidx = O.bwt_cyclic(b.T.tobytes())
        assert L == b.L.tobytes() and pidx == b.pidx, (name, k)
        sym, used = S.mtf_symbols(b.L)
        assert sym == st["sym"].tolist(), (name, k, "the oracle's symbols differ from the model's")
        sel, tables, _, _ = ci.searches[k]
        assert sel.tolist() == st["sel"].tolist(), (name, k, "selectors")
        assert np.array_equal(np.array(tables, np.uint8), st["lens"]), (name, k, "code lengths")
    for what, ok in c.claims:
        assert ok(ci), "%s: %s" % (name, what)


def test_corpus_reaches_the_table_search_seams():
    """Across the corpus: every table count, the 20-bit limit, the empty thread runs of the selector MTF (nsel not a
    multiple of 256), and a block whose selectors fill every thread run."""
    ngroups, limit, nsel = set(), False, set()
    for c in MC.cases():
        for st in MC.info(c.name).blocks:
            ngroups.add(int(st["trace"].ngroups))
            nsel.add(int(st["trace"].nsel))
            limit |= int(st["lens"].max()) == MC.MAX_LEN
    assert ngroups == {2, 3, 4, 5, 6} and limit
    assert {0, 1, 255} <= {k % MC.TILE_GROUPS for k in nsel} and min(nsel) < MC.TILE_GROUPS and max(nsel) >= 17900


def test_unmtf_inverts_the_rank_model():
    g = np.random.default_rng(3)
    used = sorted(g.choice(256, size=37, replace=False).tolist())
    ranks = np.concatenate([np.arange(1, 37), g.integers(0, 37, size=5000)])   # every byte used
    L = MC.unmtf(ranks, used)
    assert sorted(set(L.tolist())) == used
    assert np.array_equal(MC.mtf_ranks(L), ranks)


def test_merge_cycles_gives_one_cycle_and_a_block():
    g = np.random.default_rng(4)
    L0 = MC.unmtf(g.integers(0, 9, size=3000), list(range(97, 106)))
    L, swaps = MC.merge_cycles(L0)
    assert MC.cycles(L)[0] == 1 and swaps > 0
    assert int((L != L0).sum()) <= 2 * swaps
    T = S.model_ibwt(L, 0)[0]
    assert O.bwt_cyclic(T.tobytes())[0] == L.tobytes()


def test_merge_cycles_reaches_fixed_points_inside_a_run():
    """L = a a a a a b c: rows 0..4 are fixed points of LF inside the run of a, which covers a's own F bucket, and rows
    1..3 have no different neighbour; swapping the run's edge byte pass after pass merges them all."""
    L0 = np.frombuffer(b"aaaaabc", np.uint8).copy()
    assert MC.cycles(L0)[0] == 7
    L, swaps = MC.merge_cycles(L0)
    assert MC.cycles(L)[0] == 1 and swaps >= 6
    T = S.model_ibwt(L, 0)[0]
    assert O.bwt_cyclic(T.tobytes())[0] == L.tobytes()


def test_construction_repairs():
    """The RLE1 repair, which recomputes the column from a changed block, is left to three small designs; the claims
    of every case are checked on the column it ended up with."""
    rle1 = [c.name for c in MC.cases() if any(b.rle1_repair for b in MC.info(c.name).built)]
    assert rle1 == ["len_4096k_plus_1", "len_4096k_plus_31", "nsel_511"]
