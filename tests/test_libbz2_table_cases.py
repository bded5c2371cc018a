"""The designed table-search corpus of tests/libbz2_table_cases.py reaches every corner it claims in the libbz2 model,
the model writes libbz2's bytes for every case, and its per-block trace tiles the input.  For every case of
tests/mtfhuff_cases.py it also states whether libbz2's block cut keeps the designed blocks (the GPU test runs both
corpora through the libbz2 flavor)."""
import bz2

import pytest

from tests import libbz2_model as M
from tests import libbz2_table_cases as TC
from tests.test_libbz2_model import needs_libbz2

NAMES = [c.name for c in TC.cases()]


def test_case_names_are_unique():
    assert len(NAMES) == len(set(NAMES))


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_claims(name):
    ci = TC.info(name)
    assert len(ci.blocks) == 1, "%s: %d blocks" % (name, len(ci.blocks))
    assert not ci.holds(), "%s misses: %s" % (name, ci.holds())


def test_largest_rescale_count():
    """One rescale flattens a chain a lot: the most any build of the corpus reaches is two (recorded, not a corner)."""
    most = max(x["rescales"] for n in NAMES for b in TC.info(n).blocks for rd in b["report"]["rounds"]
               for x in rd["tables"])
    assert most == 2


@needs_libbz2
@pytest.mark.parametrize("name", NAMES)
def test_model_matches_libbz2(name):
    ci = TC.info(name)
    for lv in ci.case.levels:
        z = ci.stream if lv == ci.case.levels[0] else M.compress(ci.raw, lv)
        assert z == bz2.compress(ci.raw, lv), "%s level %d" % (name, lv)


@needs_libbz2
@pytest.mark.parametrize("name", NAMES)
def test_model_trace_is_the_reference_trace(name):
    """The GPU test holds b2_last_trace to reference_trace (oracle blocks, bit lengths from libbz2's stream), which
    takes no Python model run: here the model's trace is that trace."""
    ci = TC.info(name)
    lv = ci.case.levels[0]
    ref = TC.reference_trace(ci.raw, lv, bz2.compress(ci.raw, lv)).tolist()
    assert ref == [[b[f] for f in M.TRACE_FIELDS] for b in ci.blocks]


@pytest.mark.parametrize("name", NAMES)
def test_trace_tiles_the_input(name):
    ci = TC.info(name)
    pos = 0
    for b in ci.blocks:
        assert b["raw_start"] == pos and b["raw_len"] > 0
        assert b["nsel"] == (b["m"] + 49) // 50 and b["ngroups"] == M.n_groups(b["m"])
        pos += b["raw_len"]
    assert pos == len(ci.raw)


# mtfhuff cases whose designed blocks libbz2's cut does not keep (a full block that libbz2 ends on another whole RLE1
# piece); none today: every designed full block ends where both cuts end it
MTFHUFF_RECUT = set()


def _mtfhuff_names():
    from tests import mtfhuff_cases as MC
    return [c.name for c in MC.cases()]


@pytest.mark.parametrize("name", _mtfhuff_names())
def test_mtfhuff_case_blocks_under_libbz2_cut(name):
    from tests import mtfhuff_cases as MC
    ci = MC.info(name)
    for lv in ci.case.levels:
        keep = [b[2] for b in M.cut(ci.raw, lv)] == [b.T.tobytes() for b in ci.built]
        if len(ci.built) == 1:
            assert keep, "%s level %d: libbz2's cut does not keep the single designed block" % (name, lv)
        elif lv == ci.case.levels[0]:
            assert keep == (name not in MTFHUFF_RECUT), "%s level %d: libbz2's cut %s the designed blocks" % (
                name, lv, "keeps" if keep else "moves")
