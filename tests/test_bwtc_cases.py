"""The BWTC case corpus (tests/bwtc_cases.py) reaches what each case claims, on the oracle's trace; the oracle's streams
decode back; every stream fits the coder's output window (bwtc_window_bound), and the worst-growth cases exceed the
parent's bound, which they were built to break."""
import pytest

from oracle import oracle as O
from tests import bwtc_cases as BC

JOBS = [(c.name, lv) for c in BC.cases() for lv in c.levels]


@pytest.mark.parametrize("name,level", JOBS, ids=["%s@%d" % j for j in JOBS])
def test_case_reaches_its_claims(name, level):
    ci = BC.info(name, level)
    missed = [what for what, f in BC.case(name).claims if not f(ci)]
    assert not missed, missed
    assert O.bwtc_decompress(ci.z) == ci.raw
    nb = len(ci.blocks)
    assert nb == max(1, -(-len(ci.raw) // BC.block_size(level))) or (not ci.raw and nb == 0)
    assert ci.coded() + ci.file.max_help <= BC.window_bound(len(ci.raw), nb, level)
    # r = umulhi(range, 0xFFFFFFFF / tot) is at most one short of range / tot (range <= 2^31, so the product's error is
    # under 1): k_bwtc_code's correction loop never takes a second step.
    assert ci.file.corr2 == 0
    # the level byte is coded first and leaves low's top byte at the level: nothing carries into the size field's last group
    assert ci.file.first_carry == 0


@pytest.mark.parametrize("level", [6, 9])
def test_worst_growth_exceeds_the_parent_bound(level):
    """One block of cycling ranks grows by 14 %, past n + n / 8 + 3 KiB + 64; three of them past the bound of three."""
    one, three = BC.info("worst_growth_l%d" % level, level), BC.info("worst_growth_l%d_x3" % level, level)
    assert one.coded() > BC.old_bound(len(one.raw)) and one.coded() > 1.14 * len(one.raw)
    assert three.coded() > BC.old_bound(len(three.raw))
