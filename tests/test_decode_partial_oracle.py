"""What a failed decode has delivered, pinned on the CPU: for every synthetic case (tests/partial_cases.py), the oracle
decoder's bytes and table rows in front of the error equal the model's, for decompress, table and decompressBlock, with
the error code the unchanged oracle and model give."""
import pytest

from oracle import oracle as O
from tests import bz2synth as W
from tests import partial_cases as P

FILES = {name: (f, ms) for name, f, ms in P.files()}


def _code(fn, *a, **kw):
    try:
        return ("ok", fn(*a, **kw))
    except O.OracleError as e:
        return ("err", e.errorCode)


@pytest.mark.parametrize("name", sorted(FILES))
def test_partial_output_matches_model(name):
    f, ms = FILES[name]
    exp = f.expect(ms)
    got = P.oracle_decompress(f.data, ms)
    assert got == (exp if exp[0] == "ok" else ("err", exp[1], P.expect_partial(f, ms)))
    assert got[:2] == _code(O.bzip2_decompress, f.data, multistream=ms)[:2]
    t = f.expect_table()
    got = P.oracle_table(f.data)
    assert got == (t if t[0] == "ok" else ("err", t[1], P.expect_table_partial(f)))
    assert got[:2] == _code(O.bzip2_table, f.data)[:2]
    for pos, b in f.member_blocks[0]:
        got = P.oracle_decompress_block(f.data, pos)
        assert got == P.block_expect(b), pos
        assert got[:2] == _code(O.bzip2_decompress_block, f.data, pos)[:2], pos


def test_variants_reach_what_they_name():
    """The variants fail after some output: a CRC-failing block delivers its bytes, a later member's error the earlier
    members."""
    n_crc = 0
    for name, (f, ms) in FILES.items():
        if name.endswith("+crc"):
            n_crc += 1
            assert f.expect(ms)[0] == "err" and len(P.expect_partial(f, ms)) > len(f.members[0].blocks[0].out), name
            assert len(P.expect_table_partial(f)) >= 1, name
    assert n_crc >= 40
    first = b"".join(b.out for b in FILES["multistream"][0].members[0].blocks)
    f, ms = FILES["multistream+level0"]
    assert f.expect(ms) == ("err", W.NOT_BZIP) and P.expect_partial(f, ms) == first
    f, ms = FILES["multistream+stream_crc"]
    assert f.expect(ms) == ("err", W.DATA_ERROR)
    assert P.expect_partial(f, ms) == first + b"".join(b.out for b in f.members[1].blocks)


def test_no_output_on_error_without_a_prefix():
    """A header the decoder rejects delivers nothing; the model's partial is empty there too."""
    f = W.File(W.Member([P.lead()], level_byte=ord("0")))
    assert f.expect() == ("err", W.NOT_BZIP) and P.expect_partial(f) == b""
    assert P.oracle_decompress(f.data) == ("err", W.NOT_BZIP, b"")


def test_oracle_results_on_success_are_the_oracles():
    from tests import util as T
    for k in range(5):
        z = T.fixture("sample%d.bz2" % k)
        assert P.oracle_decompress(z) == ("ok", O.bzip2_decompress(z))
        assert P.oracle_table(z) == ("ok", O.bzip2_table(z))
