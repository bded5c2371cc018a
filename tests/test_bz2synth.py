"""The synthetic-stream writer (tests/bz2synth.py) pinned on the CPU: it reproduces the oracle encoder bit for bit, and
every corpus case (tests/synth_corpus.py) reaches the condition it names and decodes, with the oracle and with
libbz2 where the stream is in libbz2's language, to the writer's expected bytes or error code."""
import bz2

import numpy as np
import pytest

from oracle import oracle as O
from tests import bz2synth as W
from tests import synth_corpus as C
from tests import util as T


def _oracle(fn, *a, **kw):
    try:
        return ("ok", fn(*a, **kw))
    except O.OracleError as e:
        return ("err", e.errorCode)


def test_crc_matches_oracle():
    for n, seed in ((0, 1), (1, 2), (1000, 3), (65537, 4)):
        d = T.rng(seed).integers(0, 256, size=n, dtype=np.uint8).tobytes()
        assert W.crc32(d) == O.crc32(d)


@pytest.mark.parametrize("kind", ["ascii", "text", "runs"])
def test_writer_reproduces_oracle_encoder(kind):
    """Tables, selectors and symbols from the oracle encoder, fed to the writer: the block body bits are identical."""
    raw = {"ascii": T.ascii_random, "text": T.texty, "runs": T.runs}[kind](60000, 5)
    _, lens_, crcs, blocks = O.rle1_split(raw, 1)
    blk = blocks[0][:int(lens_[0])].tobytes()
    st = O.compress_block_stages(blk)
    tr = st["trace"]
    b = W.block(st["sym"].tolist(), sorted(set(blk)), tr.pidx, level=1, lens=st["lens"].tolist(), tables=st["sel"].tolist())
    want = np.unpackbits(np.frombuffer(st["bits"], np.uint8))[:st["nbits"]]
    assert b.bits.size - 80 == st["nbits"]
    assert np.array_equal(b.bits[80:], want)
    assert b.report["B"].tobytes() == blk           # the inverse-BWT model recovers the block
    assert b.crc == int(crcs[0])


def test_decode_bits_plants_a_pattern():
    lens = [8] * 255
    lens[2] = 7
    syms = W.decode_bits("{:048b}".format(W.BLOCK_MAGIC), lens)
    codes = W.canonical_codes(lens)
    assert "".join("{:0{}b}".format(codes[s], lens[s]) for s in syms) == "{:048b}".format(W.BLOCK_MAGIC)


def test_selector_mtf_list_is_zero_filled():
    # index groupCount pulls slot groupCount (0); that slot then holds the old last entry
    assert W.selectors_from_mtf([6, 0, 6, 6], 6) == [0, 0, 5, 4]
    with pytest.raises(W.ModelError):
        W.selectors_from_mtf([7], 6)


@pytest.mark.parametrize("name", sorted(C.CASES))
def test_corpus_case_vs_oracle(name):
    c = C.build(name)
    assert all(c.cond.values()), {k: v for k, v in c.cond.items() if not v}
    f = c.file
    exp = f.expect()
    assert _oracle(O.bzip2_decompress, f.data) == exp
    t = f.expect_table()
    got = _oracle(O.bzip2_table, f.data)
    assert got == (t if t[0] == "err" else ("ok", t[1]))
    for pos, b in f.member_blocks[0]:
        e = ("err", b.err) if b.err is not None else (("ok", b.out) if W.crc32(b.out) == b.crc else ("err", W.DATA_ERROR))
        assert _oracle(O.bzip2_decompress_block, f.data, pos) == e


@pytest.mark.parametrize("name", sorted(n for n in C.CASES if C.build(n).libbz2))
def test_corpus_case_vs_libbz2(name):
    f = C.build(name).file
    exp = f.expect()
    if exp[0] == "ok":
        assert bz2.decompress(f.data) == exp[1]
    else:
        with pytest.raises((OSError, ValueError, EOFError)):
            bz2.decompress(f.data)


def test_multistream_file():
    f = C.multistream_file()
    assert f.expect(True)[0] == "ok" and f.expect(True) != f.expect(False)
    assert _oracle(O.bzip2_decompress, f.data, multistream=True) == f.expect(True)
    assert _oracle(O.bzip2_decompress, f.data) == f.expect(False)
    assert bz2.decompress(f.data) == f.expect(True)[1]


def test_model_rle1_loop():
    # the reference's loop: the byte behind four equal bytes is a count, then the run starts afresh
    out, is_count, pending = W.model_rle1(np.frombuffer(b"aaaa\x02aaaa\x00cbbbb", np.uint8))
    assert out.tobytes() == b"aaaaaa" + b"aaaa" + b"c" + b"bbbb" and pending
    assert np.flatnonzero(is_count).tolist() == [4, 9]


def test_error_blocks_carry_the_crc_of_their_unchecked_output():
    """A rejected block's CRC is that of what it decodes to without the failing check, so a decoder that skips the
    check returns bytes instead of the error; the only exception is a block without a defined output."""
    for name in sorted(C.CASES):
        for b in C.build(name).file.members[0].blocks:
            if b.err is not None:
                assert b.would_be is not None and b.crc == W.crc32(b.would_be), (name, b.failed)
    rel = C.relevelled()
    assert {n for n, _, _ in rel} >= {"run_past_dbuf", "run18_l1", "run19_l1", "n_dbuf_plus1_l1"}
    for name, f, would_be in rel:
        assert _oracle(O.bzip2_decompress, f.data) == ("ok", would_be), name
