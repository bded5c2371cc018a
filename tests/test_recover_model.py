"""The recovery model (tests/recover_model.py) against a second, independent side: bzip2recover's cut of seeded damaged
files and what libbz2 accepts of its rec*.bz2 files (tests/golden/recover.json, made by
tests/golden/make_recover_golden.py), and the properties every recovery must have."""
import bz2
import hashlib
import json
import os

import pytest

from oracle import oracle as O
from tests import bz2synth as W
from tests import recover_cases as RC
from tests import recover_golden_cases as G
from tests import recover_model as M
from tests import util as T

GOLDEN = json.load(open(os.path.join(T.ROOT, "tests", "golden", "recover.json")))


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_model_matches_bzip2recover_and_libbz2(case):
    spec = {k: case[k] for k in ("name", "seed", "n", "level", "damage")}
    assert spec in G.SPECS
    data = G.build(spec)
    assert hashlib.sha256(data).hexdigest() == case["sha256"]   # the input is the one the golden was made from
    m = M.recover(data)
    before = W.magic_positions(G.undamaged(spec))
    if W.magic_positions(data) == before and len(case["files"]) == len(case["ranges"]):
        # every magic survived: the blocks libbz2 accepts from bzip2recover's files are the model's intact ones
        accepted = [(s - 48, f["sha256"]) for (s, _), f in zip(case["ranges"], case["files"]) if f["ok"]]
        intact = [r for r in m.rows if r.status == M.INTACT]
        assert [p for p, _ in accepted] == [r.bitpos for r in intact]
        B = b"BZh9" + data
        assert [h for _, h in accepted] == [hashlib.sha256(M.decode_block(B, r.bitpos + 32)[2]).hexdigest() for r in intact]
        assert m.rows == [r for r in m.rows if r.status != M.INSIDE] and len(m.rows) == len(case["ranges"])
    check_properties(data, m)
    assert bz2.decompress(m.stream) == m.data


def check_properties(data, m):
    """The properties of include/b2bz.h b2_bzip2_recover that hold for every input."""
    off = 0
    end = 0
    for r in m.rows:
        assert r.out_off == off
        if r.status == M.INSIDE:
            assert r.bitpos < end and (r.endbit, r.size, r.got) == (0, 0, 0)
            continue
        assert r.bitpos >= end
        if r.status in (M.INTACT, M.BAD_CRC):
            assert r.endbit > r.bitpos and (r.got == r.crc) == (r.status == M.INTACT)
        else:
            assert (r.endbit, r.size, r.got) == (0, 0, 0)
        if r.status == M.INTACT:
            off += r.size
            end = r.endbit
    assert off == len(m.data)
    assert O.bzip2_decompress(m.stream) == m.data      # the repaired stream decodes to the recovered bytes
    if not any(r.status == M.INTACT for r in m.rows):
        assert len(m.stream) == 14


@pytest.mark.parametrize("name", sorted(RC.by_name()))
def test_corpus_case(name):
    c = RC.by_name()[name]
    m = M.recover(c.data)
    c.check(m.rows)
    check_properties(c.data, m)
    if M.libbz2_language(c.data, m.rows):
        assert bz2.decompress(m.stream) == m.data


def test_undamaged_properties():
    for name in ("undamaged_l1", "undamaged_l9", "multistream_levels_1_9", "undamaged_compressjs"):
        data = RC.by_name()[name].data
        assert M.recover(data).data == O.bzip2_decompress(data, True)
    data = RC.by_name()["undamaged_l1"].data
    assert M.recover(data).stream == data[:3] + b"9" + data[4:]


def test_candidates_match_a_second_scan():
    for c in RC.cases():
        assert M.candidates(c.data) == W.magic_positions(c.data)[0], c.name
