"""The libbz2 model (tests/libbz2_model.py) writes the bytes of bz2.compress, the case corpus (tests/libbz2_cases.py)
reaches every corner it claims, and tests/golden/libbz2.json holds libbz2's output for that corpus.
tests/test_gpu_bzip2_libbz2.py then holds the GPU's libbz2 flavor to all three."""
import bz2
import hashlib
import json
import os

import numpy as np
import pytest

from tests import libbz2_cases as LC
from tests import libbz2_model as M
from tests.util import ascii_random, runs, texty

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "libbz2.json")


def _libbz2_ok():
    """bz2 is linked against libbz2 1.0.3 or later (the table search this flavor writes)."""
    import ctypes
    import ctypes.util
    import _bz2
    try:
        lib = ctypes.CDLL(_bz2.__file__)
        lib.BZ2_bzlibVersion.restype = ctypes.c_char_p
        v = lib.BZ2_bzlibVersion().decode().split(",")[0]
    except (OSError, AttributeError):
        name = ctypes.util.find_library("bz2")
        if not name:
            return False
        lib = ctypes.CDLL(name)
        lib.BZ2_bzlibVersion.restype = ctypes.c_char_p
        v = lib.BZ2_bzlibVersion().decode().split(",")[0]
    return tuple(int(x) for x in v.split(".")[:3]) >= (1, 0, 3)


needs_libbz2 = pytest.mark.skipif(not _libbz2_ok(), reason="bz2 is not linked against libbz2 1.0.3 or later")

SMALL = [(b"", 1), (b"a", 1), (b"hello world\n", 9), (b"ab" * 50, 1), (b"a" * 1000 + b"b" * 300 + b"a" * 4, 1),
         (ascii_random(3000, 1), 1), (texty(22000, 2), 1), (texty(22000, 2), 9), (runs(40000, 3), 1)]


@needs_libbz2
@pytest.mark.parametrize("k", range(len(SMALL)))
def test_model_matches_libbz2(k):
    data, level = SMALL[k]
    assert M.compress(data, level) == bz2.compress(data, level)


@needs_libbz2
def test_model_matches_libbz2_across_blocks():
    data = texty(210000, 4)
    assert M.compress(data, 1) == bz2.compress(data, 1)


def _cut_names():
    return [c[0] for c in LC.cut_cases()]


def _table_names():
    return [c[0] for c in LC.table_cases()]


def test_case_names_are_unique():
    names = _cut_names() + _table_names()
    assert len(names) == len(set(names))


@pytest.mark.parametrize("name", _cut_names())
def test_cut_case_hits_its_corner(name):
    _, data, level, expect = next(c for c in LC.cut_cases() if c[0] == name)
    LC.check_cut_case(data, level, expect)


@pytest.mark.parametrize("name", _table_names())
def test_table_case_hits_its_corner(name):
    _, data, level, corner = next(c for c in LC.table_cases() if c[0] == name)
    LC.check_table_case(data, level, corner)


@needs_libbz2
@pytest.mark.parametrize("name", _table_names() + ["runfree_then_aaaa"])
def test_model_matches_libbz2_on_case(name):
    _, data, level, _ = next(c for c in LC.cut_cases() + LC.table_cases() if c[0] == name)
    assert M.compress(data, level) == bz2.compress(data, level)


def test_cut_is_independent_of_feeding():
    """libbz2's cut does not depend on how the input reaches it: BZ2Compressor fed in odd pieces gives bz2.compress."""
    data = LC.motivating() + runs(300000, 5)
    c = bz2.BZ2Compressor(1)
    parts, i, rng = [], 0, np.random.default_rng(3)
    while i < len(data):
        k = int(rng.integers(1, 70000))
        parts.append(c.compress(data[i:i + k]))
        i += k
    parts.append(c.flush())
    assert b"".join(parts) == bz2.compress(data, 1)


def test_motivating_case_is_what_the_issue_says():
    """compressjs would close block 1 on four equal bytes: 99 977 run-free bytes leave 4 RLE1 bytes of room."""
    blocks = M.cut(LC.motivating(), 1)
    assert blocks[0][1] == 99977 + 255 and len(blocks[0][2]) == LC.nmax(1) + 1


@needs_libbz2
def test_golden_file_matches_libbz2():
    gold = json.load(open(GOLDEN))
    keys = set()
    for key, data, level in LC.golden_corpus():
        z = bz2.compress(data, level)
        assert gold[key] == {"size": len(z), "sha256": hashlib.sha256(z).hexdigest()}, key
        keys.add(key)
    assert keys == set(gold)
