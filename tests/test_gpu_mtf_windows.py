"""GPU parity of the move-to-front ranks and the zero-run coder on blocks shaped for their step and tile structure.

`k_mtf_ranks` ranks 32 bytes per step and orders the bytes of a step that repeat each other by their previous use in the
step; it summarises each 4 KiB chunk's zero runs from the bitmap of its non-zero ranks after the last step.  These
blocks put every step's bytes into a repeat (2-4 symbol alphabets), make one run of rank 0 span many chunks and tiles
(a periodic input, whose BWT column is a few long runs), use all 256 byte values, and fill a block to the byte (an
input of exactly 900 000 bytes: one full block of 899 981 bytes at -9 and a short one behind it).  Each stream is
compared to the oracle's at level 9 and decoded back.
"""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import util as T

pytestmark = pytest.mark.gpu


def _low_alphabet(n, k, seed):
    """n bytes over k symbols with no run of 4 (RLE1 leaves the block as it is)."""
    g = T.rng(seed)
    d = g.integers(0, k, size=n, dtype=np.uint8)
    d[2::3] = (d[1::3][: d[2::3].size] + 1) % k  # the last byte of every aligned triple differs from the one before
    return (d + 97).tobytes()


def _periodic(n, word):
    return (word * (n // len(word) + 1))[:n]


def _all_bytes(n, seed):
    g = T.rng(seed)
    d = g.integers(0, 256, size=n, dtype=np.uint8)
    d[g.permutation(n)[:256]] = np.arange(256, dtype=np.uint8)
    return d.tobytes()


CASES = {
    "alphabet2": lambda: _low_alphabet(600000, 2, 71),
    "alphabet3": lambda: _low_alphabet(600000, 3, 72),
    "alphabet4": lambda: _low_alphabet(600000, 4, 73),
    "rank0_run_abc": lambda: _periodic(899981, b"abc"),
    "rank0_run_text": lambda: _periodic(700000, b"the quick brown fox ") + T.ascii_random(50000, 74),
    "all_bytes": lambda: _all_bytes(899981, 75),
    "exact_900000": lambda: _all_bytes(900000, 76),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_mtf_windows_vs_oracle(name):
    from compressjs_b200 import Bzip2
    data = CASES[name]()
    got = Bzip2.compressFile(data, None, 9)
    exp = O.bzip2_compress(data, 9, threads=min(os.cpu_count() or 1, 8))
    assert got == exp
    assert Bzip2.decompressFile(got) == data
