"""GPU parity of the MTF stage on blocks that hold all 256 byte values, most of them rare.

The MTF kernels (mtf.cu) split a block into 4 KiB chunks.  A rare byte's previous use lies many chunks back, its recency
key sits deep in the list at a chunk start, and its key moves across the bucket boundaries of the live-key bitmap.  The
other parity inputs (ASCII, text, small fuzz) never put a full 256-value alphabet with rare values into a 900k block.
"""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import util as T

pytestmark = pytest.mark.gpu


def _rare_symbols(n, seed, a=2.0):
    """All 256 byte values with Zipf(a) weights over a seeded permutation; every value occurs at least once."""
    g = T.rng(seed)
    w = 1.0 / np.arange(1, 257) ** a
    d = g.permutation(256).astype(np.uint8)[g.choice(256, size=n, p=w / w.sum())]
    d[g.permutation(n)[:256]] = np.arange(256, dtype=np.uint8)
    return d.tobytes()


def test_rare_symbols_full_alphabet_vs_oracle():
    from compressjs_b200 import Bzip2
    bs = 899981
    # Zipf(2): the rarest values occur 5-8 times per block; Zipf(1.2): a flatter tail; then ASCII behind them
    data = _rare_symbols(2 * bs, 44) + _rare_symbols(bs, 45, 1.2) + T.ascii_random(bs // 2, 46)
    got = Bzip2.compressFile(data, None, 9)
    exp = O.bzip2_compress(data, 9, threads=min(os.cpu_count() or 1, 8))
    assert got == exp
    assert Bzip2.decompressFile(got) == data
