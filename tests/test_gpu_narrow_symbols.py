"""GPU parity of the one-byte symbol format on blocks that use every byte value.

The zero-run coder (mtf.cu) stores every symbol in one byte; the two that do not fit, 256 (MTF rank 255) and 257 (the
end of block when all 256 byte values occur), set a bit in a per-group mask instead.  The Huffman search, the packer
and the BWTC models all read that format back.  Under uniform random bytes the MTF rank is uniform on 0..255, so
symbol 256 lands about 3,500 times in a 900k block: at every residue mod 50 and on both sides of the 4096-rank tiles
of the zero-run coder.  ASCII and text never produce either symbol.
"""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import util as T

pytestmark = pytest.mark.gpu

THREADS = min(os.cpu_count() or 1, 8)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _uniform(n, seed):
    return T.rng(seed).integers(0, 256, size=n, dtype=np.uint8).tobytes()


def _data(level):
    bs = level * 100000 - 19
    if level == 1:
        # a batch that mixes blocks with and without symbols >= 256, and a short last block
        return _uniform(3 * bs, 71) + T.ascii_random(2 * bs, 72) + _uniform(bs + bs // 3, 73)
    return _uniform(2 * bs + bs // 2, 91)


def _stages(block):
    st = O.compress_block_stages(block)
    sym = st["sym"]
    assert int(sym[-1]) == 257  # every byte value occurs: the end of block symbol does not fit a byte
    return sym


def test_uniform_blocks_reach_every_group_residue():
    """The inputs below do what the module promises: symbol 256 at every position of a group."""
    sym = _stages(_uniform(899981, 91))
    pos = np.flatnonzero(sym == 256)
    assert len(pos) > 2000
    assert set((pos % 50).tolist()) == set(range(50))


@pytest.mark.parametrize("level", [1, 9])
def test_uniform_bytes_vs_oracle(level):
    from compressjs_b200 import Bzip2
    data = _data(level)
    got = Bzip2.compressFile(data, None, level)
    assert got == O.bzip2_compress(data, level, threads=THREADS)
    assert Bzip2.decompressFile(got) == data


def _eob_residue_blocks():
    """Single blocks whose end of block symbol 257 sits at different positions of its group, found by trimming one
    random buffer: m % 50 == 0 puts it at the end of a full group."""
    base = _uniform(40000, 5)
    want = {0: None, 1: None, 2: None, 25: None, 49: None}
    n = len(base)
    while any(v is None for v in want.values()):
        m = len(_stages(base[:n]))
        if m % 50 in want and want[m % 50] is None:
            want[m % 50] = base[:n]
        n -= 1
        assert n > 30000
    return want


def test_eob_257_at_group_residues_vs_oracle():
    from compressjs_b200 import BWTC, Bzip2
    for r, block in sorted(_eob_residue_blocks().items()):
        for level in (1, 9):
            got = Bzip2.compressFile(block, None, level)
            assert got == O.bzip2_compress(block, level), (r, level)
            assert Bzip2.decompressFile(got) == block
        z = BWTC.compressFile(block, None, 9)
        assert z == O.bwtc_compress(block, 9), r
        assert BWTC.decompressFile(z) == block


@pytest.mark.parametrize("level", [1, 9])
def test_bwtc_uniform_bytes_vs_oracle(level):
    from compressjs_b200 import BWTC
    data = _data(level)
    z = BWTC.compressFile(data, None, level)
    assert z == O.bwtc_compress(data, level)
    assert BWTC.decompressFile(z) == data


def _seam_data():
    """Level-1 blocks: uniform, uniform, ASCII, ASCII, ASCII, uniform, short uniform.  In batches of two blocks, the
    ASCII batch reuses the two slots whose masks the first batch set, and the later batches flag other slots."""
    bs = 99981
    return (_uniform(2 * bs, 81) + T.ascii_random(3 * bs, 82) + _uniform(bs, 83) + _uniform(bs // 2, 84))


_SEAM_SCRIPT = r"""
import sys, hashlib
sys.path.insert(0, %(root)r)
from compressjs_b200 import BWTC, Bzip2
from tests import test_gpu_narrow_symbols as M
data = M._seam_data()
z = Bzip2.compressFile(data, None, 1)
assert Bzip2.decompressFile(z) == data
w = BWTC.compressFile(data, None, 1)
assert BWTC.decompressFile(w) == data
print("RESULT", hashlib.sha256(z).hexdigest(), hashlib.sha256(w).hexdigest())
"""


def test_masks_across_batches_vs_oracle():
    """Slots flagged by one batch are cleared before the next batch reuses them (B2_BWT_BATCH=2)."""
    env = dict(os.environ, B2_BWT_BATCH="2")
    r = subprocess.run([sys.executable, "-c", _SEAM_SCRIPT % {"root": ROOT}], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT")][-1].split()
    data = _seam_data()
    assert line[1] == hashlib.sha256(O.bzip2_compress(data, 1)).hexdigest()
    assert line[2] == hashlib.sha256(O.bwtc_compress(data, 1)).hexdigest()
