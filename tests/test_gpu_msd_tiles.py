"""The forward BWT's MSD scatter (k_msd_scatter) at the seams of its existing 4 KiB text tiles, against the oracle.

Every case is one batch of ASCII blocks that takes the MSD path (B2_BWT_PREFIX8=0 starts every batch there): last
tiles of 1 to 5 bytes, whose rotations read their key cyclically from the block's first bytes; rotation 0 as the first
and as the last record its tile stages (byte 0 the only smallest or the only largest byte of tile 0); blocks shorter
than one tile; and block lengths on, one short of and one past a multiple of the tile (tests/bwt_cases.py has such
lengths too, but not under B2_MSD_CTAS=4).  Each batch runs with the default scatter occupancy and with
B2_MSD_CTAS=4, which the library reads once, so each configuration runs in a child process of its own.  U and pidx
must equal the oracle's bwt_cyclic for every block, and the batch must finish on the MSD path.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import bwt_cases as BC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 4096  # MSD_TILE in bwt_msd.h

_CHILD = r"""
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from compressjs_b200 import _native
src = np.load(sys.argv[1])
L = _native.lib()
out = {}
for ci in range(int(src["ncases"])):
    lens = src["lens%%d" %% ci].astype(np.int32)
    cat = src["data%%d" %% ci]
    offs = np.zeros(lens.size, dtype=np.uint64)
    offs[1:] = np.cumsum(lens[:-1].astype(np.uint64))
    u = np.zeros(cat.size, dtype=np.uint8)
    pidx = np.zeros(lens.size, dtype=np.int32)
    rc = L.b2_bwt_cyclic_batch(cat.ctypes.data, u.ctypes.data, offs.ctypes.data, lens.ctypes.data, pidx.ctypes.data, lens.size)
    assert rc == 0, _native.last_error()
    st = _native.stats()
    out["u%%d" %% ci] = u
    out["pidx%%d" %% ci] = pidx
    out["msd%%d" %% ci] = np.array([st["bwt_msd_done"], st["bwt_msd_fallback_why"]], dtype=np.int64)
np.savez(sys.argv[2], **out)
"""


def _rot0_block(n, seed, smallest):
    """ASCII block whose byte 0 is the only smallest (or only largest) byte of tile 0: its record is staged first (last)."""
    a = BC.ascii_arr(n, seed)
    lo, hi = int(BC.ASCII.min()), int(BC.ASCII.max())
    t0 = a[:TILE]
    t0[(t0 == lo) | (t0 == hi)] = ord("m")
    a[0] = lo if smallest else hi
    return a.tobytes()


def cases():
    big = 200000  # a block of many tiles keeps every batch on the MSD path
    return {
        "tile_multiples": [BC.ascii_arr(n, 10 + i).tobytes()
                           for i, n in enumerate((4 * TILE - 1, 4 * TILE, 4 * TILE + 1, 61 * TILE - 1, 61 * TILE, 61 * TILE + 1))],
        "shorter_than_a_tile": [BC.ascii_arr(n, 20 + i).tobytes() for i, n in enumerate((big, TILE - 1, 100, 9))],
        "cyclic_lookahead": [BC.ascii_arr(n, 30 + i).tobytes() for i, n in enumerate([big] + [7 * TILE + k for k in range(1, 6)])],
        "rot0_first_and_last": [BC.ascii_arr(big, 40).tobytes(), _rot0_block(5 * TILE + 3, 41, True), _rot0_block(5 * TILE + 3, 42, False),
                                _rot0_block(TILE - 5, 43, True), _rot0_block(TILE - 5, 44, False)],
    }


CONFIGS = {"default": {}, "ctas4": {"B2_MSD_CTAS": "4"}}


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("msd_tiles")
    cs = cases()
    src = {"ncases": np.array(len(cs))}
    for ci, blocks in enumerate(cs.values()):
        src["lens%d" % ci] = np.array([len(b) for b in blocks], dtype=np.int64)
        src["data%d" % ci] = np.frombuffer(b"".join(blocks), dtype=np.uint8)
    np.savez(tmp / "cases.npz", **src)
    oracle = {name: [O.bwt_cyclic(b) for b in blocks] for name, blocks in cs.items()}
    return tmp, cs, oracle


@pytest.mark.parametrize("config", list(CONFIGS))
def test_msd_tile_seams_match_oracle(config, corpus):
    tmp, cs, oracle = corpus
    e = {k: v for k, v in os.environ.items() if not k.startswith(("B2_BWT_", "B2_MSD_"))}
    e.update(CONFIGS[config], B2_BWT_PREFIX8="0")
    out = tmp / (config + ".npz")
    r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT}, str(tmp / "cases.npz"), str(out)],
                       env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(out)
    failures = []
    for ci, (name, blocks) in enumerate(cs.items()):
        u, pidx = got["u%d" % ci], got["pidx%d" % ci]
        done, why = (int(x) for x in got["msd%d" % ci])
        if done != 1 or why != 0:
            failures.append("%s: bwt_msd_done %d, bwt_msd_fallback_why %d (the batch left the MSD path)" % (name, done, why))
        off = 0
        for bi, (blk, (eu, ep)) in enumerate(zip(blocks, oracle[name])):
            gu = u[off:off + len(blk)].tobytes()
            off += len(blk)
            if gu != eu or int(pidx[bi]) != ep:
                diff = next((k for k in range(len(blk)) if gu[k] != eu[k]), None)
                failures.append("%s block %d (n=%d): first differing row %s, pidx %d vs oracle %d" % (name, bi, len(blk), diff, int(pidx[bi]), ep))
    assert not failures, "%s:\n" % config + "\n".join(failures)
