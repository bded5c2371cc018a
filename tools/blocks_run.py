"""Random access into a 1 GiB .bz2: Bzip2.decompressBlocks on 1, 132 and all block positions of the table against one
decompressBlock call per position, and decompressFile.

The input is the config-2 workload (uniform ASCII, tests/util.py ascii_random, the generator bench.py uses), compressed
at level 9 on the GPU and tabled once.  Times are host wall clock around calls that end in a device synchronise (every
call of the library is synchronous), after one warm-up call of each kind; the median and the range of REPS repeats are
printed, with the card's name and power limit.

    python tools/blocks_run.py [MiB] [repeats]
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from compressjs_b200 import Bzip2, _native
from tests import util as T

mb = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the figures still stand with the torch device name
        return "%s (nvidia-smi: %r)" % (torch.cuda.get_device_name(0), e)


def timed(fn):
    fn()   # warm-up: pools, pinned buffers, module load
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return {"median_ms": round(1e3 * float(np.median(ts)), 1), "min_ms": round(1e3 * min(ts), 1), "max_ms": round(1e3 * max(ts), 1)}


assert torch.cuda.is_available(), "needs a CUDA device"
print("card:", card())
rc = _native.lib().b2_init(0)
assert rc == 0, _native.last_error()
data = T.ascii_random(mb << 20)
z = Bzip2.compressFile(data, None, 9)
rows = []
Bzip2.table(z, lambda p, s: rows.append((p, s)))
offs = np.concatenate([[0], np.cumsum([s for _, s in rows])])
print("input %d MiB -> %d bytes, %d blocks" % (mb, len(z), len(rows)))
order = list(range(len(rows)))
T.rng(2026).shuffle(order)

res = {}
for k in (1, 132, len(rows)):
    idx = order[:k]
    poss = [rows[i][0] for i in idx]
    got = Bzip2.decompressBlocks(z, poss)
    assert all(g == data[offs[i]:offs[i + 1]] for g, i in zip(got, idx)), "decompressBlocks differs from the table's slices"
    res["decompressBlocks_%d" % k] = timed(lambda: Bzip2.decompressBlocks(z, poss))
    if k <= 132:
        res["decompressBlock_x%d" % k] = timed(lambda: [Bzip2.decompressBlock(z, p) for p in poss])
assert Bzip2.decompressFile(z) == data
res["decompressFile"] = timed(lambda: Bzip2.decompressFile(z))
for name, r in res.items():
    print("%-24s %s" % (name, r))
