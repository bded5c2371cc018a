"""Every forward-BWT path and fallback against the oracle, one path at a time.

The corpus of tests/bwt_cases.py runs through b2_bwt_cyclic_batch (b2_bwt_cyclic for single blocks) under each
configuration of bwt_cases.CONFIGS: the default, every batch starting on the MSD path, the 4-byte LSD path, the wide
mode, and 1 and 3 blocks per batch for the mode hand-over.  The library reads these settings once, when its context
is created, so every configuration runs in a child process.  For every case the test checks:
- U and pidx equal the oracle's bwt_cyclic, block by block;
- the path counters of b2_stats equal the CPU model's prediction (finish and fallback bits of every batch);
- for a few cases, Bzip2.compressFile at level 9 equals the oracle's stream byte for byte (the encoder also hands the
  BWT's byte histograms to the MTF symbol map).
"""
import os
import subprocess
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import oracle as O
from tests import bwt_cases as BC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r"""
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from compressjs_b200 import Bzip2, _native
from tests import bwt_cases as BC
src = np.load(sys.argv[1])
L = _native.lib()
out = {}
for ci in range(int(src["ncases"])):
    lens = src["lens%%d" %% ci].astype(np.int32)
    cat = src["data%%d" %% ci]
    offs = np.zeros(lens.size, dtype=np.uint64)
    offs[1:] = np.cumsum(lens[:-1].astype(np.uint64))
    u = np.zeros(max(cat.size, 1), dtype=np.uint8)
    pidx = np.zeros(lens.size, dtype=np.int32)
    if lens.size == 1 and lens[0] >= 2:
        pidx[0] = L.b2_bwt_cyclic(cat.ctypes.data, u.ctypes.data, int(lens[0]))
        assert pidx[0] >= 0, _native.last_error()
    else:
        rc = L.b2_bwt_cyclic_batch(cat.ctypes.data, u.ctypes.data, offs.ctypes.data, lens.ctypes.data, pidx.ctypes.data, lens.size)
        assert rc == 0, _native.last_error()
    st = _native.stats()
    out["u%%d" %% ci] = u[:cat.size]
    out["pidx%%d" %% ci] = pidx
    out["stats%%d" %% ci] = np.array([st[f] for f in BC.Counters.FIELDS], dtype=np.uint64)
    if src["compress%%d" %% ci]:
        out["z%%d" %% ci] = np.frombuffer(Bzip2.compressFile(cat.tobytes(), None, 9), dtype=np.uint8)
np.savez(sys.argv[2], **out)
"""


@pytest.fixture(scope="module")
def corpus():
    cs = BC.cases()
    with ThreadPoolExecutor(max_workers=min(os.cpu_count() or 1, 16)) as ex:
        blocks = [b for c in cs for b in c.blocks]
        oracle = list(ex.map(O.bwt_cyclic, blocks))
        models = list(ex.map(lambda c: BC.Model(c), cs))
        streams = dict(zip([c.name for c in cs if c.compress],
                           ex.map(lambda c: O.bzip2_compress(b"".join(c.blocks), 9), [c for c in cs if c.compress])))
    it = iter(oracle)
    return cs, [[next(it) for _ in c.blocks] for c in cs], models, streams


def _default_batch():
    import torch
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count  # api.cu: two blocks per SM


@pytest.fixture(scope="module")
def gpu_runs(tmp_path_factory):
    """One child process per configuration, started in the background while the oracle runs."""
    tmp = tmp_path_factory.mktemp("bwt_paths")
    cs = BC.cases()
    src = {"ncases": np.array(len(cs))}
    for ci, c in enumerate(cs):
        src["lens%d" % ci] = np.array([len(b) for b in c.blocks], dtype=np.int64)
        src["data%d" % ci] = np.frombuffer(b"".join(c.blocks), dtype=np.uint8)
        src["compress%d" % ci] = np.array(c.compress)
    np.savez(tmp / "cases.npz", **src)
    results = {}

    def run_all():
        for name, (env, _) in BC.CONFIGS.items():
            out = tmp / ("%s.npz" % name)
            e = {k: v for k, v in os.environ.items() if not k.startswith("B2_BWT_")}
            e.update(env)
            r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT}, str(tmp / "cases.npz"), str(out)],
                               env=e, capture_output=True, text=True, timeout=900)
            results[name] = (r, out)

    th = threading.Thread(target=run_all)
    th.start()
    return th, results


@pytest.mark.parametrize("config", list(BC.CONFIGS))
def test_bwt_path_matches_oracle_and_model(config, gpu_runs, corpus):
    cs, oracle, models, streams = corpus
    th, results = gpu_runs
    th.join()
    r, out = results[config]
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(out)
    env, cfg = BC.CONFIGS[config]
    cfg = dict(cfg)
    cfg.setdefault("batch", _default_batch())
    failures = []
    for ci, (c, exp, m) in enumerate(zip(cs, oracle, models)):
        u, pidx = got["u%d" % ci], got["pidx%d" % ci]
        off = 0
        for bi, (blk, (eu, ep)) in enumerate(zip(c.blocks, exp)):
            gu = u[off:off + len(blk)].tobytes()
            off += len(blk)
            if gu != eu or int(pidx[bi]) != ep:
                diff = next((k for k in range(len(blk)) if gu[k] != eu[k]), None)
                failures.append("%s block %d (n=%d): first differing row %s, pidx %d vs oracle %d"
                                % (c.name, bi, len(blk), diff, int(pidx[bi]), ep))
                break
        want = m.predict(**cfg)
        have = tuple(int(x) for x in got["stats%d" % ci])
        if have != want.as_tuple():
            failures.append("%s: counters %s, model %s (batches: %s)" % (
                c.name, dict(zip(BC.Counters.FIELDS, have)), dict(zip(BC.Counters.FIELDS, want.as_tuple())),
                [b[:4] for b in want.batches]))
        if c.compress and got["z%d" % ci].tobytes() != streams[c.name]:
            failures.append("%s: level-9 stream differs from the oracle's" % c.name)
    assert not failures, "%s:\n" % config + "\n".join(failures)
