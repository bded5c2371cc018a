"""The encoder's move-to-front + zero-run coder and Huffman table search against the oracle at every chunk, window,
group, tile and table-count seam.

Every case of tests/mtfhuff_cases.py (blocks designed by their BWT column, with what they reach asserted on the CPU)
runs through Bzip2.compressFile at its levels in a child process, once with the default BWT batch and once with
B2_BWT_BATCH=2 (designed blocks then share batches, slots and mask clears with their neighbours).  For every case the
test checks:
- the stream equals the oracle's byte for byte;
- the per-block trace (n, pidx, m, alpha, ngroups, nsel, crc, bit_len) equals the oracle's (the first differing block
  and field is reported);
- decompressFile gives the input back, and libbz2 does when the stream is in its language;
- BWTC, which runs the same MTF kernels on the sentinel BWT's column, equals the oracle's BWTC stream.
The whole corpus is also compressed as one file and compared by SHA-256.  That is a parity check only: the encoder
cuts the joined inputs into new blocks, so the designed columns do not survive in it; designed blocks share batches,
slots and mask clears in the per-case runs with B2_BWT_BATCH=2.  The corpus is built once, in the parent, and handed
to the children as a file of raw inputs.
"""
import bz2
import hashlib
import os
import pickle
import subprocess
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import oracle as O
from tests import bz2synth as S
from tests import mtfhuff_cases as MC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("n", "pidx", "m", "alpha", "ngroups", "nsel", "crc", "bit_len")
CONFIGS = {"default": {}, "batch2": {"B2_BWT_BATCH": "2"}}

_CHILD = r"""
import hashlib, pickle, sys
sys.path.insert(0, %(root)r)
import numpy as np
from compressjs_b200 import BWTC, Bzip2, _native
raws = pickle.load(open(sys.argv[1], "rb"))
out = {}
for j, (name, level) in enumerate(raws["jobs"]):
    key = "j%%d_" %% j
    try:
        data = raws[name]
        z = Bzip2.compressFile(data, None, level)
        out[key + "trace"] = np.array([[getattr(t, f) for f in %(fields)r] for t in _native.last_trace()], dtype=np.int64).reshape(-1, %(nf)d)
        out[key + "z"] = np.frombuffer(z, dtype=np.uint8)
        out[key + "back"] = np.array(Bzip2.decompressFile(z) == data)
        w = BWTC.compressFile(data, None, level)
        out[key + "bwtc"] = np.frombuffer(w, dtype=np.uint8)
    except Exception as ex:   # reported by the parent with the job it belongs to
        out[key + "err"] = np.array(repr(ex))
try:
    whole = b"".join(raws[name] for name in raws["names"])
    z = Bzip2.compressFile(whole, None, 9)
    out["whole_sha"] = np.array(hashlib.sha256(z).hexdigest())
    out["whole_back"] = np.array(Bzip2.decompressFile(z) == whole)
except Exception as ex:
    out["whole_err"] = np.array(repr(ex))
np.savez(sys.argv[2], **out)
"""


def _jobs():
    return [(c.name, lv) for c in MC.cases() for lv in c.levels]


@pytest.fixture(scope="module")
def gpu_runs(tmp_path_factory):
    """One child process per configuration, started in the background while the oracle runs."""
    tmp = tmp_path_factory.mktemp("mtfhuff_seams")
    results = {}
    names = [c.name for c in MC.cases()]
    raws = {name: MC.info(name).raw for name in names}
    raws.update(jobs=_jobs(), names=names)
    corpus = tmp / "corpus.pkl"
    with open(corpus, "wb") as f:
        pickle.dump(raws, f)

    def run_all():
        for name, env in CONFIGS.items():
            out = tmp / ("%s.npz" % name)
            e = {k: v for k, v in os.environ.items() if k != "B2_BWT_BATCH"}
            e.update(env)
            r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT, "fields": FIELDS, "nf": len(FIELDS)},
                                str(corpus), str(out)], env=e, capture_output=True, text=True, timeout=3000)
            results[name] = (r, out)

    th = threading.Thread(target=run_all)
    th.start()
    return th, results


@pytest.fixture(scope="module")
def oracle():
    """(case, level) -> (stream, trace rows, BWTC stream); and the SHA-256 of the whole corpus at level 9."""
    def one(k):
        data = MC.info(k[0]).raw
        z, tr = O.bzip2_compress(data, k[1], trace=True)
        rows = np.array([[getattr(t, f) for f in FIELDS] for t in tr], dtype=np.int64).reshape(-1, len(FIELDS))
        return k, (z, rows, O.bwtc_compress(data, k[1]))

    with ThreadPoolExecutor(max_workers=4) as ex:
        res = dict(ex.map(one, _jobs()))
    whole = b"".join(MC.info(c.name).raw for c in MC.cases())
    return res, hashlib.sha256(O.bzip2_compress(whole, 9, threads=min(os.cpu_count() or 1, 16))).hexdigest()


def _libbz2(name):
    """libbz2 rejects a block that ends on a 4th byte without its count byte; every other stream is in its language."""
    return not any(S.rle1_classes(b.T)[1] for b in MC.info(name).built)


def _trace_diff(got, exp):
    if got.shape == exp.shape and np.array_equal(got, exp):
        return None
    for k in range(min(len(got), len(exp))):
        for f, name in enumerate(FIELDS):
            if got[k, f] != exp[k, f]:
                return "block %d: %s %d, oracle %d" % (k, name, got[k, f], exp[k, f])
    return "%d blocks, oracle %d" % (len(got), len(exp))


@pytest.mark.parametrize("config", list(CONFIGS))
def test_mtf_and_huffman_seams_match_oracle(config, gpu_runs, oracle):
    th, results = gpu_runs
    th.join()
    r, out = results[config]
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(out)
    res, _ = oracle
    failures = []
    for j, (name, lv) in enumerate(_jobs()):
        key, tag = "j%d_" % j, "%s level %d" % (name, lv)
        if key + "err" in got:
            failures.append("%s: %s" % (tag, got[key + "err"]))
            continue
        stream, rows, bwtc = res[(name, lv)]
        d = _trace_diff(got[key + "trace"], rows)
        if d:
            failures.append("%s: trace differs: %s" % (tag, d))
        z = got[key + "z"].tobytes()
        if z != stream:
            failures.append("%s: stream differs from the oracle's (%d vs %d bytes)" % (tag, len(z), len(stream)))
        if not bool(got[key + "back"]):
            failures.append("%s: decompressFile does not give the input back" % tag)
        elif _libbz2(name) and bz2.decompress(z) != MC.info(name).raw:
            failures.append("%s: libbz2 does not decode the stream" % tag)
        if got[key + "bwtc"].tobytes() != bwtc:
            failures.append("%s: BWTC stream differs from the oracle's" % tag)
    assert not failures, "%s:\n" % config + "\n".join(failures)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_whole_corpus_as_one_file(config, gpu_runs, oracle):
    th, results = gpu_runs
    th.join()
    r, out = results[config]
    assert r.returncode == 0, r.stderr[-4000:]
    got = np.load(out)
    assert "whole_err" not in got, str(got["whole_err"])
    assert str(got["whole_sha"]) == oracle[1]
    assert bool(got["whole_back"])
