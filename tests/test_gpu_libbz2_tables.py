"""The libbz2 flavor's Huffman table search (csrc/huff.cu k_huffman_libbz2) against libbz2 and the libbz2 model at
every 17-bit rescale, partition, tie and tile seam.

Every case of tests/libbz2_table_cases.py (designed blocks whose corners the CPU test asserts in the model) and every
case of tests/mtfhuff_cases.py runs through Bzip2.compressFile(..., flavor="libbz2") at its levels in a child process,
once with the default BWT batch and once with B2_BWT_BATCH=2.  For every case the test checks:
- the stream equals bz2.compress (or, without libbz2 1.0.3+, the size and SHA-256 of tests/golden/libbz2.json); on a
  difference the block headers of both streams are parsed and the first differing selector or code length is named;
- the per-block trace (n, pidx, m, alpha, ngroups, nsel, crc, bit_len) equals the reference trace (first differing
  block and field): the oracle's blocks with the bit lengths of libbz2's stream, all in C and numpy.  The CPU test
  (tests/test_libbz2_table_cases.py) holds the model's trace to the same rows;
- decompressFile and bz2.decompress give the input back.
The designed corpus is also compressed as one level-9 file, and a few cases once more through the device entry point.
The corpus is built once, in the parent, and handed to the children as a file of raw inputs."""
import bz2
import hashlib
import json
import os
import pickle
import subprocess
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests import libbz2_model as M
from tests import libbz2_table_cases as TC
from tests import mtfhuff_cases as MC
from tests.test_libbz2_model import GOLDEN, _libbz2_ok

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = M.TRACE_FIELDS
CONFIGS = {"default": {}, "batch2": {"B2_BWT_BATCH": "2"}}
LIVE = _libbz2_ok()
DEV_CASES = ("rescale_written", "exhausted_alpha2", "nsel_257", "l9_six_kinds")

_CHILD = r"""
import ctypes as C, pickle, sys
sys.path.insert(0, %(root)r)
import numpy as np
import torch
from compressjs_b200 import Bzip2, _native
raws = pickle.load(open(sys.argv[1], "rb"))
out = {}
for j, (key, level) in enumerate(raws["jobs"]):
    k = "j%%d_" %% j
    try:
        data = raws[key]
        z = Bzip2.compressFile(data, None, level, flavor="libbz2")
        out[k + "trace"] = np.array([[getattr(t, f) for f in %(fields)r] for t in _native.last_trace()], dtype=np.int64).reshape(-1, %(nf)d)
        out[k + "z"] = np.frombuffer(z, dtype=np.uint8)
        out[k + "back"] = np.array(Bzip2.decompressFile(z) == data)
    except Exception as ex:   # reported by the parent with the job it belongs to
        out[k + "err"] = np.array(repr(ex))
try:
    whole = b"".join(raws[key] for key in raws["whole"])
    out["whole"] = np.frombuffer(Bzip2.compressFile(whole, None, 9, flavor="libbz2"), dtype=np.uint8)
except Exception as ex:
    out["whole_err"] = np.array(repr(ex))
L = _native.lib()
for key, level in raws["dev"]:
    data = raws[key]
    a = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = L.b2_bzip2_bound(len(data))
    o = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    n = C.c_size_t()
    rc = L.b2_bzip2_compress_dev_flavor(a.data_ptr(), len(data), level, o.data_ptr(), cap, C.byref(n), 1)
    torch.cuda.synchronize()
    out["dev_" + key] = o[:n.value].cpu().numpy() if rc == 0 else np.array(_native.last_error())
np.savez(sys.argv[2], **out)
"""


def _jobs():
    """(key, name, level): table2_<case> and mtfhuff_<case> at each of their levels."""
    return ([("table2_" + c.name, c.name, lv) for c in TC.cases() for lv in c.levels] +
            [("mtfhuff_" + c.name, c.name, lv) for c in MC.cases() for lv in c.levels])


def _raw(key):
    name = key.split("_", 1)[1]
    return TC.raw(name) if key.startswith("table2_") else MC.info(name).raw


@pytest.fixture(scope="module")
def gpu_runs(tmp_path_factory):
    """One child process per configuration, started in the background while the references run."""
    tmp = tmp_path_factory.mktemp("libbz2_tables")
    results = {}
    keys = sorted({k for k, _, _ in _jobs()})
    raws = {k: _raw(k) for k in keys}
    raws.update(jobs=[(k, lv) for k, _, lv in _jobs()], whole=["table2_" + c.name for c in TC.cases()],
                dev=[("table2_" + n, TC.case(n).levels[0]) for n in DEV_CASES])
    corpus = tmp / "corpus.pkl"
    with open(corpus, "wb") as f:
        pickle.dump(raws, f)

    def run_all():
        for name, env in CONFIGS.items():
            out = tmp / ("%s.npz" % name)
            e = {k: v for k, v in os.environ.items() if k != "B2_BWT_BATCH"}
            e.update(env)
            r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT, "fields": FIELDS, "nf": len(FIELDS)},
                                str(corpus), str(out)], env=e, capture_output=True, text=True, timeout=1200)
            results[name] = (r, out)

    th = threading.Thread(target=run_all)
    th.start()
    return th, results, raws


def _reference(job):
    """(key, level) -> (the libbz2 stream or None, the reference trace rows or None).  All in C (the oracle, libbz2) and
    numpy: the CPU test holds the model's trace to the same rows."""
    key, lv = job
    data = _raw(key)
    if not LIVE:
        return job, (None, None)
    ref = bz2.compress(data, lv)
    return job, (ref, TC.reference_trace(data, lv, ref))


@pytest.fixture(scope="module")
def references(gpu_runs):
    gold = json.load(open(GOLDEN))
    with ThreadPoolExecutor(max_workers=4) as ex:
        res = dict(ex.map(_reference, [(k, lv) for k, _, lv in _jobs()]))
    return res, gold


class _Reader:
    def __init__(self, z, bit):
        self.z, self.p = z, bit

    def bits(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | ((self.z[self.p >> 3] >> (7 - (self.p & 7))) & 1)
            self.p += 1
        return v


def _headers(z):
    """Per block (selectors, code lengths) parsed from the block headers of a bzip2 stream, each read from its magic."""
    out = []
    for start in TC.block_edges(z)[:-1]:
        r = _Reader(z, start + 48)
        r.bits(32 + 1 + 24)
        used = [i for i in range(16) if r.bits(1)]
        A = sum(r.bits(1) for _ in used for _ in range(16)) + 2
        ng, nsel = r.bits(3), r.bits(15)
        mt, sel = list(range(ng)), []
        for _ in range(nsel):
            j = 0
            while r.bits(1):
                j += 1
            mt.insert(0, mt.pop(j))
            sel.append(mt[0])
        lens = []
        for _ in range(ng):
            cur, ln = r.bits(5), []
            for _ in range(A):
                while r.bits(1):
                    cur += -1 if r.bits(1) else 1
                ln.append(cur)
            lens.append(ln)
        out.append((sel, lens))
    return out


def _stream_diff(got, exp):
    """The first differing block and its first differing selector or table symbol length."""
    try:
        hg, he = _headers(got), _headers(exp)
    except (IndexError, ValueError) as ex:
        return "the GPU stream's block headers do not parse (%r)" % ex
    for b, ((sg, lg), (se, le)) in enumerate(zip(hg, he)):
        if len(sg) != len(se) or len(lg) != len(le):
            return "block %d: %d selectors / %d tables, libbz2 %d / %d" % (b, len(sg), len(lg), len(se), len(le))
        for i, (x, y) in enumerate(zip(sg, se)):
            if x != y:
                return "block %d: selector %d is %d, libbz2 %d" % (b, i, x, y)
        for t, (x, y) in enumerate(zip(lg, le)):
            for v, (p, q) in enumerate(zip(x, y)):
                if p != q:
                    return "block %d: table %d symbol %d has length %d, libbz2 %d" % (b, t, v, p, q)
    return "block headers equal over %d blocks (libbz2 %d): the difference is in the symbols" % (len(hg), len(he))


def _trace_diff(got, exp):
    if got.shape == exp.shape and np.array_equal(got, exp):
        return None
    for k in range(min(len(got), len(exp))):
        for f, name in enumerate(FIELDS):
            if got[k, f] != exp[k, f]:
                return "block %d: %s %d, reference %d" % (k, name, got[k, f], exp[k, f])
    return "%d blocks, reference %d" % (len(got), len(exp))


def _check_stream(tag, key, lv, z, ref, gold, failures):
    if ref is not None:
        if z != ref:
            failures.append("%s: stream differs from libbz2's (%d vs %d bytes): %s" % (tag, len(z), len(ref), _stream_diff(z, ref)))
    else:
        g = gold.get("%s_-%d" % (key, lv))
        if g is None or (len(z), hashlib.sha256(z).hexdigest()) != (g["size"], g["sha256"]):
            failures.append("%s: stream differs from the golden size and SHA-256" % tag)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_table_search_matches_libbz2(config, gpu_runs, references):
    th, results, raws = gpu_runs
    th.join()
    r, out = results[config]
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(out)
    res, gold = references
    failures = []
    for j, (key, name, lv) in enumerate(_jobs()):
        k, tag = "j%d_" % j, "%s level %d" % (key, lv)
        if k + "err" in got:
            failures.append("%s: %s" % (tag, got[k + "err"]))
            continue
        ref, rows = res[(key, lv)]
        d = _trace_diff(got[k + "trace"], rows) if rows is not None else None
        if d:
            failures.append("%s: trace differs: %s" % (tag, d))
        z = got[k + "z"].tobytes()
        _check_stream(tag, key, lv, z, ref, gold, failures)
        if not bool(got[k + "back"]):
            failures.append("%s: decompressFile does not give the input back" % tag)
        elif bz2.decompress(z) != raws[key]:
            failures.append("%s: libbz2 does not give the input back" % tag)
    if "whole_err" in got:
        failures.append("whole corpus: %s" % got["whole_err"])
    else:
        _check_stream("whole corpus level 9", "table2_whole", 9, got["whole"].tobytes(),
                      bz2.compress(TC.whole(), 9) if LIVE else None, gold, failures)
    for key, lv in raws["dev"]:
        dz = got["dev_" + key]
        if dz.dtype.kind != "u":
            failures.append("%s: device entry point: %s" % (key, dz))
        else:
            _check_stream("%s level %d (device entry point)" % (key, lv), key, lv, dz.tobytes(), res[(key, lv)][0], gold, failures)
    assert not failures, "%s:\n" % config + "\n".join(failures)
