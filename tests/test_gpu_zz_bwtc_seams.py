"""The BWTC container's models, range coder and output windows against the oracle at every rescale, escape, carry and
batch seam.

Every case of tests/bwtc_cases.py (inputs designed from the model's symbols, with what they reach asserted on the CPU by
tests/test_bwtc_cases.py) runs at its levels in a child process per B2_BWT_BATCH (the default, 1, 2 and 3 blocks per
batch: the designed seams, slots and mask clears then fall on batch seams) through b2_bwtc_compress,
b2_bwtc_compress_unsized and b2_bwtc_compress_stream with an odd read pattern.  Each stream must equal the oracle's (the
unsized one tests/bwtc_unsized.py's) byte for byte; a mismatch names the first block whose bytes differ, from the
oracle's trace.  Every configuration must give the oracle's bytes, so the streams are decoded once, in the default
configuration: the sized stream through b2_bwtc_decompress and the unsized one through b2_bwtc_decompress_stream, with a
64 KiB decode window and one block per decode batch, so that bytes pending across a block's end also straddle the
decode windows.  The decoder is one serial thread (under 0.6 MB/s, slower at levels 1..5), so only the cases of up to
400 000 bytes are decoded: among them every case built for the coder's pending bytes, header and trailer.
"""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from tests import bwtc_cases as BC
from tests import bwtc_unsized as UNS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = {"default": None, "batch1": "1", "batch2": "2", "batch3": "3"}

_CHILD = r"""
import ctypes as C, pickle, sys
sys.path.insert(0, %(root)r)
import numpy as np
from compressjs_b200 import _native as N
from tests.test_gpu_zz_bwtc_callbacks import stream_compress, stream_decompress
L = N.lib()
jobs = pickle.load(open(sys.argv[1], "rb"))

def call(f, data, *args):
    a = np.frombuffer(data, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = f(a.ctypes.data if a.size else None, a.size, *args, C.byref(out), C.byref(n))
    if rc:
        return "rc %%d: %%s" %% (rc, N.last_error())
    z = C.string_at(out, n.value)
    L.b2_free(out)
    return z

res = {}
for key, (data, level) in jobs.items():
    r = {}
    r["sized"] = call(L.b2_bwtc_compress, data, level)
    r["unsized"] = call(L.b2_bwtc_compress_unsized, data, level)
    rc, z, err, _ = stream_compress(data, level, len(data), "odd" if len(data) < (4 << 20) else "all")
    r["stream"] = z if rc == 0 else "rc %%d: %%s" %% (rc, err)
    back = {}
    if len(data) <= 400000 and sys.argv[3] == "default":
        if isinstance(r["sized"], bytes):
            d = call(L.b2_bwtc_decompress, r["sized"])
            back["sized_buf"] = d == data if isinstance(d, bytes) else d
        if isinstance(r["unsized"], bytes):
            rc, d, err, _ = stream_decompress(r["unsized"], "odd")
            back["unsized_stream"] = d == data if rc == 0 else "rc %%d: %%s" %% (rc, err)
    r["back"] = back
    res[key] = r
pickle.dump(res, open(sys.argv[2], "wb"))
"""


def _jobs():
    return [(c.name, lv) for c in BC.cases() for lv in c.levels]


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """The raw inputs of every (case, level), written once for the child processes."""
    path = tmp_path_factory.mktemp("bwtc_seams") / "corpus.pkl"
    with open(path, "wb") as f:
        pickle.dump({"%s@%d" % (n, lv): (BC.raw(n), lv) for n, lv in _jobs()}, f)
    return path


def _run(config, corpus):
    out = corpus.parent / ("%s.pkl" % config)
    e = {k: v for k, v in os.environ.items() if k not in ("B2_BWT_BATCH", "B2_DEC_WINDOW", "B2_BWTC_DEC_BATCH")}
    e.update(B2_DEC_WINDOW="65536", B2_BWTC_DEC_BATCH="1")
    if CONFIGS[config]:
        e["B2_BWT_BATCH"] = CONFIGS[config]
    r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT}, str(corpus), str(out), config], env=e,
                       capture_output=True, text=True, timeout=3000, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    with open(out, "rb") as f:
        return pickle.load(f)


def _first_diff(got, exp, blocks):
    """Where two streams part: the first block (by the oracle's bytes out at each block's end) holding the byte."""
    i = next((k for k in range(min(len(got), len(exp))) if got[k] != exp[k]), min(len(got), len(exp)))
    blk = next((k for k, b in enumerate(blocks) if i < b.bytes_out), len(blocks))
    where = "block %d" % blk if blk < len(blocks) else "the trailer"
    return "%d vs %d bytes, first difference at byte %d (%s)" % (len(got), len(exp), i, where)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_bwtc_seams_match_oracle(config, corpus):
    got = _run(config, corpus)
    failures = []
    for name, lv in _jobs():
        key = "%s@%d" % (name, lv)
        ci = BC.info(name, lv)
        g = got[key]
        exp = {"sized": ci.z, "stream": ci.z, "unsized": UNS.unsized(ci.raw, lv)}
        for which, z in exp.items():
            if not isinstance(g[which], bytes):
                failures.append("%s %s: %s" % (key, which, g[which]))
            elif g[which] != z:
                failures.append("%s %s: %s" % (key, which, _first_diff(g[which], z, ci.blocks)))
        for which, ok in g["back"].items():
            if ok is not True:
                failures.append("%s decode of the %s stream: %s" % (key, which, ok))
    assert not failures, "%s:\n" % config + "\n".join(failures)
