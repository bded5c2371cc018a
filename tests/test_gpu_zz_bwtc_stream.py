"""BWTC streams of unknown size, the batched BWTC decode, and the command line end to end on the GPU.

Sorts last, like test_gpu_zz_bwtc.py.  The oracle is oracle/bwtc_oracle.c for sized streams, tests/bwtc_unsized.py for
streams of unknown size, and, for the command line, the library's own Bzip2 / BWTC calls."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import bwtc_unsized as U
from tests import util as T

pytestmark = pytest.mark.gpu


def _unsized(data, level):
    from compressjs_b200 import bwtc
    return bwtc._compress_unsized(data, level)


@pytest.mark.parametrize("level", [1, 5, 6, 9])
@pytest.mark.parametrize("name", ["sample0", "sample1", "sample2", "sample3"])
def test_unsized_samples(name, level):
    from compressjs_b200 import BWTC
    d = T.fixture(name + ".ref")
    z = _unsized(d, level)
    assert z == U.unsized(d, level)
    assert BWTC.decompressFile(z) == d


@pytest.mark.parametrize("level", [1, 5, 6, 9])
def test_unsized_edges(level):
    from compressjs_b200 import BWTC
    for n in (0, 1, level * 100000 - 1, level * 100000, level * 100000 + 1):
        d = T.texty(n, 200 + n)
        z = _unsized(d, level)
        assert z == U.unsized(d, level), n
        assert BWTC.decompressFile(z) == d, n


def test_unsized_c_abi():
    from compressjs_b200 import _native
    L = _native.lib()
    d = np.frombuffer(T.runs(250000, 7), dtype=np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    assert L.b2_bwtc_compress_unsized(d.ctypes.data, d.size, 12, C.byref(out), C.byref(n)) == 0   # 12 means 9
    z = C.string_at(out, n.value)
    L.b2_free(out)
    assert z == U.unsized(d.tobytes(), 9)


# ---- batches, in a child process: the library reads $B2_BWTC_DEC_BATCH per call, the tests share one library ----
CHILD = r"""
import json, sys
sys.path.insert(0, %r)
from tests import util as T
from tests import bwtc_unsized as U
from oracle import oracle as O
from compressjs_b200 import BWTC, bwtc
def outcome(z):
    try:
        return ["ok", len(BWTC.decompressFile(z))]
    except Exception as e:
        return ["err", type(e).__name__, str(e)]
data = T.runs(260000, 71) + T.texty(310000, 72) + b"q" * 120000 + T.ascii_random(80000, 73) + bytes(range(256)) * 100
res = {}
for level in (1,):              # 795600 bytes: 7 full blocks and a short one
    for sized in (True, False):
        z = BWTC.compressFile(data, None, level) if sized else bwtc._compress_unsized(data, level)
        assert z == (O.bwtc_compress(data, level) if sized else U.unsized(data, level))
        assert BWTC.decompressFile(z) == data, (level, sized)
        cases = {"flip%%d" %% i: z[:p] + bytes([z[p] ^ 0x5A]) + z[p + 1:] for i, p in enumerate((len(z) * 7 // 10, len(z) * 9 // 10))}
        cases.update({"cut%%d" %% i: z[:k] for i, k in enumerate((len(z) // 2, len(z) - 8))})
        res["%%d-%%d" %% (level, sized)] = {k: outcome(v) for k, v in cases.items()}
print(json.dumps(res))
""" % T.ROOT


def _child(batch):
    env = dict(os.environ)
    env.pop("B2_BWTC_DEC_BATCH", None)
    if batch:
        env["B2_BWTC_DEC_BATCH"] = str(batch)
    r = subprocess.run([sys.executable, "-c", CHILD], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_batch_seams_and_errors():
    """Sized and unknown-size streams of 8 blocks decode to the same bytes with batches of 1, 2, 3 blocks and the
    default; a byte flipped in a later batch and cut streams give the same result (the same error) in every case.
    A cut stream of unknown size is an error; a cut stream with a size may decode to garbage of the right size, as in
    the reference, which has no check there either."""
    ref = _child(None)
    for b in (1, 2, 3):
        assert _child(b) == ref, b
    for k in ("cut0", "cut1"):
        v = ref["1-0"][k]
        assert v[0] == "err" and v[1] == "RuntimeError" and "code -5" in v[2], (k, v)
    assert any(v[0] == "err" for cases in ref.values() for k, v in cases.items() if k.startswith("flip"))


def test_unsized_stream_of_many_blocks():
    """An unknown-size stream of several MB decodes: sizing the L columns by the compressed size (n / 2 + 2 blocks of
    1 MiB each) would have asked for terabytes."""
    from compressjs_b200 import BWTC
    d = T.ascii_random(5 << 20, 81)
    z = _unsized(d, 1)
    assert len(z) > (4 << 20)
    assert BWTC.decompressFile(z) == d


def test_sized_stream_longer_than_one_batch():
    """More blocks than one default batch (two per SM: 264 on an H100 SXM)."""
    import torch
    from compressjs_b200 import BWTC
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    d = T.ascii_random((2 * sms + 3) * 100000 + 4321, 91)
    z = BWTC.compressFile(d, None, 1)
    assert BWTC.decompressFile(z) == d


def test_size_field_checks():
    """A size field one below the blocks fails when the last block passes it, one above when the stream ends; both with
    the reference's size error (lib/Util.js:69-71)."""
    from compressjs_b200 import BWTC
    d = T.texty(250000, 5)
    z = BWTC.compressFile(d, None, 1)
    # size + 1 = 250001 = 15 * 128^2 + 33 * 128 + 17; the last group's byte is not read by the range decoder
    assert z[4:7] == bytes([15, 33, 0x80 | 17])
    for last in (0x80 | 16, 0x80 | 18):
        with pytest.raises(RuntimeError, match="outputsize does not match decoded input"):
            BWTC.decompressFile(z[:6] + bytes([last]) + z[7:])


# ---- the command line, end to end ----
def _cli(*args, stdin=None):
    return subprocess.run([sys.executable, "-m", "compressjs_b200"] + [str(a) for a in args], input=stdin, capture_output=True,
                          cwd=T.ROOT, timeout=600)


def test_cli_bzip2(tmp_path):
    from compressjs_b200 import Bzip2
    d = T.texty(700000, 31)
    f = tmp_path / "in"
    f.write_bytes(d)
    r = _cli("-z", "-t", "bzip2", "-9", f)
    assert r.returncode == 0, r.stderr
    assert r.stdout == Bzip2.compressFile(d, None, 9)
    r = _cli("-t", "BZIP", f, tmp_path / "z7")               # no -d: compress; no level: 7
    assert r.returncode == 0, r.stderr
    z7 = (tmp_path / "z7").read_bytes()
    assert z7[:4] == b"BZh7" and z7 == Bzip2.compressFile(d, None, 7)
    r = _cli("-d", "-t", "bzip2", stdin=z7)
    assert r.returncode == 0 and r.stdout == d
    r = _cli("-d", "-t", "bzip2", tmp_path / "z7", tmp_path / "back")
    assert r.returncode == 0 and (tmp_path / "back").read_bytes() == d


def test_cli_bwtc_size_rule(tmp_path):
    """From a regular file the header has the size, from a pipe or an empty file it says "unknown"; -d reads both."""
    d = T.texty(450000, 32)
    f = tmp_path / "in"
    f.write_bytes(d)
    sized, unsized = O.bwtc_compress(d, 3), U.unsized(d, 3)
    r = _cli("-z", "-t", "bwtc", "-3", f)
    assert r.returncode == 0 and r.stdout == sized, r.stderr
    with open(f, "rb") as h:                                   # stdin redirected from the file: still a regular file
        r = subprocess.run([sys.executable, "-m", "compressjs_b200", "-t", "bwtc", "-3"], stdin=h, capture_output=True, cwd=T.ROOT, timeout=600)
    assert r.returncode == 0 and r.stdout == sized, r.stderr
    r = _cli("-z", "-t", "bwtc", "-3", stdin=d)                # a pipe
    assert r.returncode == 0 and r.stdout == unsized, r.stderr
    e = tmp_path / "empty"
    e.write_bytes(b"")
    r = _cli("-t", "bwtc", e, tmp_path / "e.bwtc")
    assert r.returncode == 0 and (tmp_path / "e.bwtc").read_bytes() == U.unsized(b"", 7)
    for z in (sized, unsized):
        zf = tmp_path / "z"
        zf.write_bytes(z)
        r = _cli("-d", "-t", "bwtc", zf, tmp_path / "out")
        assert r.returncode == 0 and (tmp_path / "out").read_bytes() == d, r.stderr
        r = _cli("-d", "-t", "bwtc", stdin=z)
        assert r.returncode == 0 and r.stdout == d, r.stderr
    r = _cli("-d", "-t", "bwtc", tmp_path / "e.bwtc")
    assert r.returncode == 0 and r.stdout == b""


def test_cli_block():
    for f, pos, blk in [("sample2", 544888, "sample2.544888"), ("sample4", 32, "sample4.32"),
                        ("sample4", 1596228, "sample4.1596228"), ("sample4", 2342106, "sample4.2342106")]:
        r = _cli("-d", "-t", "bzip2", "-b", pos, stdin=T.fixture(f + ".bz2"))
        assert r.returncode == 0 and r.stdout == T.fixture(blk), (f, pos, r.stderr)


def test_cli_decode_error_keeps_the_flushed_prefix(tmp_path):
    """bin/compressjs:103-115 flushes its 4096-byte buffer only when the next byte arrives: on an error the output has
    the decoded bytes cut down to a multiple of 4096, then the message and status 1."""
    from compressjs_b200 import Bzip2

    class Sink:
        def __init__(self):
            self.b = bytearray()

        def writeByte(self, x):
            self.b.append(x)

    d = T.texty(430000, 33)
    z = Bzip2.compressFile(d, None, 1)
    rows = []
    Bzip2.table(z, lambda p, s: rows.append((p, s)))
    assert len(rows) >= 4
    for blk, off in ((2, 200), (3, 40), (0, 300)):
        p = rows[blk][0] // 8 + off
        bad = z[:p] + bytes([z[p] ^ 0x21]) + z[p + 1:]
        s = Sink()
        with pytest.raises(Exception) as ei:
            Bzip2.decompressFile(bad, s)
        k = len(s.b)
        r = _cli("-d", "-t", "bzip2", stdin=bad)
        assert r.returncode == 1
        assert r.stdout == bytes(s.b[:4096 * ((k - 1) // 4096)] if k else b""), (blk, k, len(r.stdout))
        assert r.stderr.decode().strip() == str(ei.value)
