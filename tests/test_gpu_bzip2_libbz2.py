"""The libbz2 flavor of the GPU bzip2 encoder against libbz2 (bz2.compress) and tests/golden/libbz2.json, byte for
byte, on the corpus of tests/libbz2_cases.py, the compressjs samples at every level, and at the seams of the
encoder: batches, stream windows, upload chunks, read splits, the device entry point and the command line."""
import bz2
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import libbz2_cases as LC
from tests import libbz2_model as M
from tests import util as T
from tests.test_libbz2_model import GOLDEN, _libbz2_ok

pytestmark = pytest.mark.gpu
ROOT = T.ROOT
LIVE = _libbz2_ok()


def enc(data, level):
    from compressjs_b200 import Bzip2
    return bytes(Bzip2.compressFile(data, None, level, flavor="libbz2"))


def dec(z):
    from compressjs_b200 import Bzip2
    return bytes(Bzip2.decompressFile(z))


def _gold():
    return json.load(open(GOLDEN))


def _check(key, data, level, got):
    g = _gold()[key]
    assert (len(got), hashlib.sha256(got).hexdigest()) == (g["size"], g["sha256"]), key
    if LIVE:
        assert got == bz2.compress(data, level), key


def _trace_matches_model(data, level):
    from compressjs_b200 import _native
    tr = _native.last_trace()
    blocks = M.cut(data, level)
    assert [(t.raw_start, t.raw_len, t.n) for t in tr] == [(s, l, len(b)) for s, l, b in blocks]
    return tr


@pytest.mark.parametrize("name", [c[0] for c in LC.cut_cases()])
def test_cut_corner(name):
    _, data, level, _ = next(c for c in LC.cut_cases() if c[0] == name)
    got = enc(data, level)
    _trace_matches_model(data, level)
    _check("%s_-%d" % (name, level), data, level, got)


@pytest.mark.parametrize("name", [c[0] for c in LC.table_cases()])
def test_table_corner(name):
    _, data, level, _ = next(c for c in LC.table_cases() if c[0] == name)
    got = enc(data, level)
    tr = _trace_matches_model(data, level)
    facts = M.block_facts(data, level)
    assert [(t.m, t.ngroups, t.nsel) for t in tr] == [(f["m"], f["ngroups"], f["nsel"]) for f in facts]
    _check("%s_-%d" % (name, level), data, level, got)


@pytest.mark.parametrize("i", range(6))
def test_samples_every_level(i):
    data = T.fixture("sample%d.ref" % i)
    for level in range(1, 10):
        _check("sample%d_-%d" % (i, level), data, level, enc(data, level))
    if i < 5:
        assert enc(data, (9, 1, 2, 3, 1)[i]) == T.fixture("sample%d.bz2" % i)


@pytest.mark.skipif(not LIVE, reason="bz2 is not linked against libbz2 1.0.3 or later")
def test_basic_inputs():
    for data in (b"", b"a", b"hello world\n", b"abc" * 1000, bytes(range(256))):
        for level in (1, 9):
            assert enc(data, level) == bz2.compress(data, level)


def test_motivating_case():
    """The compressjs flavor's stream ends block 1 on four equal bytes, which libbz2 rejects; the libbz2 flavor's
    stream is libbz2's, and this library decodes both."""
    from compressjs_b200 import Bzip2
    data = LC.motivating()
    cj = bytes(Bzip2.compressFile(data, None, 1))
    lb = enc(data, 1)
    with pytest.raises(OSError):
        bz2.decompress(cj)
    assert bz2.decompress(lb) == data
    if LIVE:
        assert lb == bz2.compress(data, 1)
    assert dec(cj) == data and dec(lb) == data


@pytest.mark.skipif(not LIVE, reason="bz2 is not linked against libbz2 1.0.3 or later")
def test_level9_block_of_runs():
    """One level-9 block of 255-pieces spans 899 985 / 5 * 255 ~ 45.9 MB of raw input."""
    data = b"a" * 46_000_000 + T.ascii_random(100000, 8) + b"b" * 3_000_000
    got = enc(data, 9)
    _trace_matches_model(data, 9)
    assert got == bz2.compress(data, 9)


@pytest.mark.skipif(not LIVE, reason="bz2 is not linked against libbz2 1.0.3 or later")
def test_stream_with_random_read_splits():
    from compressjs_b200 import Bzip2
    data = LC.motivating() + T.runs(400000, 9) + T.texty(300000, 10)
    rng = np.random.default_rng(4)

    class Src:
        pos = 0

        def read(self, buf, off, length):
            k = min(length, int(rng.integers(1, 90000)), len(data) - self.pos)
            buf[off:off + k] = data[self.pos:self.pos + k]
            self.pos += k
            return k

        def readByte(self):
            if self.pos >= len(data):
                return -1
            self.pos += 1
            return data[self.pos - 1]

    class Dst:
        out = bytearray()

        def writeByte(self, b):
            self.out.append(b)

        def write(self, buf, off, length):
            self.out += bytes(buf[off:off + length])
            return length

    d = Dst()
    Bzip2.compressFile(Src(), d, 1, flavor="libbz2")
    assert bytes(d.out) == bz2.compress(data, 1)


@pytest.mark.skipif(not LIVE, reason="bz2 is not linked against libbz2 1.0.3 or later")
def test_device_entry_point():
    import torch
    from compressjs_b200 import _native
    L = _native.lib()
    data = T.texty(700000, 12) + LC.motivating()
    a = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = L.b2_bzip2_bound(len(data))
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    n = C.c_size_t()
    rc = L.b2_bzip2_compress_dev_flavor(a.data_ptr(), len(data), 2, out.data_ptr(), cap, C.byref(n), 1)
    assert rc == 0, _native.last_error()
    torch.cuda.synchronize()
    assert out[:n.value].cpu().numpy().tobytes() == bz2.compress(data, 2)


def test_unknown_flavor_is_rejected_before_reading():
    from compressjs_b200 import Bzip2, _native

    class Src:
        def readByte(self):
            raise AssertionError("read before the flavor was checked")

    class Dst:
        def writeByte(self, b):
            raise AssertionError

    with pytest.raises(ValueError):
        Bzip2.compressFile(Src(), Dst(), 1, flavor="gzip")
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    assert _native.lib().b2_bzip2_compress_flavor(b"abc", 3, 1, C.byref(out), C.byref(n), 2) == -101


_CHILD = r"""
import bz2, sys
sys.path.insert(0, %(root)r)
from tests import libbz2_cases as LC, util as T
from compressjs_b200 import Bzip2
# with a 1 MiB stream window no block may take more raw bytes than that: long runs only where the window is large
runs = T.runs(3_000_000, 21) if sys.argv[1] == "runs" else T.texty(3_000_000, 24)
data = LC.motivating() + runs + T.texty(2_000_000, 22) + LC.run_free(99981, 23) + b"z" * 700
for level in (1, 3):
    got = bytes(Bzip2.compressFile(data, None, level, flavor="libbz2"))
    assert got == bz2.compress(data, level), level
print("ok")
"""


@pytest.mark.skipif(not LIVE, reason="bz2 is not linked against libbz2 1.0.3 or later")
@pytest.mark.parametrize("env", [{"B2_BWT_BATCH": "1"}, {"B2_BWT_BATCH": "3"},
                                 {"B2_STREAM_WINDOW": str(1 << 20), "B2_H2D_CHUNK": "65536"},
                                 {"B2_H2D_CHUNK": "4096"}, {"B2_RLE_SCAN_GROUPS": "1"}])
def test_seams_in_a_child(env):
    e = dict(os.environ)
    e.update(env)
    kind = "text" if "B2_STREAM_WINDOW" in env else "runs"
    r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT}, kind], env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr[-3000:]


@pytest.mark.skipif(not LIVE, reason="bz2 is not linked against libbz2 1.0.3 or later")
def test_config2_256mib():
    data = T.ascii_random(256 << 20, 20260923)
    got = enc(data, 9)
    assert got == bz2.compress(data, 9)
    assert dec(got) == data


def test_cli(tmp_path):
    data = T.texty(500000, 30) + LC.motivating()
    src = tmp_path / "in"
    src.write_bytes(data)
    r = subprocess.run([sys.executable, "-m", "compressjs_b200", "-z", "-t", "bzip2", "--libbz2", "-9", str(src)], cwd=ROOT,
                       capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr
    if LIVE:
        assert r.stdout == bz2.compress(data, 9)
    assert dec(r.stdout) == data
