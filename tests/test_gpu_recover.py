"""Block recovery on the GPU (b2_bzip2_recover, b2_bzip2_recover_stream, Bzip2.recover) against the model of
tests/recover_model.py, over the damage corpus of tests/recover_cases.py: rows, recovered bytes and repaired streams must
be identical, and the repaired streams must decode to the recovered bytes."""
import bz2
import ctypes as C
import os
import subprocess
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from tests import recover_cases as RC
from tests import recover_model as M
from tests import util as T

pytestmark = pytest.mark.gpu

CASES = RC.by_name()
MODEL = {}


def model(name):
    if name not in MODEL:
        MODEL[name] = M.recover(CASES[name].data)
    return MODEL[name]


class Reader:
    """A read() stream that hands out at most `step` bytes per call."""

    def __init__(self, data, step):
        self.data, self.pos, self.step = data, 0, step

    def read(self, buf, off, length):
        k = min(length, self.step, len(self.data) - self.pos)
        buf[off:off + k] = self.data[self.pos:self.pos + k]
        self.pos += k
        return k

    def readByte(self):
        if self.pos >= len(self.data):
            return -1
        self.pos += 1
        return self.data[self.pos - 1]


class Writer:
    def __init__(self, fail_after=None):
        self.buf, self.fail_after = bytearray(), fail_after

    def write(self, buf, off, length):
        if self.fail_after is not None and len(self.buf) + length > self.fail_after:
            raise IOError("disk full")
        self.buf += bytes(buf[off:off + length])

    def writeByte(self, b):
        self.buf.append(b)


def rows_of(blocks):
    return [M.Row(*b) for b in blocks]


def raw_call(data, mode):
    """b2_bzip2_recover itself: (rc, bytes, rows)."""
    from compressjs_b200 import _native
    from compressjs_b200.bzip2 import REC_STATUS
    L = _native.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rows, cnt = C.POINTER(_native.RecoveredBlock)(), C.c_size_t()
    rc = L.b2_bzip2_recover(a.ctypes.data if a.size else None, a.size, mode, C.byref(out), C.byref(n), C.byref(rows), C.byref(cnt))
    assert rc == 0, _native.last_error()
    got = C.string_at(out, n.value) if n.value else b""
    rs = [M.Row(r.bitpos, r.endbit, r.out_off, r.size, r.crc, r.got, REC_STATUS[r.status]) for r in (rows[i] for i in range(cnt.value))]
    L.b2_free(out)
    L.b2_free(rows)
    return got, rs


def check_case(name, streams=True):
    from compressjs_b200 import Bzip2
    m = model(name)
    data = CASES[name].data
    got, rs = raw_call(data, 0)
    assert rs == m.rows, name
    assert got == m.data, name
    got, rs = raw_call(data, 1)
    assert rs == m.rows and got == m.stream, name
    out, blocks = Bzip2.recover(data)
    assert out == m.data and rows_of(blocks) == m.rows
    out, blocks = Bzip2.recover(data, None, repair=True)
    assert out == m.stream and rows_of(blocks) == m.rows
    if streams:
        for repair in (False, True):
            w = Writer()
            out, blocks = Bzip2.recover(Reader(data, 65521), w, repair=repair)
            assert out is w and bytes(w.buf) == (m.stream if repair else m.data) and rows_of(blocks) == m.rows
    # the repaired stream decodes to the recovered bytes
    assert Bzip2.decompressFile(m.stream) == m.data
    if M.libbz2_language(data, m.rows):
        assert bz2.decompress(m.stream) == m.data


@pytest.mark.parametrize("name", sorted(CASES))
def test_case(name):
    CASES[name].check(model(name).rows)   # the case tests what it is named for
    check_case(name)


def test_undamaged_properties():
    from compressjs_b200 import Bzip2
    for name in ("undamaged_l1", "undamaged_l9", "undamaged_compressjs", "multistream_levels_1_9"):
        data = CASES[name].data
        out, blocks = Bzip2.recover(data)
        assert out == Bzip2.decompressFile(data, None, True)
    data = CASES["undamaged_l1"].data
    out, _ = Bzip2.recover(data, None, repair=True)
    assert out == data[:3] + b"9" + data[4:]


_SEAM_SCRIPT = r"""
import sys
sys.path.insert(0, %(root)r)
from tests import test_gpu_recover as G
for name in sorted(G.CASES):
    G.check_case(name, streams=False)
print("ok")
"""


@pytest.mark.parametrize("env", [dict(B2_DEC_WINDOW="65536", B2_DEC_BATCH="1"), dict(B2_DEC_WINDOW="65536", B2_DEC_BATCH="7")],
                         ids=["w64k_b1", "w64k_b7"])
def test_window_and_batch_seams(env):
    """Every case with 64 KiB windows and batches of 1 and 7 candidates, so that candidates and damage land on window and
    batch seams and damaged candidates reach past a window.  A child process: the library reads the hooks per call but
    the tests share it."""
    r = subprocess.run([sys.executable, "-c", _SEAM_SCRIPT % {"root": T.ROOT}], env=dict(os.environ, **env),
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stdout + r.stderr[-3000:]


@pytest.mark.parametrize("step", [1, 7, 4093])
def test_stream_read_sizes(step):
    from compressjs_b200 import Bzip2
    for name in ("garbage_between_blocks", "planted_inside_bad_crc", "truncated_last_block"):
        m = model(name)
        data = CASES[name].data
        for repair in (False, True):
            w = Writer()
            Bzip2.recover(Reader(data, step), w, repair=repair)
            assert bytes(w.buf) == (m.stream if repair else m.data), (name, step, repair)


def test_stream_aborts():
    from compressjs_b200 import Bzip2
    data = CASES["huffman_flip_bad_crc"].data
    m = model("huffman_flip_bad_crc")
    with pytest.raises(IOError):
        Bzip2.recover(Reader(data, 4096), Writer(fail_after=len(m.data) // 2))
    class BadReader(Reader):
        def read(self, buf, off, length):
            if self.pos > 20000:
                raise ValueError("read failed")
            return super().read(buf, off, length)
    with pytest.raises(ValueError):
        Bzip2.recover(BadReader(data, 4096), Writer(), repair=True)
    # the library is usable after an abort
    assert Bzip2.recover(data)[0] == m.data


def test_bad_arguments():
    from compressjs_b200 import _native
    L = _native.lib()
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rows, cnt = C.POINTER(_native.RecoveredBlock)(), C.c_size_t()
    assert L.b2_bzip2_recover(None, 0, 2, C.byref(out), C.byref(n), C.byref(rows), C.byref(cnt)) == -101
    assert L.b2_bzip2_recover(None, 0, 0, C.byref(out), C.byref(n), None, C.byref(cnt)) == -101
    assert L.b2_bzip2_recover(None, 0, 0, None, C.byref(n), C.byref(rows), C.byref(cnt)) == -101


# ---- scale: a 256 MiB multistream file of one-block members, every 37th member damaged ----
CHUNK = 850000


def _member(i):
    chunk = T.ascii_random(CHUNK, 1000 + i)
    z = bz2.compress(chunk, 9)
    if i % 37 == 5:
        g = T.rng(i)
        for _ in range(100):
            off = int(g.integers(100, len(z) - 100))
            d = bytearray(z)
            d[off] ^= 0x5A
            try:
                bz2.decompress(bytes(d))
            except (OSError, ValueError):
                return bytes(d), b""   # libbz2 rejects the damaged member
        raise AssertionError("no damage that libbz2 rejects")
    return z, chunk


# The command line's peak resident memory.  ru_maxrss of a child starts at its parent's resident size at fork, and the
# test process holds the whole expected output: the command runs under a small launcher, whose size is what it starts
# from, and the launcher writes the command's ru_maxrss (KiB) to a file.
_LAUNCH = r"""
import os, subprocess, sys
p = subprocess.Popen([sys.executable, "-m", "compressjs_b200"] + sys.argv[2:])
_, status, ru = os.wait4(p.pid, 0)
with open(sys.argv[1], "w") as f:
    f.write(str(ru.ru_maxrss))
sys.exit(os.waitstatus_to_exitcode(status))
"""


def _run_cli(args, src, dst, env):
    """The command line over files; (exit status, stderr, its peak resident memory in KiB)."""
    with open(src, "rb") as fi, open(dst, "wb") as fo:
        r = subprocess.run([sys.executable, "-c", _LAUNCH, dst + ".rss"] + args, stdin=fi, stdout=fo, stderr=subprocess.PIPE,
                           env=env, cwd=T.ROOT, timeout=1800)
    with open(dst + ".rss") as f:
        return r.returncode, r.stderr.decode(), int(f.read())


def test_scale_256mib_cli(tmp_path):
    n = (256 << 20) // CHUNK
    with ProcessPoolExecutor(max_workers=max(1, min(32, os.cpu_count() or 1))) as ex:
        members = list(ex.map(_member, range(n), chunksize=4))
    src = str(tmp_path / "in.bz2")
    with open(src, "wb") as f:
        for z, _ in members:
            f.write(z)
    expect = b"".join(c for _, c in members)
    lost = sum(1 for _, c in members if not c)
    env = dict(os.environ, B2_DEC_WINDOW=str(4 << 20), PYTHONPATH=T.ROOT)
    small = str(tmp_path / "small.bz2")
    with open(small, "wb") as f:
        f.write(members[0][0])
    rss0 = {flag: _run_cli(["-d", "-t", "bzip2", flag], small, str(tmp_path / "small.out"), env)[2] for flag in ("--recover", "--repair")}
    # the launcher keeps the parent's size out: what remains is the command's own (a Python process with a CUDA context)
    assert max(rss0.values()) < 4 << 20, rss0
    rc, err, rss = _run_cli(["-d", "-t", "bzip2", "--recover"], src, str(tmp_path / "out"), env)
    assert rc == 1
    lines = err.strip().split("\n")
    assert lines[-1] == "%d of %d blocks intact" % (n - lost, n) and len(lines) == lost + 1, err[-2000:]
    with open(str(tmp_path / "out"), "rb") as f:
        assert f.read() == expect
    # host memory of the stream call: under 3 max(W, 48 MiB) above the same command on a one-member file
    assert (rss - rss0["--recover"]) * 1024 < 3 * (48 << 20), (rss, rss0)
    rc, err, rss = _run_cli(["-d", "-t", "bzip2", "--repair"], src, str(tmp_path / "rep"), env)
    assert rc == 1 and (rss - rss0["--repair"]) * 1024 < 3 * (48 << 20), (rss, rss0)
    with open(str(tmp_path / "rep"), "rb") as f:
        assert bz2.decompress(f.read()) == expect
