"""b2_bzip2_compress_stream / b2_bzip2_decompress_stream: read and write callbacks instead of whole buffers.

- compress: the bytes written are those of b2_bzip2_compress on the bytes read, however the input is split into reads;
- decompress: the bytes written, the code and the message are those of b2_bzip2_decompress_partial, and nothing past
  that prefix is ever written;
- an abort in a callback, a callback that calls the library, and a read that claims too much all leave the library
  usable;
- device memory stays within the bounds of the whole-buffer calls, and the command line pipes a stream many windows
  long through separate compress and decompress processes in bounded memory."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests import partial_cases as P
from tests import rle1_cases as RC
from tests import util as T

pytestmark = pytest.mark.gpu

ONE_BYTE_MAX = 300000    # 1-byte reads only up to this size (one Python call per byte)


def _N():
    from compressjs_b200 import _native
    return _native


# read patterns: the sizes of successive reads (cycled), each cut to what the library asks for; None = all it asks for
PATTERNS = {"ones": [1], "odd": [1, 3, 7, 4093, 65537, 999983, 2], "all": None}


def _patterns(n):
    return [p for p in PATTERNS if p != "ones" or n <= ONE_BYTE_MAX]


class Calls:
    """The two callbacks over `data`, with a read pattern; records everything written."""

    def __init__(self, data, pattern="all", abort_read_at=None, abort_write_at=None, inside=None):
        self.data, self.sizes = data, PATTERNS[pattern]
        self.pos = self.k = 0
        self.out = bytearray()
        self.writes = self.reads = 0
        self.after_abort = 0
        self.aborted = False
        self.abort_read_at, self.abort_write_at, self.inside = abort_read_at, abort_write_at, inside
        N = _N()
        self.rd = N.READ_FN(self._read)
        self.wr = N.WRITE_FN(self._write)

    def _read(self, user, buf, cap):
        self.reads += 1
        if self.aborted:
            self.after_abort += 1
        if self.inside:
            self.inside()
        if self.abort_read_at is not None and self.pos >= self.abort_read_at:
            self.aborted = True
            return -1
        want = cap if self.sizes is None else self.sizes[self.k % len(self.sizes)]
        self.k += 1
        k = min(want, cap, len(self.data) - self.pos)
        if k:
            C.memmove(buf, self.data[self.pos:self.pos + k], k)
        self.pos += k
        return k

    def _write(self, user, buf, n):
        self.writes += 1
        if self.aborted:
            self.after_abort += 1
        if self.abort_write_at is not None and self.writes >= self.abort_write_at:
            self.aborted = True
            return 7
        self.out += C.string_at(buf, n)
        return 0


def stream_compress(data, level, pattern="all", **kw):
    L = _N().lib()
    cb = Calls(data, pattern, **kw)
    rc = L.b2_bzip2_compress_stream(cb.rd, cb.wr, None, level)
    return rc, bytes(cb.out), _N().last_error(), cb


def stream_decompress(data, ms, pattern="all", **kw):
    L = _N().lib()
    cb = Calls(data, pattern, **kw)
    rc = L.b2_bzip2_decompress_stream(cb.rd, cb.wr, None, int(ms))
    return rc, bytes(cb.out), _N().last_error(), cb


def one_shot(data, level):
    N = _N()
    L = N.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = L.b2_bzip2_compress(a.ctypes.data if a.size else None, a.size, level, C.byref(out), C.byref(n))
    assert rc == 0, N.last_error()
    z = C.string_at(out, n.value)
    L.b2_free(out)
    return z


def partial(data, ms):
    N = _N()
    L = N.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = L.b2_bzip2_decompress_partial(a.ctypes.data if a.size else None, a.size, int(ms), C.byref(out), C.byref(n))
    z = C.string_at(out, n.value) if out else None
    L.b2_free(out)
    return rc, z, N.last_error()


def check_compress(data, level, patterns=None):
    exp = one_shot(data, level)
    tr = [(t.raw_start, t.raw_len, t.bit_start, t.crc) for t in _N().last_trace()]
    for p in patterns or _patterns(len(data)):
        rc, z, err, _ = stream_compress(data, level, p)
        assert rc == 0, err
        assert z == exp, (p, len(data), level)
        assert [(t.raw_start, t.raw_len, t.bit_start, t.crc) for t in _N().last_trace()] == tr
        st = _N().stats()
        assert st["raw_bytes"] == len(data) and st["comp_bytes"] == len(exp)


def check_decompress(data, ms, patterns=None):
    rc0, exp, err0 = partial(data, ms)
    assert rc0 in (0, -2, -5, -7), err0
    for p in patterns or _patterns(len(data)):
        rc, out, err, cb = stream_decompress(data, ms, p)
        assert (rc, err) == (rc0, err0), p
        assert out == exp, (p, len(out), len(exp))   # everything ever written: nothing past the prefix
        assert cb.pos <= len(data)


# ---- compress ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sample0", "sample1", "sample2", "sample3", "sample4", "sample5"])
@pytest.mark.parametrize("level", [1, 9])
def test_compress_samples(name, level):
    check_compress(T.fixture(name + ".ref"), level)


def test_compress_fuzz():
    g = T.rng(20261016)
    for i in range(10):
        n = int(g.integers(0, 3 << 20)) if i else 0
        kind = ("texty", "runs")[i % 2]
        data = (T.texty if kind == "texty" else T.runs)(n, 700 + i)
        check_compress(data, int(g.integers(1, 10)))


def test_compress_empty_gives_the_14_byte_file():
    rc, z, err, cb = stream_compress(b"", 9)
    assert rc == 0 and z == one_shot(b"", 9) and len(z) == 14 and cb.reads == 1


def test_compress_rle1_seam_cases(monkeypatch):
    for c in RC.cases():
        for lv in c.levels:
            check_compress(c.data, lv, [p for p in ("odd", "all", "ones") if p != "ones" or len(c.data) <= 100000])
        for w in c.window:
            monkeypatch.setenv("B2_STREAM_WINDOW", str(RC.window_bytes(c, w)))
            check_compress(c.data, c.levels[0], ["odd", "all"])
            monkeypatch.delenv("B2_STREAM_WINDOW")


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_compress_window_edges(delta, monkeypatch):
    """Inputs of one window and one window +- 1 byte: the stream only knows a window is the last one after a read
    returns 0, and must still cut the windows b2_bzip2_compress cuts."""
    W = 1 << 20
    monkeypatch.setenv("B2_STREAM_WINDOW", str(W))
    for level, data in ((1, T.texty(W + delta, 5)), (1, T.ascii_random(2 * W + delta, 6)), (2, T.texty(3 * W + delta, 7))):
        check_compress(data, level, ["odd", "all"])


def test_compress_many_windows_under_one_byte_reads_at_the_start(monkeypatch):
    monkeypatch.setenv("B2_STREAM_WINDOW", str(1 << 20))
    data = T.texty(200000, 8) + T.ascii_random(3 << 20, 9)
    check_compress(data, 1, ["ones", "odd"])


# ---- decompress --------------------------------------------------------------------------------------------------
@pytest.fixture
def small_windows(monkeypatch):
    monkeypatch.setenv("B2_DEC_WINDOW", str(64 << 10))
    monkeypatch.setenv("B2_DEC_BATCH", "3")


def test_decompress_partial_cases(small_windows):
    for name, f, _ in P.files():
        for ms in (0, 1):
            check_decompress(f.data, ms)


def test_decompress_fixtures(small_windows):
    for name in ("sample0", "sample1", "sample2", "sample3", "sample4"):
        z = T.fixture(name + ".bz2")
        check_decompress(z, 0, ["odd", "all"])
        check_decompress(z, 1, ["all"])
    # members of different levels back to back, and garbage behind the last
    z = one_shot(T.texty(300000, 3), 1) + one_shot(T.runs(500000, 4), 9) + one_shot(b"", 5)
    for tail in (b"", b"BZh9", b"BZh", b"junk", b"BZh91AY&SY"):
        check_decompress(z + tail, 1, ["odd", "all"])
        check_decompress(z + tail, 0, ["all"])


def test_decompress_truncation_sweep(small_windows):
    data = T.ascii_random(150000, 21) + T.runs(200000, 22) + T.texty(250000, 23)
    z = one_shot(data, 1)
    g = T.rng(5)
    cuts = sorted(set([0, 1, 3, 4, 5, 10, 11, len(z) - 1, len(z) - 4, len(z) - 10, len(z) - 11])
                  | set(int(x) for x in g.integers(0, len(z), 40)))
    for cut in cuts:
        check_decompress(z[:cut], 0, ["odd", "all"])
    # a flipped bit in each block, too
    for bit in g.integers(32, len(z) * 8, 12):
        b = bytearray(z)
        b[int(bit) // 8] ^= 0x80 >> (int(bit) % 8)
        check_decompress(bytes(b), 0, ["all"])


def test_decompress_round_trip_large(monkeypatch):
    monkeypatch.setenv("B2_DEC_WINDOW", str(1 << 20))
    data = T.texty(20 << 20, 31) + T.runs(4 << 20, 32)
    z = one_shot(data, 9)
    rc, out, err, _ = stream_decompress(z, 0, "odd")
    assert rc == 0 and out == data, err


# ---- aborts, re-entry, bad arguments ---------------------------------------------------------------------------
def test_read_abort_then_next_call_works(monkeypatch):
    monkeypatch.setenv("B2_STREAM_WINDOW", str(1 << 20))
    data = T.texty(5 << 20, 41)
    rc, z, err, cb = stream_compress(data, 1, "odd", abort_read_at=2500000)
    assert rc == -103 and "read callback" in err and cb.after_abort == 0
    check_compress(data[:300000], 1, ["all"])
    zz = one_shot(data, 1)
    rc, out, err, cb = stream_decompress(zz, 0, "odd", abort_read_at=len(zz) // 2)
    assert rc == -103 and "read callback" in err and cb.after_abort == 0
    assert data.startswith(out)
    check_decompress(zz, 0, ["all"])


def test_write_abort_then_next_call_works(monkeypatch):
    monkeypatch.setenv("B2_STREAM_WINDOW", str(1 << 20))
    monkeypatch.setenv("B2_DEC_WINDOW", str(256 << 10))
    data = T.texty(5 << 20, 42)
    rc, z, err, cb = stream_compress(data, 1, "all", abort_write_at=2)
    assert rc == -103 and "write callback" in err and cb.after_abort == 0 and one_shot(data, 1).startswith(z)
    zz = one_shot(data, 1)
    rc, out, err, cb = stream_decompress(zz, 0, "all", abort_write_at=2)
    assert rc == -103 and "write callback" in err and cb.after_abort == 0 and data.startswith(out)
    check_compress(data, 1, ["all"])
    check_decompress(zz, 0, ["all"])


def test_bad_level_and_bad_reads():
    rc, z, err, cb = stream_compress(b"abc", 10)
    assert rc == -100 and cb.reads == 0 and cb.writes == 0

    class Liar(Calls):
        def _read(self, user, buf, cap):
            return cap + 1

    L = _N().lib()
    cb = Liar(b"")
    assert L.b2_bzip2_compress_stream(cb.rd, cb.wr, None, 1) == -101 and cb.writes == 0
    assert L.b2_bzip2_decompress_stream(cb.rd, cb.wr, None, 0) == -101 and cb.writes == 0
    check_compress(b"after", 3, ["all"])


def test_python_exceptions_are_raised_after_the_call():
    """An exception inside a callback aborts the call (never taken for the end of the input) and is raised again."""
    from compressjs_b200 import Bzip2

    class In:
        def __init__(self, d, fail_at):
            self.d, self.p, self.fail_at = d, 0, fail_at

        def read(self, buf, off, n):
            if self.p >= self.fail_at:
                raise KeyError("input went away")
            k = min(n, 5000, len(self.d) - self.p)
            buf[off:off + k] = self.d[self.p:self.p + k]
            self.p += k
            return k

        def readByte(self):
            raise AssertionError

    class Out:
        def __init__(self):
            self.b = bytearray()

        def writeByte(self, x):
            self.b.append(x)

        def write(self, buf, off, n):
            self.b += buf[off:off + n]

    data = T.texty(400000, 44)
    with pytest.raises(KeyError):
        Bzip2.compressFile(In(data, 200000), Out(), 1)
    o = Out()
    assert Bzip2.compressFile(In(data, len(data) + 1), o, 1) is o and bytes(o.b) == Bzip2.compressFile(data, None, 1)
    z = bytes(o.b)
    with pytest.raises(KeyError):
        Bzip2.decompressFile(In(z, len(z) // 2), Out())
    o = Out()
    assert Bzip2.decompressFile(In(z, len(z) + 1), o) is o and bytes(o.b) == data
    with pytest.raises(ValueError, match="Invalid block size multiplier"):
        Bzip2.compressFile(In(data, 0), Out(), 11)   # before any read (the read would raise KeyError)
    # a decode error is raised after the prefix went out, as on the buffer path
    bad = bytearray(z)
    bad[len(z) // 2] ^= 0x10
    o, s = Out(), Out()
    with pytest.raises(Exception) as e1:
        Bzip2.decompressFile(In(bytes(bad), len(z) + 1), o)
    with pytest.raises(Exception) as e2:
        Bzip2.decompressFile(bytes(bad), s)
    assert type(e1.value) is type(e2.value) and str(e1.value) == str(e2.value) and o.b == s.b


def test_library_call_from_a_callback_fails_instead_of_deadlocking():
    code = textwrap.dedent("""
        import ctypes as C, sys
        sys.path.insert(0, %r)
        from compressjs_b200 import _native as N
        L = N.lib()
        seen = []
        data = b"hello stream " * 1000
        pos = [0]
        def rd(user, buf, cap):
            seen.append((L.b2_crc32_bzip2(None, 0), N.last_error()))
            k = min(cap, len(data) - pos[0])
            C.memmove(buf, data[pos[0]:pos[0] + k], k)
            pos[0] += k
            return k
        out = bytearray()
        def wr(user, buf, n):
            z = (C.c_size_t * 1)()
            seen.append((L.b2_bzip2_decompress(None, 0, 0, None, z), N.last_error()))
            out.extend(C.string_at(buf, n))
            return 0
        rc = L.b2_bzip2_compress_stream(N.READ_FN(rd), N.WRITE_FN(wr), None, 9)
        assert rc == 0, N.last_error()
        assert N.last_error() == ""
        assert seen and all(s == (0xFFFFFF9B, "called from inside a stream callback") or s == (-101, "called from inside a stream callback") for s in seen), seen
        assert L.b2_crc32_bzip2(b"abc", 3) != 0xFFFFFF9B
        print("ok", len(out))
    """ % T.ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stdout + r.stderr


# ---- memory ------------------------------------------------------------------------------------------------------
def test_device_memory_within_the_whole_buffer_bounds(monkeypatch):
    W = 8 << 20
    monkeypatch.setenv("B2_STREAM_WINDOW", str(W))
    data = T.texty(40 << 20, 51)
    z = one_shot(data, 9)
    peak_one = _N().stats()["dev_peak_bytes"]
    rc, out, err, _ = stream_compress(data, 9, "odd")
    assert rc == 0 and out == z
    assert _N().stats()["dev_peak_bytes"] <= peak_one
    monkeypatch.setenv("B2_DEC_WINDOW", str(W))
    monkeypatch.setenv("B2_DEC_BATCH", "16")
    rc, back, err, _ = stream_decompress(z, 0, "odd")
    assert rc == 0 and back == data
    peak = _N().stats()["dev_peak_bytes"]
    magics = len(data) // 800000 + 16
    assert peak <= 2 * max(W, 48 << 20) + 16 * (24 << 20) + 16 * magics, peak


PRODUCER = """
import hashlib, sys
sys.path.insert(0, %(root)r)
from tests import util as T
n, seed, digest = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
base = T.texty(8 << 20, seed)
h = hashlib.sha256()
out = sys.stdout.buffer
i = 0
while n > 0:
    k = (i * 1000003) %% len(base)
    piece = (b"%%012d" %% i + base[k:] + base[:k])[:min(n, len(base))]
    h.update(piece)
    out.write(piece)
    n -= len(piece)
    i += 1
out.flush()
open(digest, "w").write(h.hexdigest())
"""

CONSUMER = """
import hashlib, sys
h, n = hashlib.sha256(), 0
while True:
    b = sys.stdin.buffer.read(1 << 20)
    if not b:
        break
    h.update(b)
    n += len(b)
open(sys.argv[1], "w").write("%s %d" % (h.hexdigest(), n))
"""

WRAPPER = """
import resource, subprocess, sys
rc = subprocess.call(sys.argv[2:])
open(sys.argv[1], "w").write(str(resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss * 1024))
sys.exit(rc)
"""


def _pipeline(tmp_path, n, W, keep_compressed=False):
    """producer | CLI -z | CLI -d | consumer, as separate processes; (producer digest, (consumer digest, bytes), rss)."""
    for name, src in (("producer.py", PRODUCER % {"root": T.ROOT}), ("consumer.py", CONSUMER), ("wrapper.py", WRAPPER)):
        (tmp_path / name).write_text(src)
    py = sys.executable
    t = str(tmp_path)
    tee = "tee %s/z.bz2 |" % t if keep_compressed else ""
    cmd = ("set -o pipefail; %(py)s %(t)s/producer.py %(n)d 77 %(t)s/pdigest | "
           "%(py)s %(t)s/wrapper.py %(t)s/rss_z %(py)s -m compressjs_b200 -z -t bzip2 -9 | %(tee)s"
           "%(py)s %(t)s/wrapper.py %(t)s/rss_d %(py)s -m compressjs_b200 -d -t bzip2 | "
           "%(py)s %(t)s/consumer.py %(t)s/cdigest") % dict(py=py, t=t, n=n, tee=tee)
    env = dict(os.environ, B2_STREAM_WINDOW=str(W), B2_DEC_WINDOW=str(W))
    r = subprocess.run(["bash", "-c", cmd], cwd=T.ROOT, env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stderr
    pd = (tmp_path / "pdigest").read_text()
    cd, cn = (tmp_path / "cdigest").read_text().split()
    return pd, (cd, int(cn)), {k: int((tmp_path / ("rss_" + k)).read_text()) for k in ("z", "d")}


def test_cli_pipeline_small_matches_one_shot(tmp_path, monkeypatch):
    """At a size that fits in memory, the command line's stream is b2_bzip2_compress's."""
    W = 64 << 20
    n = 5 * W + 12345
    pd, (cd, cn), rss = _pipeline(tmp_path, n, W, keep_compressed=True)
    assert cd == pd and cn == n
    proc = subprocess.run([sys.executable, str(tmp_path / "producer.py"), str(n), "77", str(tmp_path / "p2")],
                          capture_output=True, check=True, timeout=600)
    monkeypatch.setenv("B2_STREAM_WINDOW", str(W))
    assert (tmp_path / "z.bz2").read_bytes() == one_shot(proc.stdout, 9)


def test_cli_pipeline_bounded_memory(tmp_path):
    """A stream of 2 GiB + 1 MiB, 32 windows long, through `-z | -d` as separate processes: the bytes come back and
    each process stays far below the stream's size -- within the library's bound (include/b2bz.h) plus what the
    interpreter and the CUDA runtime take, measured on a 1 KiB stream."""
    W = 64 << 20
    n = (2 << 30) + (1 << 20)
    base = tmp_path / "tiny"
    base.mkdir()
    _, _, rss0 = _pipeline(base, 1024, W)
    pd, (cd, cn), rss = _pipeline(tmp_path, n, W)
    assert cd == pd and cn == n
    slack = 96 << 20
    assert rss["z"] - rss0["z"] <= 3 * W + (1 << 20) + slack, (rss, rss0)
    assert rss["d"] - rss0["d"] <= 3 * max(W, 48 << 20) + slack, (rss, rss0)
    assert max(rss.values()) < n // 2, rss
    print("rss", rss, "baseline", rss0)
