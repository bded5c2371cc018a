"""b2_bwtc_compress_stream / b2_bwtc_decompress_stream: BWTC through read and write callbacks, in bounded memory.

- compress: the bytes written are those of b2_bwtc_compress (size given) or b2_bwtc_compress_unsized (size -1) on the
  bytes read, and the oracle's, however the input is split into reads and whatever $B2_BWT_BATCH is;
- decompress: the code and message are those of b2_bwtc_decompress, and the bytes written are its result, or on a data
  error the blocks decoded before the failing check, the same whatever the window, the batch and the reads;
- aborts, re-entry and over-long reads leave the library usable;
- device memory does not grow with the input, and stays within include/b2bz.h's bounds;
- the Python streams and the command line go through them.

Sorts last, like the other BWTC tests.  $B2_BWT_BATCH is read once per process: those cases run in a child process."""
import ctypes as C
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import oracle as O
from tests import bwtc_unsized as U
from tests import util as T
from tests.test_gpu_stream import Calls

pytestmark = pytest.mark.gpu

MiB = 1 << 20


def _N():
    from compressjs_b200 import _native
    return _native


def buf_compress(data, level, sized=True):
    N = _N()
    L = N.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    f = L.b2_bwtc_compress if sized else L.b2_bwtc_compress_unsized
    rc = f(a.ctypes.data if a.size else None, a.size, level, C.byref(out), C.byref(n))
    assert rc == 0, N.last_error()
    z = C.string_at(out, n.value)
    L.b2_free(out)
    return z


def buf_decompress(z):
    N = _N()
    L = N.lib()
    a = np.frombuffer(z, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    rc = L.b2_bwtc_decompress(a.ctypes.data if a.size else None, a.size, C.byref(out), C.byref(n))
    d = C.string_at(out, n.value) if rc == 0 else None
    if rc == 0:
        L.b2_free(out)
    return rc, d, N.last_error()


def stream_compress(data, level, size, pattern="all", **kw):
    cb = Calls(data, pattern, **kw)
    rc = _N().lib().b2_bwtc_compress_stream(cb.rd, cb.wr, None, level, size)
    return rc, bytes(cb.out), _N().last_error(), cb


def stream_decompress(z, pattern="all", **kw):
    cb = Calls(z, pattern, **kw)
    rc = _N().lib().b2_bwtc_decompress_stream(cb.rd, cb.wr, None)
    return rc, bytes(cb.out), _N().last_error(), cb


def header(size):
    """"bwtc" and the size field's groups as written: the last group is the range coder's first byte (lib/Util.js:105-141)."""
    v, g = size + 1, []
    while True:
        g.append(v & 0x7F)
        v >>= 7
        if not v:
            break
    return b"bwtc" + bytes(reversed(g[1:]))


def _child(code, env, timeout=1200):
    e = dict(os.environ)
    for k in ("B2_BWT_BATCH", "B2_BWTC_DEC_BATCH", "B2_DEC_WINDOW"):
        e.pop(k, None)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % T.ROOT + textwrap.dedent(code)],
                       env=e, capture_output=True, text=True, timeout=timeout, cwd=T.ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


# ---- compress --------------------------------------------------------------------------------------------------
COMPRESS_CHILD = """
import json
from oracle import oracle as O
from tests import bwtc_unsized as U
from tests import util as T
from tests.test_gpu_zz_bwtc_callbacks import buf_compress, stream_compress, _N
res = []
for level, k in ((1, 3), (5, 1), (6, 1), (9, 1)):
    bs = level * 100000
    for n in (0, 1, k * bs - 1, k * bs, k * bs + 1):
        data = T.texty(n, 1000 * level + n % 997)
        sized = buf_compress(data, level)
        st = _N().stats()
        ref = (st["raw_bytes"], st["comp_bytes"], st["blocks"])
        unsized = buf_compress(data, level, False)
        if ORACLE:
            assert sized == O.bwtc_compress(data, level), (level, n)
            assert unsized == U.unsized(data, level), (level, n)
        for p in ("ones", "odd", "all"):
            if p == "ones" and n > 400000:
                continue
            rc, z, err, cb = stream_compress(data, level, n, p)
            assert rc == 0 and z == sized, (level, n, p, rc, err)
            st = _N().stats()
            assert (st["raw_bytes"], st["comp_bytes"], st["blocks"]) == ref, (level, n, p)
            if p != "all" or n < 1000:
                rc, z, err, cb = stream_compress(data, level, -1, p)
                assert rc == 0 and z == unsized, (level, n, p, rc, err)
        res.append([level, n, len(sized)])
print(json.dumps(res))
"""


@pytest.mark.parametrize("batch", [1, 3, None])
def test_compress_matches_buffer_calls_and_oracle(batch):
    """Levels 1, 5, 6, 9 at 0, 1, k blockSize - 1, k blockSize, k blockSize + 1 bytes, every read pattern: reads,
    blocks and batches meet at every kind of seam.  The oracle checks the default batch."""
    env = {"B2_BWT_BATCH": str(batch)} if batch else {}
    res = _child("ORACLE = %r\n" % (batch is None) + COMPRESS_CHILD, env)
    assert len(res) == 20


@pytest.mark.parametrize("delta", [-1, 1])
def test_compress_declared_size(delta):
    """A size that differs from the bytes read goes into the header as given; decoding then fails the size check."""
    data = T.texty(250000, 11)
    rc, z, err, _ = stream_compress(data, 1, len(data) + delta, "odd")
    assert rc == 0, err
    # 250 001 +- 1 differ in the last 7-bit group only: the byte behind the written groups, the coder's first
    z0, i = buf_compress(data, 1), len(header(len(data)))
    assert header(len(data) + delta) == z0[:i] and len(z) == len(z0)
    assert z[:i] == z0[:i] and z[i] == z0[i] + delta and z[i + 1:] == z0[i + 1:]
    rc, d, err = buf_decompress(z)
    assert rc == -5 and "outputsize does not match decoded input" in err
    rc2, out, err2, _ = stream_decompress(z)
    assert (rc2, err2) == (rc, err)


# ---- decompress ------------------------------------------------------------------------------------------------
DATA = None


def _data():
    global DATA
    if DATA is None:   # 370 000 bytes: three full level-1 blocks and a short one
        DATA = T.runs(90000, 71) + T.texty(150000, 72) + b"q" * 50000 + T.ascii_random(80000, 73)
    return DATA


def _streams():
    d = _data()
    return {"sized": buf_compress(d, 1), "unsized": buf_compress(d, 1, False)}


CONFIGS = [(64 << 10, 1, "all"), (64 << 10, 2, "odd"), (70001, 3, "all"), (64 << 10, 3, "ones"), (None, None, "odd")]


def _set(monkeypatch, window, batch):
    for k, v in (("B2_DEC_WINDOW", window), ("B2_BWTC_DEC_BATCH", batch)):
        if v:
            monkeypatch.setenv(k, str(v))
        else:
            monkeypatch.delenv(k, raising=False)


def test_decompress_round_trip(monkeypatch):
    d = _data()
    for name, z in _streams().items():
        for window, batch, p in CONFIGS:
            _set(monkeypatch, window, batch)
            rc, out, err, cb = stream_decompress(z, p)
            assert rc == 0 and out == d, (name, window, batch, p, rc, err)
            assert cb.pos <= len(z)
            st = _N().stats()
            assert st["raw_bytes"] == len(d) and st["blocks"] == 4


def _front(streams, name, p):
    """The blocks whose decode never reads byte p of stream `name`: what a cut of the unsized stream there delivers
    (its coded bytes are the sized stream's, behind a header shorter by `shift` bytes)."""
    shift = len(header(len(_data()))) - 4 if name == "sized" else 0
    rc, out, err, _ = stream_decompress(streams["unsized"][:p - shift])
    assert rc == -5, err
    return out


def test_decompress_corruption_delivers_the_blocks_in_front(monkeypatch):
    """The flip and cut corruptions of test_batch_seams_and_errors: the code and message of the buffer call, the same
    bytes written in every configuration, and the blocks in front of the corrupted byte as they were.  A cut stream of
    unknown size delivers a whole number of blocks."""
    d = _data()
    streams = _streams()
    for name, z in streams.items():
        cases = {"flip%d" % i: (p, z[:p] + bytes([z[p] ^ 0x5A]) + z[p + 1:]) for i, p in enumerate((len(z) * 3 // 10, len(z) * 7 // 10, len(z) * 9 // 10))}
        cases.update({"cut%d" % i: (k, z[:k]) for i, k in enumerate((len(z) // 2, len(z) - 8))})
        for case, (p, bad) in cases.items():
            _set(monkeypatch, None, None)
            rc0, d0, err0 = buf_decompress(bad)
            front = _front(streams, name, p)
            seen = set()
            for window, batch, pat in CONFIGS:
                _set(monkeypatch, window, batch)
                rc, out, err, _ = stream_decompress(bad, pat)
                assert (rc, err) == (rc0, err0), (name, case, window, batch)
                if rc == 0:
                    assert out == d0
                seen.add(out)
            assert len(seen) == 1, (name, case)
            out = seen.pop()
            assert len(out) >= len(front) and out[:len(front)] == front == d[:len(front)], (name, case, len(out), len(front))
            if rc0 and name == "unsized" and case.startswith("cut"):
                assert rc0 == -5 and d.startswith(out) and (len(out) % 100000 == 0 or len(out) == len(d)), (case, len(out))
    # the size field one below the blocks fails when the last block passes it (that block is not written), one above
    # when the stream ends (every block is written); its last group is the byte behind the written groups
    z = streams["sized"]
    i = len(header(len(d)))
    for delta, blocks in ((-1, 3), (1, 4)):
        bad = z[:i] + bytes([z[i] + delta]) + z[i + 1:]
        rc0, _, err0 = buf_decompress(bad)
        assert rc0 == -5 and "outputsize" in err0
        for window, batch, pat in CONFIGS:
            _set(monkeypatch, window, batch)
            rc, out, err, _ = stream_decompress(bad, pat)
            assert (rc, err) == (rc0, err0) and out == d[:min(len(d), blocks * 100000)], (delta, window, batch)


def test_decompress_window_grows_for_a_long_block(monkeypatch):
    """A level-9 block whose coded bytes are more than three times the window: the window widens and the block decodes."""
    d = T.ascii_random(300000, 81)
    z = buf_compress(d, 9)
    assert len(z) > 3 * (64 << 10)
    for batch in (1, 2):
        _set(monkeypatch, 64 << 10, batch)
        rc, out, err, _ = stream_decompress(z, "odd")
        assert rc == 0 and out == d, err


def test_decompress_bad_input_writes_nothing(monkeypatch):
    _set(monkeypatch, 64 << 10, 2)
    z = _streams()["sized"]
    for bad in (b"", b"b", b"bwtc", b"bwt", b"bzzt\x81\x00\x00\x00", b"bwtc\x00", b"bwtc" + b"\x01" * 12,
                b"bwtc\x00\x00\x00\x00\x00\x00\x00\x00\x00\x81\x00", b"BZh91AY&SY" + z):
        rc0, _, err0 = buf_decompress(bad)
        assert rc0 in (-102, -5), (bad, rc0)
        for p in ("ones", "all"):
            rc, out, err, cb = stream_decompress(bad, p)
            assert (rc, err) == (rc0, err0) and out == b"" and cb.writes == 0, bad


def test_decompress_trailing_bytes(monkeypatch):
    """Bytes behind a stream: accepted exactly when the buffer call accepts them, with the same result."""
    d = _data()
    for name, z in _streams().items():
        for tail in (b"junk", b"\x00" * 100, b"\xff" * 7, z):
            rc0, d0, err0 = buf_decompress(z + tail)
            for window, batch, p in CONFIGS[:3]:
                _set(monkeypatch, window, batch)
                rc, out, err, _ = stream_decompress(z + tail, p)
                assert (rc, err) == (rc0, err0), (name, tail[:8], window, batch)
                if rc0 == 0:
                    assert out == d0 == d


# ---- aborts, re-entry, bad arguments ---------------------------------------------------------------------------
def test_aborts_then_next_call_works(monkeypatch):
    _set(monkeypatch, 64 << 10, 1)
    d = _data()
    z = buf_compress(d, 1)
    rc, out, err, cb = stream_compress(d, 1, len(d), "odd", abort_read_at=200000)
    assert rc == -103 and "read callback" in err and cb.after_abort == 0
    rc, out, err, cb = stream_compress(d, 1, len(d), "all", abort_write_at=2)
    assert rc == -103 and "write callback" in err and cb.after_abort == 0 and z.startswith(out)
    rc, out, err, cb = stream_compress(d, 1, len(d), "odd")
    assert rc == 0 and out == z
    rc, out, err, cb = stream_decompress(z, "odd", abort_read_at=len(z) // 2)
    assert rc == -103 and "read callback" in err and cb.after_abort == 0 and d.startswith(out)
    rc, out, err, cb = stream_decompress(z, "all", abort_write_at=2)
    assert rc == -103 and "write callback" in err and cb.after_abort == 0 and d.startswith(out) and len(out) == 100000
    rc, out, err, cb = stream_decompress(z, "all")
    assert rc == 0 and out == d


def test_bad_arguments_and_over_long_reads():
    class Liar(Calls):
        def _read(self, user, buf, cap):
            return cap + 1

    L = _N().lib()
    cb = Liar(b"")
    assert L.b2_bwtc_compress_stream(cb.rd, cb.wr, None, 1, -1) == -101 and cb.writes <= 1
    cb = Liar(b"")
    assert L.b2_bwtc_decompress_stream(cb.rd, cb.wr, None) == -101 and cb.writes == 0
    cb = Calls(b"abc")
    assert L.b2_bwtc_compress_stream(cb.rd, cb.wr, None, 1, -2) == -101 and cb.reads == 0 and cb.writes == 0
    rc, z, err, _ = stream_compress(b"after", 3, 5)
    assert rc == 0 and z == buf_compress(b"after", 3)


def test_library_call_from_a_callback_fails_instead_of_deadlocking():
    res = _child("""
        import ctypes as C, json
        from compressjs_b200 import _native as N
        from tests import util as T
        L = N.lib()
        seen = []
        data = T.texty(250000, 3)
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
            seen.append((L.b2_bwtc_decompress(None, 0, None, z), N.last_error()))
            out.extend(C.string_at(buf, n))
            return 0
        rc = L.b2_bwtc_compress_stream(N.READ_FN(rd), N.WRITE_FN(wr), None, 1, len(data))
        assert rc == 0 and N.last_error() == "", N.last_error()
        ok = all(s in ((0xFFFFFF9B, "called from inside a stream callback"), (-101, "called from inside a stream callback")) for s in seen)
        pos[0] = 0
        data = bytes(out)
        out.clear()
        rc2 = L.b2_bwtc_decompress_stream(N.READ_FN(rd), N.WRITE_FN(wr), None)
        print(json.dumps([rc, rc2, ok and len(seen) > 2, bytes(out) == T.texty(250000, 3)]))
    """, {})
    assert res == [0, 0, True, True]


# ---- memory ----------------------------------------------------------------------------------------------------
MEMORY_CHILD = """
import json
from compressjs_b200 import _native as N
from tests import util as T
from tests.test_gpu_zz_bwtc_callbacks import buf_compress, buf_decompress, stream_compress, stream_decompress
block = T.texty(100000, 5)   # every batch the same: the peak can only grow with the input, not with the data
res = {}
for nbatch in (2, 8):
    d = block * (4 * nbatch)
    z = buf_compress(d, 1)
    pb = N.stats()["dev_peak_bytes"]
    rc, zs, err, _ = stream_compress(d, 1, len(d), "odd")
    assert rc == 0 and zs == z, err
    ps = N.stats()["dev_peak_bytes"]
    rc, back, err = buf_decompress(z)
    assert rc == 0 and back == d, err
    qb = N.stats()["dev_peak_bytes"]
    rc, back, err, _ = stream_decompress(z, "odd")
    assert rc == 0 and back == d, err
    qs = N.stats()["dev_peak_bytes"]
    res[nbatch] = [pb, ps, qb, qs, len(z)]
print(json.dumps(res))
"""


def test_device_memory_does_not_grow_with_the_input():
    """Inputs 2 and 8 batches long (four blocks per batch, a 64 KiB decode window that both streams exceed): the buffer
    and the stream calls have the same device peak, the same for both inputs, within include/b2bz.h's bounds.  "The
    same" allows for the order in which stream-ordered frees and allocations meet; a peak that grew with the input
    would grow by the input and its output (compress) or by the compressed stream (decompress), far more."""
    W, B = 64 << 10, 4
    res = _child(MEMORY_CHILD, {"B2_BWT_BATCH": str(B), "B2_BWTC_DEC_BATCH": str(B), "B2_DEC_WINDOW": str(W)})
    (pb2, ps2, qb2, qs2, z2), (pb8, ps8, qb8, qs8, z8) = res["2"], res["8"]
    print("bwtc device peaks", res)
    assert z2 > W and z8 > 3 * z2
    assert max(pb2, ps2, pb8, ps8) - min(pb2, ps2, pb8, ps8) <= 256 << 10, res   # the input grows by 2.4 MB
    assert max(qb2, qs2, qb8, qs8) - min(qb2, qs2, qb8, qs8) <= 16 << 10, res    # the stream grows by more than 200 KB
    assert max(pb8, ps8) <= B * 96 * MiB + 8 * MiB, res
    assert max(qb8, qs8) <= W + B * 17 * MiB + 8 * MiB, res


# ---- Python streams --------------------------------------------------------------------------------------------
class In:
    def __init__(self, d, size=None):
        self.d, self.p = d, 0
        if size is not None:
            self.size = size

    def read(self, buf, off, n):
        k = min(n, 7777, len(self.d) - self.p)
        buf[off:off + k] = self.d[self.p:self.p + k]
        self.p += k
        return k

    def readByte(self):
        if self.p >= len(self.d):
            return -1
        self.p += 1
        return self.d[self.p - 1]


class Out:
    def __init__(self):
        self.b = bytearray()

    def writeByte(self, x):
        self.b.append(x)


def test_python_stream_pairs():
    from compressjs_b200 import BWTC
    d = T.texty(330000, 91)
    o = Out()
    assert BWTC.compressFile(In(d, len(d)), o, 2) is o and bytes(o.b) == O.bwtc_compress(d, 2)
    o = Out()
    assert BWTC.compressFile(In(d), o, 2) is o and bytes(o.b) == U.unsized(d, 2)   # no size: "size unknown"
    o = Out()
    BWTC.compressFile(In(d, -1), o, 12)
    assert bytes(o.b) == U.unsized(d, 9)
    z = O.bwtc_compress(d, 2)
    o = Out()
    assert BWTC.decompressFile(In(z), o) is o and bytes(o.b) == d
    bad = z[:len(z) * 8 // 10] + bytes([z[len(z) * 8 // 10] ^ 0x41]) + z[len(z) * 8 // 10 + 1:]
    o = Out()
    with pytest.raises(RuntimeError) as e1:
        BWTC.decompressFile(In(bad), o)
    with pytest.raises(RuntimeError) as e2:
        BWTC.decompressFile(bad)
    assert str(e1.value) == str(e2.value) and "code -5" in str(e1.value)
    rc, out, err, _ = stream_decompress(bad)
    assert bytes(o.b) == out
    o = Out()
    with pytest.raises(ValueError, match="Bad magic"):
        BWTC.decompressFile(In(b"bzzt\x81"), o)
    assert o.b == b""


# ---- the command line ------------------------------------------------------------------------------------------
def _cli(*args, stdin=None, env=None):
    return subprocess.run([sys.executable, "-m", "compressjs_b200"] + [str(a) for a in args], input=stdin, capture_output=True,
                          cwd=T.ROOT, timeout=900, env=env)


def test_cli_compress_gives_todays_bytes(tmp_path):
    d = T.texty(640000, 92)
    f = tmp_path / "in"
    f.write_bytes(d)
    sized, unsized = O.bwtc_compress(d, 4), U.unsized(d, 4)
    r = _cli("-z", "-t", "bwtc", "-4", f)
    assert r.returncode == 0 and r.stdout == sized, r.stderr
    with open(f, "rb") as h:
        r = subprocess.run([sys.executable, "-m", "compressjs_b200", "-z", "-t", "bwtc", "-4"], stdin=h, capture_output=True,
                           cwd=T.ROOT, timeout=900)
    assert r.returncode == 0 and r.stdout == sized, r.stderr
    r = _cli("-z", "-t", "bwtc", "-4", stdin=d)
    assert r.returncode == 0 and r.stdout == unsized, r.stderr


def test_cli_decode_error_keeps_the_flushed_prefix():
    from compressjs_b200 import BWTC
    d = T.texty(450000, 93)
    z = O.bwtc_compress(d, 1)
    for frac in (0.5, 0.85):
        p = int(len(z) * frac)
        bad = z[:p] + bytes([z[p] ^ 0x21]) + z[p + 1:]
        s = Out()
        with pytest.raises(Exception) as ei:
            BWTC.decompressFile(In(bad), s)
        k = len(s.b)
        r = _cli("-d", "-t", "bwtc", stdin=bad)
        assert r.returncode == 1
        assert r.stdout == bytes(s.b[:4096 * ((k - 1) // 4096)] if k else b""), (frac, k, len(r.stdout))
        assert r.stderr.decode().strip() == str(ei.value)


def test_cli_pipeline_bounded_memory(tmp_path):
    """`-z -t bwtc -1 | -d -t bwtc` as separate processes with small knobs: the bytes come back, and the resident memory
    of each process does not grow with the stream (a ~24 MiB stream against a 1 MiB one)."""
    from tests.test_gpu_stream import CONSUMER, PRODUCER, WRAPPER
    for name, src in (("producer.py", PRODUCER % {"root": T.ROOT}), ("consumer.py", CONSUMER), ("wrapper.py", WRAPPER)):
        (tmp_path / name).write_text(src)
    env = dict(os.environ, B2_BWT_BATCH="2", B2_BWTC_DEC_BATCH="2", B2_DEC_WINDOW=str(64 << 10))
    py, t = sys.executable, str(tmp_path)
    res = {}
    for n in (1 << 20, 24 << 20):
        cmd = ("set -o pipefail; %(py)s %(t)s/producer.py %(n)d 78 %(t)s/pdigest | "
               "%(py)s %(t)s/wrapper.py %(t)s/rss_z %(py)s -m compressjs_b200 -z -t bwtc -1 | "
               "%(py)s %(t)s/wrapper.py %(t)s/rss_d %(py)s -m compressjs_b200 -d -t bwtc | "
               "%(py)s %(t)s/consumer.py %(t)s/cdigest") % dict(py=py, t=t, n=n)
        import time
        t0 = time.perf_counter()
        r = subprocess.run(["bash", "-c", cmd], cwd=T.ROOT, env=env, capture_output=True, text=True, timeout=1500)
        dt = time.perf_counter() - t0
        assert r.returncode == 0, r.stderr
        cd, cn = (tmp_path / "cdigest").read_text().split()
        assert cd == (tmp_path / "pdigest").read_text() and int(cn) == n
        res[n] = {k: int((tmp_path / ("rss_" + k)).read_text()) for k in ("z", "d")}
        res[n]["wall_s"] = round(dt, 2)
    print("bwtc pipeline", res)
    small, big = res[1 << 20], res[24 << 20]
    for k in ("z", "d"):
        assert big[k] - small[k] <= 16 * MiB, res
