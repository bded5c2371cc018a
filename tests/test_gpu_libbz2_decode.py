"""The libbz2 decoder flavor on the GPU (Bzip2.decompressFile(flavor="libbz2"), b2_bzip2_decompress*_flavor) against the
model of tests/libbz2_read_cases.py: the same bytes, error code and partial-output prefix for every case, from bytes and
from streams, across window and batch seams; the default flavor unchanged; the command line; a 256 MiB multistream file
of randomised blocks; and round trips of both encoders' streams."""
import os
import subprocess
import sys

import pytest

from tests import bz2synth as W
from tests import libbz2_cases as LBC
from tests import libbz2_read_cases as LC
from tests import synth_corpus as SC
from tests import util as T
from tests.test_gpu_recover import Reader, Writer

pytestmark = pytest.mark.gpu

NAMES = sorted(LC.CASES)


def _dec(data, ms=True, flavor="libbz2"):
    from compressjs_b200 import bzip2
    out, err = bzip2._file(data, ms, bzip2._flavor(flavor))
    return ("ok", out.tobytes()) if err is None else ("err", err.errorCode, out.tobytes())


def _stream(data, step, ms=True):
    from compressjs_b200 import Bzip2, Bzip2Error
    w = Writer()
    try:
        Bzip2.decompressFile(Reader(data, step), w, ms, flavor="libbz2")
    except Bzip2Error as e:
        return ("err", e.errorCode, bytes(w.buf))
    return ("ok", bytes(w.buf))


def _short(r):
    return r[:2] + (len(r[2]),) if r[0] == "err" else (r[0], len(r[1]))


@pytest.mark.parametrize("name", NAMES)
def test_case(name):
    c = LC.build(name)
    for ms in (True, False):
        exp, got = c.expect(ms), _dec(c.data, ms)
        assert got == exp, (name, ms, _short(got), _short(exp))


@pytest.mark.parametrize("name", [n for n in NAMES if LC.build(n).cut is None and not LC.build(n).tail])
def test_default_flavor_unchanged(name):
    f = LC.build(name).f
    for ms in (True, False):
        got = _dec(f.data, ms, "compressjs")
        exp = f.expect(ms)
        assert got[:2] == exp[:2] if exp[0] == "err" else got == exp, (name, ms, _short(got))


@pytest.mark.parametrize("step", [1, 7, 4093])
def test_stream_read_sizes(step):
    bad = []
    for name in NAMES:
        c = LC.build(name)
        if step == 1 and len(c.data) > (1 << 18):
            continue   # byte-at-a-time Python reads of a megabyte: the 7- and 4093-byte runs cover these
        got, exp = _stream(c.data, step), c.expect(True)
        if got != exp:
            bad.append((name, _short(got), _short(exp)))
    assert not bad, bad


# B2_DEC_KEEP_CLS is not varied: only the sharded decode drops the count-byte classes, and it reads the compressjs
# flavor only.  The late_* cases lie behind the first 64 KiB window, where a stream's end is not known yet.
@pytest.mark.parametrize("env", [dict(B2_DEC_WINDOW="65536"), dict(B2_DEC_WINDOW="65536", B2_DEC_BATCH="1"),
                                 dict(B2_DEC_WINDOW="65536", B2_DEC_BATCH="7")],
                         ids=["w64k", "w64k_b1", "w64k_b7"])
def test_window_and_batch_seams(env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    bad = []
    for name in NAMES:
        c = LC.build(name)
        got, exp = _dec(c.data), c.expect(True)
        if got != exp:
            bad.append((name, _short(got), _short(exp)))
        for step in ((1, 4093) if name.startswith("late_") else (4093,)):
            got = _stream(c.data, step)
            if got != exp:
                bad.append((name, "stream", step, _short(got), _short(exp)))
    assert not bad, bad


@pytest.mark.parametrize("name", sorted(SC.CASES))
def test_libbz2_language_reads_the_same(name):
    """Streams in libbz2's language (synth_corpus `libbz2=True`) decode to the same bytes, code and prefix in both
    flavors."""
    c = SC.build(name)
    if not c.libbz2:
        pytest.skip("not in libbz2's language")
    for ms in (False, True):
        assert _dec(c.file.data, ms, "libbz2") == _dec(c.file.data, ms, "compressjs"), (name, ms)


@pytest.mark.parametrize("name", ["sample%d.bz2" % i for i in range(5)])
def test_samples_read_the_same(name):
    data = T.fixture(name)
    for ms in (False, True):
        got = _dec(data, ms, "libbz2")
        assert got[0] == "ok" and got == _dec(data, ms, "compressjs"), (name, ms)


def _cli(tmp_path, data, *args):
    src, dst = str(tmp_path / "in.bz2"), str(tmp_path / "out")
    with open(src, "wb") as f:
        f.write(data)
    r = subprocess.run([sys.executable, "-m", "compressjs_b200", "-d", "-t", "bzip2", "--libbz2-decode", *args, src, dst],
                       capture_output=True, cwd=T.ROOT, env=dict(os.environ, PYTHONPATH=T.ROOT), timeout=600)
    with open(dst, "rb") as f:
        return r.returncode, r.stderr.decode(), f.read()


@pytest.mark.parametrize("name,msg", [("rand_mixed_members", ""), ("tail_mib_nuls", ""), ("two_members_then_garbage", ""),
                                      ("cut_behind_block", "Unexpected input EOF"), ("rand_run4_at_end", "Data error"),
                                      ("tail_BZh", "Unexpected input EOF"), ("rand_bad_crc", "Data error: Bad block CRC")])
def test_cli(tmp_path, name, msg):
    c = LC.build(name)
    rc, err, out = _cli(tmp_path, c.data)
    exp = c.expect(True)
    if exp[0] == "ok":
        assert (rc, err, out) == (0, "", exp[1])
    else:
        k = len(exp[2])
        assert rc == 1 and err.startswith(msg), (rc, err)
        assert out == (exp[2][:4096 * ((k - 1) // 4096)] if k else b"")


def test_scale_256mib_randomised_multistream():
    """About 256 MiB of decoded output: members of one randomised 900 000-byte block each, three distinct ones repeated."""
    from compressjs_b200 import Bzip2
    import numpy as np
    members, outs = [], []
    for s in range(3):
        P = np.frombuffer(T.ascii_random(900000, 500 + s), np.uint8)
        b = LC.rand_block(P)
        members.append(W.Member([b], 9).data)
        outs.append(W.model_rle1(P)[0].tobytes())
    n = (256 << 20) // 900000
    data = b"".join(members[i % 3] for i in range(n))
    exp = b"".join(outs[i % 3] for i in range(n))
    assert bytes(Bzip2.decompressFile(data, None, True, flavor="libbz2")) == exp
    w = Writer()
    Bzip2.decompressFile(Reader(data, 1 << 20), w, True, flavor="libbz2")
    assert bytes(w.buf) == exp


def test_round_trips_of_both_encoders():
    from compressjs_b200 import Bzip2
    for data, level in ((T.texty(3 << 20, 3), 9), (T.runs(1 << 20, 4), 1), (b"", 9), (b"a" * 5, 1)):
        for enc in ("compressjs", "libbz2"):
            z = bytes(Bzip2.compressFile(data, None, level, flavor=enc))
            if enc == "libbz2" or _dec(z, True, "libbz2")[0] == "ok":
                assert _dec(z, True, "libbz2") == ("ok", data)
            assert _dec(z, True, "compressjs") == ("ok", data)
    # the compressjs encoder ends block 1 of this input on four equal bytes without their count byte: libbz2 rejects it
    data = LBC.motivating()
    cj, lb = bytes(Bzip2.compressFile(data, None, 1)), bytes(Bzip2.compressFile(data, None, 1, flavor="libbz2"))
    assert _dec(cj, True, "libbz2")[:3] == ("err", -5, b"") and _dec(cj, True, "compressjs") == ("ok", data)
    assert _dec(lb, True, "libbz2") == ("ok", data) == _dec(lb, True, "compressjs")
