"""The command line (python -m compressjs_b200, a port of bin/compressjs) without a GPU: usage errors, --help,
--version, the size rule of BWTC input, and the streams of unknown size that the command line reproduces (derived
from the oracle's sized streams by tests/bwtc_unsized.py) decoding back through the oracle."""
import os
import subprocess
import sys

import pytest

from oracle import oracle as O
from tests import bwtc_unsized as U
from tests import util as T


def cli(*args, stdin=b""):
    # no device and no library: a usage error must be found before either is needed
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", B2_LIB=os.path.join(T.ROOT, "no-such-lib.so"))
    return subprocess.run([sys.executable, "-m", "compressjs_b200"] + list(args), input=stdin, capture_output=True,
                          cwd=T.ROOT, env=env, timeout=120)


@pytest.mark.parametrize("args,msg", [
    (["-d", "-z"], "Must specify either -d or -z."),
    (["-b", "5"], "--block can only be used with decompression"),
    (["-z", "--block", "0", "-t", "bzip2"], "--block can only be used with decompression"),
    (["-z", "-5", "-3"], "Can't specify both -3 and -5"),
    (["-9", "-1", "-4"], "Can't specify both -1 and -4"),
    (["-d", "-6"], "Compression level has no effect when decompressing."),
    (["-z", "-t", "nope"], "Unknown compressor: nope"),
    (["-d", "-t", "BzipX"], "Unknown compressor: BzipX"),
])
def test_usage_errors(args, msg):
    r = cli(*args)
    assert r.returncode == 1
    assert r.stderr.decode().strip() == msg
    assert r.stdout == b""


@pytest.mark.parametrize("args", [["-z"], [], ["-t", "lzp3"], ["-d", "-t", "PPM"], ["-t", "huffman", "-9"]])
def test_other_compressors_name_the_ones_there_are(args):
    """The reference's other compressors, and its default lzp3 (no -t), fail instead of writing bzip2 or bwtc."""
    r = cli(*args)
    assert r.returncode == 1
    err = r.stderr.decode()
    assert "bzip2" in err and "bwtc" in err
    assert r.stdout == b""


def test_block_needs_bzip2():
    r = cli("-d", "-t", "bwtc", "-b", "32")
    assert r.returncode == 1 and b"BWTC.decompressBlock" in r.stderr


def test_help_and_version():
    for a in ("-V", "--version"):
        r = cli(a)
        assert r.returncode == 0 and r.stdout == b"0.0.1\n"
    for a in ("-h", "--help"):
        r = cli(a)
        out = r.stdout.decode()
        assert r.returncode == 0
        assert "-d|-z [infile] [outfile]" in out
        for opt in ("--decompress", "--compress", "--block <n>", "-t <compressor>", "-1", "-9", "--version"):
            assert opt in out
        assert "  If <infile> is omitted, reads from stdin.\n  If <outfile> is omitted, writes to stdout.\n" in out


def test_unreadable_input_fails():
    r = cli("-z", "-t", "bzip2", os.path.join(T.ROOT, "no-such-input"))
    assert r.returncode == 1 and b"no-such-input" in r.stderr


def test_size_rule(tmp_path):
    """BWTC writes a size exactly when fstat gives one: a regular non-empty file.  An empty file and a pipe are of
    unknown size (bin/compressjs:60-65)."""
    from compressjs_b200 import cli as C
    f = tmp_path / "f"
    f.write_bytes(b"abc" * 1000)
    with open(f, "rb") as h:
        data, size = C.read_input(h.fileno())
        assert size == 3000 and bytes(data) == b"abc" * 1000
    e = tmp_path / "e"
    e.write_bytes(b"")
    with open(e, "rb") as h:
        data, size = C.read_input(h.fileno())
        assert size == 0 and bytes(data) == b""
    r, w = os.pipe()
    os.write(w, b"piped" * 100)
    os.close(w)
    try:
        data, size = C.read_input(r)
        assert size == 0 and bytes(data) == b"piped" * 100
    finally:
        os.close(r)


@pytest.mark.parametrize("level", [1, 5, 6, 9])
def test_oracle_unknown_size_round_trip(level):
    """lib/Util.js:119-124 with fileSize = -1: the size field is the single byte 0x80, handed to the range coder; the
    unchanged oracle decoder reads such streams back."""
    for n in (0, 1, level * 100000 - 1, level * 100000, level * 100000 + 1):
        d = T.texty(n, 100 + n)
        z = U.unsized(d, level)
        assert z[:4] == b"bwtc" and z[4] == 0x80
        assert O.bwtc_decompress(z) == d
