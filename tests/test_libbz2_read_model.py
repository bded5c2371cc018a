"""The libbz2 decoder flavor's model (tests/libbz2_read_cases.py) without a GPU: it agrees with libbz2's recorded
verdicts, and with live libbz2 when bz2 links one; on streams in libbz2's language it gives what the compressjs flavor
gives; the derandomise table in the CUDA source is libbz2's; and --libbz2-decode's usage errors need no GPU."""
import bz2
import ctypes
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from tests import libbz2_read_cases as LC
from tests import synth_corpus as SC
from tests import util as T
from tests.golden.make_libbz2_read_golden import libbz2_read
from tests.test_cli_host import cli
from tests.test_libbz2_model import _libbz2_ok

GOLDEN = os.path.join(T.ROOT, "tests", "golden", "libbz2_read.json")
NAMES = sorted(LC.CASES)


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", NAMES)
def test_case_conditions_and_golden(name, golden):
    c = LC.build(name)
    assert c.cond and all(isinstance(v, (bool, np.bool_)) and bool(v) for v in c.cond.values()), c.cond
    g = golden[name]
    assert hashlib.sha256(c.data).hexdigest() == g["input_sha256"]
    e = c.expect(True)
    assert (e[0] == "ok") == g["accept"]
    if e[0] == "ok":
        assert (len(e[1]), hashlib.sha256(e[1]).hexdigest()) == (g["size"], g["sha256"])
    if _libbz2_ok():
        ok, out = libbz2_read(c.data)
        assert ok == (e[0] == "ok") and (not ok or out == e[1])


def test_every_rule_is_exercised():
    """Each rule makes at least one case differ from the compressjs flavor's reading of the same stream."""
    codes = {n: LC.build(n).expect(True) for n in NAMES}
    assert any(n.startswith("rand_") and e[0] == "ok" for n, e in codes.items())
    assert codes["sel_eq_groupcount"][:2] == ("err", -5) and codes["run4_at_end"][:2] == ("err", -5)
    assert codes["cut_header_only"][:2] == ("err", -3) and codes["tail_nuls"][0] == "ok"


@pytest.mark.parametrize("name", [n for n, fn in SC.CASES.items()])
def test_libbz2_language_reads_the_same(name):
    """Streams in libbz2's language (synth_corpus `libbz2=True`) give the same result in both flavors."""
    c = SC.build(name)
    if not c.libbz2:
        pytest.skip("not in libbz2's language")
    for ms in (False, True):
        exp = c.file.expect(ms)
        got = LC.model(c.file, ms)
        assert got[0] == exp[0] and got[1] == exp[1]


@pytest.mark.parametrize("name", ["sample%d.bz2" % i for i in range(5)])
def test_samples_are_libbz2_language(name):
    """bzip2 -d's member loop accepts the compressjs samples (the GPU test reads them in both flavors)."""
    data = T.fixture(name)
    ok, out = libbz2_read(data) if _libbz2_ok() else (True, None)
    assert ok
    if out is not None:
        assert out == bz2.decompress(data)


def test_table_in_cuda_source_is_libbz2s():
    t = LC.rnums()
    assert t[:4] == [619, 720, 127, 481] and (min(t), max(t), sum(t)) == (50, 999, 278212)
    assert hashlib.sha256(struct.pack("<512i", *t)).hexdigest() == LC.RNUMS_SHA256
    f = LC.flips()
    assert f[:3].tolist() == [617, 1337, 1464] and f.size == 1655
    try:
        live = list((ctypes.c_int32 * 512).in_dll(ctypes.CDLL("libbz2.so.1.0"), "BZ2_rNums"))
    except (OSError, ValueError):
        pytest.skip("libbz2.so.1.0 does not export BZ2_rNums here")
    assert live == t


@pytest.mark.parametrize("args,msg", [
    (["-z", "-t", "bzip2", "--libbz2-decode"], "--libbz2-decode can only be used with -d -t bzip2"),
    (["-t", "bzip2", "--libbz2-decode"], "--libbz2-decode can only be used with -d -t bzip2"),
    (["-d", "-t", "bwtc", "--libbz2-decode"], "--libbz2-decode can only be used with -d -t bzip2"),
    (["-d", "-t", "bzip2", "-b", "32", "--libbz2-decode"], "--libbz2-decode cannot be used with --block"),
    (["-d", "-t", "bzip2", "--recover", "--libbz2-decode"], "--libbz2-decode cannot be used with --recover or --repair"),
    (["-d", "-t", "bzip2", "--repair", "--libbz2-decode"], "--libbz2-decode cannot be used with --recover or --repair"),
    (["-d", "-t", "bzip2", "--libbz2", "--libbz2-decode"], "--libbz2-decode cannot be used with --libbz2"),
    (["-d", "-t", "bzip2", "--libbz2"], "--libbz2 can only be used with -z -t bzip2"),
])
def test_cli_usage_errors(args, msg):
    r = cli(*args)
    assert (r.returncode, r.stdout, r.stderr.decode().strip()) == (1, b"", msg)


def test_help_lists_libbz2_decode():
    assert "--libbz2-decode" in cli("--help").stdout.decode()


def test_unknown_flavor_raises_before_reading():
    from compressjs_b200.bzip2 import Bzip2

    class Src:
        def readByte(self):
            raise AssertionError("read before the flavor was checked")

    class Dst:
        def writeByte(self, b):
            raise AssertionError

    for flavor in ("gzip", None, 1):
        with pytest.raises(ValueError):
            Bzip2.decompressFile(Src(), Dst(), True, flavor=flavor)
        with pytest.raises(ValueError):
            Bzip2.decompressFile(b"BZh9", None, flavor=flavor)
