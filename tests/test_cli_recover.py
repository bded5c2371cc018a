"""The command line's --recover / --repair: usage errors without a GPU, and stderr, exit status and output on three
corpus cases (tests/recover_cases.py) on the GPU."""
import os
import subprocess
import sys

import pytest

from tests import recover_cases as RC
from tests import recover_model as M
from tests import util as T


def _cli(args, data=b""):
    return subprocess.run([sys.executable, "-m", "compressjs_b200"] + args, input=data, capture_output=True, cwd=T.ROOT,
                          env=dict(os.environ, PYTHONPATH=T.ROOT), timeout=600)


@pytest.mark.parametrize("args,msg", [
    (["--recover", "-t", "bzip2"], "--recover can only be used with -d -t bzip2"),
    (["-z", "--repair", "-t", "bzip2"], "--repair can only be used with -d -t bzip2"),
    (["-d", "--recover", "-t", "bwtc"], "--recover can only be used with -d -t bzip2"),
    (["-d", "--repair", "-t", "bzip2", "-b", "32"], "--repair cannot be used with --block"),
    (["-d", "--recover", "-t", "bzip2", "-9"], "--recover cannot be used with a compression level"),
    (["-d", "--repair", "-t", "bzip2", "--libbz2"], "--repair cannot be used with --libbz2"),
    (["-d", "--recover", "--repair", "-t", "bzip2"], "--recover and --repair cannot be used together"),
])
def test_usage_errors(args, msg):
    r = _cli(args)
    assert r.returncode == 1 and r.stdout == b"" and r.stderr.decode().strip() == msg


def test_help_lists_the_flags():
    out = _cli(["--help"]).stdout.decode()
    assert "--recover" in out and "--repair" in out


def _expected_stderr(rows):
    walked = [r for r in rows if r.status != M.INSIDE]
    lines = []
    for r in walked:
        if r.status == M.BAD_CRC:
            lines.append("block at bit %d: Data error: Bad block CRC (got %x expected %x)" % (r.bitpos, r.got, r.crc))
        elif r.status == M.DATA_ERROR:
            lines.append("block at bit %d: Data error" % r.bitpos)
        elif r.status == M.OBSOLETE:
            lines.append("block at bit %d: Obsolete (pre 0.9.5) bzip format not supported." % r.bitpos)
    intact = sum(r.status == M.INTACT for r in walked)
    lines.append("%d of %d blocks intact" % (intact, len(walked)))
    return "\n".join(lines) + "\n", 0 if intact == len(walked) else 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["huffman_flip_bad_crc", "planted_inside_intact", "randomised_bit"])
def test_cli_cases(name):
    data = RC.by_name()[name].data
    m = M.recover(data)
    err, status = _expected_stderr(m.rows)
    for flag, want in (("--recover", m.data), ("--repair", m.stream)):
        r = _cli(["-d", "-t", "bzip2", flag], data)
        assert r.returncode == status and r.stderr.decode() == err and r.stdout == want, (name, flag, r.stderr[-2000:])
