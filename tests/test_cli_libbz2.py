"""--libbz2 on the command line without a GPU: it is a usage error anywhere but with -z -t bzip2, found before the
library is loaded; the flavor argument of Bzip2.compressFile is checked before anything is read."""
import pytest

from tests.test_cli_host import cli


@pytest.mark.parametrize("args", [["-d", "-t", "bzip2", "--libbz2"], ["-z", "-t", "bwtc", "--libbz2"], ["-t", "bwtc", "-1", "--libbz2"]])
def test_libbz2_needs_compress_bzip2(args):
    r = cli(*args)
    assert r.returncode == 1
    assert r.stderr.decode().strip() == "--libbz2 can only be used with -z -t bzip2"
    assert r.stdout == b""


def test_help_lists_libbz2():
    assert "--libbz2" in cli("--help").stdout.decode()


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
            Bzip2.compressFile(Src(), Dst(), 9, flavor=flavor)
