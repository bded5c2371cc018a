"""GPU parity of the BWTC container path (compressjs_b200/csrc/bwtc.cu; lib/BWTC.js:12-231) against the oracle.
The file sorts last on purpose: the path is the newest one; the serial code it executes is also checked on the host
by tests/test_host_api.py::test_bwtc_core_matches_oracle."""
import pytest

from oracle import oracle as O
from tests import util as T

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("level", [1, 5, 6, 9])
@pytest.mark.parametrize("name", ["sample0", "sample1", "sample2", "sample3"])
def test_bwtc_samples(name, level):
    from compressjs_b200 import BWTC
    d = T.fixture(name + ".ref")
    z = BWTC.compressFile(d, None, level)
    assert z == O.bwtc_compress(d, level)
    assert BWTC.decompressFile(z) == d


@pytest.mark.parametrize("name", ["sample4", "sample5"])
def test_bwtc_900k_blocks(name):
    """Full 900 000-byte blocks at -9 (sample5: 900000/900000/330640, the README size 272 997 B)."""
    from compressjs_b200 import BWTC
    d = T.fixture(name + ".ref")
    z = BWTC.compressFile(d, None, 9)
    assert z == O.bwtc_compress(d, 9)
    gold = T.golden().get("bwtc_%s_-9" % name)
    if gold:
        assert len(z) == gold["size"]
    assert BWTC.decompressFile(z) == d


@pytest.mark.parametrize("data", [b"", b"a", b"ab", b"\x00" * 5000, bytes(range(256)) * 9])
def test_bwtc_edges(data):
    from compressjs_b200 import BWTC
    for level in (1, 9):
        z = BWTC.compressFile(data, None, level)
        assert z == O.bwtc_compress(data, level)
        assert BWTC.decompressFile(z) == data


def test_bwtc_multi_block_and_errors():
    from compressjs_b200 import BWTC
    d = T.ascii_random(250001, 3) + T.runs(60000, 4) + T.texty(120000, 5)
    for level in (1, 2, 6):   # 430001 bytes: full and short blocks
        z = BWTC.compressFile(d, None, level)
        assert z == O.bwtc_compress(d, level)
        assert BWTC.decompressFile(z) == d
    assert BWTC.compressFile(d, None, 12) == O.bwtc_compress(d, 9)   # lib/BWTC.js:16-19
    with pytest.raises(ValueError):
        BWTC.decompressFile(b"bzzt" + b"\x81\x00\x00\x00")
