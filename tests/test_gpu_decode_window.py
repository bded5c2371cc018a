"""The bzip2 decoder's input window ($B2_DEC_WINDOW) and decode batches ($B2_DEC_BATCH): one call holds only a window of
the compressed input and one batch of blocks on the device, so its device memory does not grow with the file.  Window
edges that fall inside a magic, a CRC, a header or the code tables, blocks longer than the window, and member headers
across window edges must not change a byte, an error code or a partial output.  Every check runs in a child process,
because the library reads the hooks per call but the tests share it."""
import os
import subprocess
import sys

import pytest

from tests import util as T

pytestmark = pytest.mark.gpu

MIB = 1 << 20
# include/b2bz.h: device bytes of one decode call for a window of W bytes and batches of B blocks
def peak_bound(W, B):
    return 2 * max(W, 48 * MIB) + B * 24 * MIB


def _child(code, env, timeout=1800):
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % T.ROOT + code],
                       env=dict(os.environ, **env), capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and "ok" in r.stdout.split(), r.stdout[-3000:] + r.stderr[-5000:]
    return r.stdout


# helpers of the child processes: the four single-GPU entry points on one stream, as bytes or the error code
_COMMON = r"""
import ctypes as C, os, bz2
import numpy as np, torch
from compressjs_b200 import Bzip2, Bzip2Error, _native
from oracle import oracle as O
from tests import util as T

def call(fn):
    try:
        return ("ok", fn())
    except Bzip2Error as e:
        return ("err", e.errorCode)

def table(z):
    rows = []
    r = call(lambda: Bzip2.table(z, lambda p, s: rows.append((p, s))))
    return r[0], rows

def dev(z, cap):
    L = _native.lib()
    d_in = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
    out = torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    n = C.c_size_t()
    rc = L.b2_bzip2_decompress_dev(d_in.data_ptr(), d_in.numel(), 0, out.data_ptr(), cap, C.byref(n))
    torch.cuda.synchronize()
    assert bool((out[cap:] == 0xA5).all())
    return ("err", rc) if rc else ("ok", out[:n.value].cpu().numpy().tobytes())

def all_four(z):
    st, rows = table(z)
    blocks = call(lambda: b"".join(Bzip2.decompressBlocks(z, [p for p, _ in rows]))) if st == "ok" else None
    return dict(file=call(lambda: bytes(Bzip2.decompressFile(z))), table=(st, rows), blocks=blocks)

def set_window(w):
    if w is None:
        os.environ.pop("B2_DEC_WINDOW", None)
    else:
        os.environ["B2_DEC_WINDOW"] = str(w)

def incompressible_stream():
    data = np.random.default_rng(7).integers(0, 256, 5 * 900000, dtype=np.uint8).tobytes()
    return data, bz2.compress(data, 9)
"""


def test_window_seams():
    """The first window ends at 12 byte offsets around the start of the first block past 1 MiB: in front of it, inside
    its magic and CRC, inside its header and code tables.  decompressFile, table, decompressBlocks over table's
    positions and b2_bzip2_decompress_dev must equal the default-window call and the oracle."""
    _child(_COMMON + r"""
data, z = incompressible_stream()
assert O.bzip2_decompress(z) == data
ref = all_four(z)
assert ref["file"] == ("ok", data)
rows = ref["table"][1]
assert ref["table"][0] == "ok" and sum(s for _, s in rows) == len(data) and len(rows) >= 5
assert ref["blocks"] == ("ok", data)
assert dev(z, len(data)) == ("ok", data)
start = next(p for p, _ in rows if p // 8 > (1 << 20)) // 8
for d in (-2, -1, 0, 1, 3, 5, 6, 8, 10, 14, 40, 300):
    set_window(start + d)
    assert all_four(z) == ref, d
    assert dev(z, len(data)) == ("ok", data), d
    assert dev(z, len(data) - 1) == ("err", -101), d
print("ok")
""", {})


def test_block_longer_than_the_window():
    """A 64 KiB window holds a sixteenth of one of these blocks: the window grows until the block fits."""
    _child(_COMMON + r"""
data, z = incompressible_stream()
set_window(64 << 10)
st, rows = table(z)
assert st == "ok" and sum(s for _, s in rows) == len(data)
assert all_four(z) == dict(file=("ok", data), table=("ok", rows), blocks=("ok", data))
assert dev(z, len(data)) == ("ok", data)
print("ok")
""", {})


@pytest.mark.parametrize("window", [64 << 10, 200000, 1 << 20])
def test_corpora_under_small_windows(window):
    """The synthetic corpus (every case, the multistream file, the relevelled blocks), the partial-output cases with the
    40-block seam file, libbz2 streams at levels 1, 5 and 9, and a file of many members whose headers fall across window
    edges, in windows of 64 KiB to 1 MiB and decode batches of 7 blocks, against the expectations they carry."""
    _child(_COMMON + r"""
from tests import synth_corpus as SC, partial_cases as P
import tests.test_gpu_decode_synthetic as TS
import tests.test_gpu_decode_partial as TP
for name in sorted(SC.CASES):
    TS.test_synthetic_case(name)
TS.test_synthetic_multistream()
TS.test_bound_is_the_only_check_that_fails()
for name in sorted(TP.FILES):
    TP.test_synthetic_case_partial(name)
exec(TP._SEAM_SCRIPT % {"root": T.ROOT})
data = T.runs(1300000, 61) + T.texty(900000, 62) + T.ascii_random(700000, 63)
for lv in (1, 5, 9):
    z = bz2.compress(data, lv)
    assert all_four(z) == dict(file=("ok", data), table=table(z), blocks=("ok", data)), lv
    assert dev(z, len(data)) == ("ok", data), lv
# many members: some header lands across every window edge; one window of each size of the sweep
parts = [T.ascii_random(500 + 37 * i, 100 + i) for i in range(120)]
cat = b"".join(bz2.compress(p, 1 + i % 9) for i, p in enumerate(parts))
whole = b"".join(parts)
w0 = int(os.environ["B2_DEC_WINDOW"])
for k in range(6):
    set_window(w0 + 29 * k)
    assert Bzip2.decompressFile(cat, None, True) == whole, k
    assert O.bzip2_decompress(cat, multistream=True) == whole
print("ok")
""", {"B2_DEC_WINDOW": str(window), "B2_DEC_BATCH": "7"}, timeout=3000)


def test_device_memory_does_not_grow_with_the_file():
    """16 MiB and 96 MiB of the same mixed content, 4 MiB windows, batches of 8 blocks: the same device high-water mark
    (within one batch's scratch) under the header's bound; the default window on the 96 MiB file needs more."""
    out = _child(_COMMON + r"""
def mixed(n):
    k = n // 3
    return (T.ascii_random(k, 11) + T.runs(k, 12) + T.texty(n - 2 * k, 13))
peaks = []
for mib in (16, 96):
    data = mixed(mib << 20)
    z = Bzip2.compressFile(data, None, 9)
    set_window(4 << 20)
    assert Bzip2.decompressFile(z) == data
    peaks.append(_native.stats()["dev_peak_bytes"])
set_window(None)
assert Bzip2.decompressFile(z) == data
peaks.append(_native.stats()["dev_peak_bytes"])
print("peaks", *peaks)
print("ok")
""", {"B2_DEC_BATCH": "8"})
    p16, p96, p96_default = [int(x) for x in out.split("peaks")[1].split()[:3]]
    assert 0 < p16 and 0 < p96
    assert abs(p96 - p16) <= 8 * 24 * MIB, (p16, p96)
    assert max(p16, p96) <= peak_bound(4 * MIB, 8), (p16, p96)
    assert p96_default > p96, (p96_default, p96)


def test_table_of_a_stream_larger_than_the_device():
    """Maximum-expansion blocks (46.6 MB each) until the decoded stream is larger than the device's memory: table lists
    every block; with one CRC broken near the end it fails there, after the rows in front of it."""
    _child(_COMMON + r"""
from tests import bz2synth as W, synth_corpus as SC, partial_cases as P
b = SC.max_expansion_block()
nb = torch.cuda.get_device_properties(0).total_memory // len(b.out) + 64
f = W.File(W.Member([b] * nb, 9))
st, rows = table(f.data)
assert st == "ok" and len(rows) == nb and all(s == len(b.out) for _, s in rows), (st, len(rows))
assert nb * len(b.out) > torch.cuda.get_device_properties(0).total_memory
k = nb - 3
bad = W.File(W.Member([b] * k + [P.with_crc(b, b.crc ^ 1)] + [b] * 2, 9))
st, rows2 = table(bad.data)
assert st == "err" and rows2 == rows[:k], (st, len(rows2))
print("ok")
""", {}, timeout=3000)
