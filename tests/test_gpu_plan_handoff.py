"""The plan that b2_bzip2_plan, b2_bzip2_plan_spec and b2_bzip2_plan_share keep for the next
b2_bzip2_encode_range_dev (include/b2bz.h, "Plan cache"), encode_range with count == 0, and a b2_init after
b2_shutdown.  Whether a call cut blocks is read from its RLE1 walk counters (rle_walk_parallel + rle_walk_serial):
an encode_range that takes the cached plan cuts nothing.  Every fragment is compared with the oracle's stream, bit
for bit, through the oracle's block trace.  Each test runs in a child process, because the cache and the sharded
decode session live as long as the library's context."""
import os
import subprocess
import sys

import pytest

from tests import util as T

pytestmark = pytest.mark.gpu

_COMMON = r"""
import bz2, ctypes as C
import numpy as np, torch
from compressjs_b200 import _native, sharded as S
from oracle import oracle as O
from tests import util as T

L = _native.lib()
LEVEL = 1
DATA = T.texty(4 * 99981 + 555, 7)   # five level-1 blocks
N = len(DATA)
EXP, TR = O.bzip2_compress(DATA, LEVEL, trace=True)
EBITS = np.unpackbits(np.frombuffer(EXP, dtype=np.uint8))

def dev(b):
    d = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    torch.cuda.synchronize()
    return d

def cut():
    st = _native.stats()
    return st["rle_walk_parallel"] + st["rle_walk_serial"]

def ok(rc, what):
    assert rc == 0, "%s: %d %s" % (what, rc, _native.last_error())

def plan(d, n=N, level=LEVEL):
    total = C.c_size_t()
    ok(L.b2_bzip2_plan(d.data_ptr(), n, level, C.byref(total)), "plan")
    return total.value

def plan_spec(d, rank, world):
    info = (C.c_uint64 * 6)()
    ok(L.b2_bzip2_plan_spec(d.data_ptr(), N, LEVEL, rank, world, info), "plan_spec")
    return [int(v) for v in info]

def encode_rc(d, n, first, count, level=LEVEL):
    cap = count * 1400000 + 4096
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    bits, crcs = C.c_uint64(), (C.c_uint32 * max(count, 1))()
    rc = L.b2_bzip2_encode_range_dev(d.data_ptr(), n, level, first, count, 0, out.data_ptr(), cap, C.byref(bits), crcs)
    return rc, out, bits.value, list(crcs)[:count]

def encode(d, first, count, n=N, level=LEVEL):
    # blocks [first, first+count) of DATA: returns whether the call cut blocks; the fragment must be the oracle's
    rc, out, nbits, crcs = encode_rc(d, n, first, count, level)
    ok(rc, "encode_range")
    did_cut = cut() > 0
    if level == LEVEL:
        s = TR[first].bit_start
        e = s + sum(TR[k].bit_len for k in range(first, first + count))
        assert nbits == e - s, (first, count, nbits, e - s)
        got = np.unpackbits(out[:(nbits + 7) // 8].cpu().numpy())
        assert np.array_equal(got[:nbits], EBITS[s:e]), (first, count)
        assert not got[nbits:].any()
        assert crcs == [TR[k].crc for k in range(first, first + count)]
    return did_cut
"""


def _child(body):
    code = "import sys; sys.path.insert(0, %r)\n" % T.ROOT + _COMMON + body + "\nprint('ok')\n"
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout.split(), r.stdout[-3000:] + r.stderr[-5000:]


def test_cached_plan_is_taken_once_and_dropped_by_compress_dev():
    _child(r"""
d = dev(DATA)
assert plan(d) == len(TR) == 5
assert not encode(d, 0, 2)                      # takes the plan
assert encode(d, 2, 3)                          # the cache is empty: plans again
plan(d); assert encode(dev(DATA), 1, 2)         # another pointer
plan(d, N - 1000); assert encode(d, 1, 2)       # another length
plan(d, level=2); assert encode(d, 1, 2)        # another level
plan(d); assert encode(d, 1, 2, level=2)        # the other way round ...
assert encode(d, 1, 2)                          # ... which dropped the plan it did not take

# b2_bzip2_compress_dev in between drops the plan
plan(d)
cap = L.b2_bzip2_bound(N)
z, zn = torch.zeros(cap, dtype=torch.uint8, device="cuda"), C.c_size_t()
ok(L.b2_bzip2_compress_dev(d.data_ptr(), N, LEVEL, z.data_ptr(), cap, C.byref(zn)), "compress_dev")
assert bytes(z[:zn.value].cpu().numpy().tobytes()) == EXP
assert encode(d, 0, 5)

# b2_bzip2_share_summary and the host b2_bzip2_compress in between leave it
plan(d)
sm = (C.c_uint64 * 4)()
ok(L.b2_bzip2_share_summary(d.data_ptr(), N, sm), "share_summary")
o, on = C.POINTER(C.c_uint8)(), C.c_size_t()
ok(L.b2_bzip2_compress(DATA, N, LEVEL, C.byref(o), C.byref(on)), "compress")
assert C.string_at(o, on.value) == EXP
L.b2_free(o)
assert not encode(d, 0, 5)

# speculative range plans of a world of 4: each is taken by the encode_range that follows
infos = []
for r in range(4):
    info = plan_spec(d, r, 4)
    assert cut() > 0
    infos.append(info)
    assert not encode(d, info[2], info[4])
assert S.spec_plan_ok(infos, N)
# a range in front of the cached range plan is refused, and the plan is gone
plan_spec(d, 2, 4)
rc = encode_rc(d, N, 0, 1)[0]
assert rc == -101 and _native.last_error() == "block range is not covered by the cached range plan", rc
assert encode(d, 0, 1)

# share plans of a world of 2 (share + halo on each rank)
bufs, summaries = [], []
for r in range(2):
    g0, ln, hold = S.share_bounds(N, r, 2, 150000)
    bufs.append(dev(DATA[g0:g0 + hold]))
    sm = (C.c_uint64 * 4)()
    ok(L.b2_bzip2_share_summary(bufs[-1].data_ptr(), ln, sm), "share_summary")
    summaries.append(tuple(int(v) for v in sm))
inputs, total, _ = S.share_plan_inputs(summaries, LEVEL)
assert total == len(TR)
for r in range(2):
    b = bufs[r]
    st_in, w_in, first, count, g0 = inputs[r]
    info = (C.c_uint64 * 6)()
    ok(L.b2_bzip2_plan_share(b.data_ptr(), b.numel(), LEVEL, st_in, w_in, first, count, info), "plan_share")
    assert cut() > 0 and info[4] == count
    assert not encode(b, first, count, n=b.numel())
""")


def test_encode_range_of_no_blocks_writes_zero_bits():
    _child(r"""
d = dev(DATA)
plan(d)
for cap in (32, 4096):
    out = torch.full((cap,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    bits, crcs = C.c_uint64(0xDEADBEEF), (C.c_uint32 * 2)(0x5A5A5A5A, 0x5A5A5A5A)
    ok(L.b2_bzip2_encode_range_dev(d.data_ptr(), N, LEVEL, 1, 0, 3, out.data_ptr(), cap, C.byref(bits), crcs), "encode_range")
    assert bits.value == 0, hex(bits.value)
    assert list(crcs) == [0x5A5A5A5A] * 2
    assert not out.any()
    assert cut() == (0 if cap == 32 else 1)     # the first call takes the plan, the second plans exactly
# the argument checks of any other range
out = torch.zeros(64, dtype=torch.uint8, device="cuda")
bits = C.c_uint64(7)
assert L.b2_bzip2_encode_range_dev(d.data_ptr(), N, LEVEL, 0, 0, 0, out.data_ptr() + 1, 63, C.byref(bits), None) == -101
assert L.b2_bzip2_encode_range_dev(d.data_ptr(), N, LEVEL, 0, 0, 0, out.data_ptr(), 16, C.byref(bits), None) == -101
assert bits.value == 7
""")


def test_init_after_shutdown_starts_clean():
    _child(r"""
d = dev(DATA)
plan_spec(d, 1, 2)
other = T.ascii_random(2 * 99981 + 99, 8)
dz = dev(bz2.compress(other, 1))
S.decode_shard_rows(L, dz, 0, 1)
L.b2_shutdown()
ok(L.b2_init(0), "init")
assert encode(d, 0, 2)                          # the cached plan went with the old context
(total, lo, hi), rows = S.decode_shard_rows(L, dz, 0, 1)
o, res = S.decode_shard_finish(L, rows, False, dz.device)
assert o is not None, res
assert bytes(o.cpu().numpy().tobytes()) == other
""")
