"""GPU: the libbz2 flavor of the multi-GPU encode with simulated ranks in one process.  Every rank cuts its share for
every entry drift (b2_bzip2_share_cut_table), the tables are chained on the host (sharded.libbz2_share_chain), and
each rank plans and range-encodes its blocks (b2_bzip2_plan_share_flavor, b2_bzip2_encode_range_dev_flavor): the
assembled stream must be bz2.compress's, byte for byte."""
import bz2
import ctypes as C

import numpy as np
import pytest
import torch

from tests import libbz2_model as M
from tests import util as T
from tests.test_libbz2_model import _libbz2_ok
from tests.test_libbz2_shares import KINDS, even_bounds, max_drift, pieces, random_bounds, w_at

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not _libbz2_ok(), reason="bz2 is not linked against libbz2 1.0.3 or later")]
LIBBZ2 = 1


def _lib():
    from compressjs_b200 import _native
    return _native.lib(), _native


def _table(L, d, share_len, level, st_in, w_in, dmax):
    tab = (C.c_uint32 * (4 * (dmax + 1)))()
    assert L.b2_bzip2_share_cut_table(d.data_ptr(), d.numel(), level, st_in, w_in, share_len, dmax, tab) == 0, _lib()[1].last_error()
    return [tuple(int(x) for x in r) for r in np.frombuffer(tab, dtype=np.uint32).reshape(-1, 4)]


def _simulate(data, bounds, level, halo):
    """Ranks holding data[a:b] + halo: returns (stream or None when the chain is refused, block starts per rank)."""
    from compressjs_b200 import sharded as S
    L, nat = _lib()
    n = len(data)
    bufs, summaries = [], []
    for a, b in bounds:
        hold = min(n, b + halo) - a
        d = torch.frombuffer(bytearray(data[a:a + hold]) + bytearray(1), dtype=torch.uint8)[:hold].cuda()
        sm = (C.c_uint64 * 4)()
        assert L.b2_bzip2_share_summary(d.data_ptr(), b - a, sm) == 0, nat.last_error()
        bufs.append(d)
        summaries.append(tuple(int(v) for v in sm))
    ins, _, w_total = S.share_plan_inputs(summaries, level)
    tables = [(_table(L, bufs[r], b - a, level, ins[r][0], ins[r][1], S.share_drift_bound(ins[r][1], level)) if b > a else None)
              for r, (a, b) in enumerate(bounds)]
    ends = [a + bufs[r].numel() == n for r, (a, _) in enumerate(bounds)]
    chain = S.libbz2_share_chain(ins, w_total, tables, level, ends)
    if chain is None:
        return None, None
    res, total = chain
    frags, bits, crcs, starts = [], [], [], []
    for r, (a, b) in enumerate(bounds):
        first, drift, count = res[r]
        d = bufs[r]
        info = (C.c_uint64 * 6)()
        assert L.b2_bzip2_plan_share_flavor(d.data_ptr(), d.numel(), level, ins[r][0], ins[r][1], first, count, drift, LIBBZ2, info) == 0, \
            nat.last_error()
        assert int(info[4]) == count and int(info[3]) == count
        f, nb, cr = S._range_encoder(L, d, d.numel(), level, "libbz2")(first, count)
        starts.append([a + t.raw_start for t in nat.last_trace()] if count else [])
        frags.append(f); bits.append(nb); crcs.append(cr)
    sh, o = [], 32
    for f, nb in zip(frags, bits):
        sh.append(S.shift_right_bits(f, nb, o % 8))
        o += nb
    out = S.assemble(level, sh, bits, crcs, frags[0].device)
    return bytes(out.cpu().numpy().tobytes()), starts


def _inputs():
    return {"ascii": T.ascii_random(6 * 99981 + 333, 3), "text": T.texty(6 * 99981 + 777, 4),
            "runs": KINDS["runs"](4000000, 5), "maxdrift": max_drift(12 * 99981 + 11)}


@pytest.mark.parametrize("kind", ["ascii", "text", "runs", "maxdrift"])
def test_world1_table_walk_equals_the_single_gpu_cut(kind):
    """Entry (0, 0) on one rank: the table's row 0 and the share plan cut exactly the blocks of the single-GPU libbz2
    walk (b2_last_trace of b2_bzip2_compress_dev_flavor)."""
    from compressjs_b200 import sharded as S
    L, nat = _lib()
    data = _inputs()[kind]
    level = 1
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    out = torch.empty(L.b2_bzip2_bound(len(data)), dtype=torch.uint8, device="cuda")
    on = C.c_size_t()
    assert L.b2_bzip2_compress_dev_flavor(d.data_ptr(), len(data), level, out.data_ptr(), out.numel(), C.byref(on), LIBBZ2) == 0
    ref = [(t.raw_start, t.raw_len, t.n) for t in nat.last_trace()]
    assert [(s, ln, len(b)) for s, ln, b in M.cut(data, level)] == ref
    rows = _table(L, d, len(data), level, 0, 0, 0)
    assert rows[0][0] == 0 and rows[0][1] == len(ref) and rows[0][3] & S.CUT_BUF_END
    info = (C.c_uint64 * 6)()
    assert L.b2_bzip2_plan_share_flavor(d.data_ptr(), len(data), level, 0, 0, 0, len(ref), 0, LIBBZ2, info) == 0
    assert [int(v) for v in info[:5]] == [0, len(data), 0, len(ref), len(ref)]
    f, nb, cr = S._range_encoder(L, d, len(data), level, "libbz2")(0, len(ref))
    assert [(t.raw_start, t.raw_len, t.n) for t in nat.last_trace()] == ref
    z = bytes(S.assemble(level, [f], [nb], [cr], d.device).cpu().numpy().tobytes())
    assert z == bytes(out[: on.value].cpu().numpy().tobytes()) == bz2.compress(data, level)


@pytest.mark.parametrize("level", [1, 9])
@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("kind", ["ascii", "text", "runs", "maxdrift"])
def test_shares_assemble_to_libbz2_bytes(kind, world, level):
    from compressjs_b200 import Bzip2
    data = _inputs()[kind] if level == 1 else KINDS[kind](3 * 899981 + 55, 6) if kind != "runs" else KINDS["runs"](12000000, 6)
    exp = bz2.compress(data, level)
    ref = [s for s, _, _ in M.cut(data, level)]
    for bounds in (even_bounds(len(data), world), random_bounds(len(data), world, T.rng(world + level))):
        z, starts = _simulate(data, bounds, level, len(data))
        assert z == exp
        assert sum(starts, []) == ref
        assert bytes(Bzip2.decompressFile(z)) == data


@pytest.mark.parametrize("level", [1, 9])
def test_seams_edges_short_and_empty_shares(level):
    from compressjs_b200 import Bzip2
    data = T.texty((6 * 99981 if level == 1 else 3 * 899981) + 999, 12)
    n = len(data)
    exp = bz2.compress(data, level)
    ref = M.cut(data, level)
    P = pieces(data)
    cases = [[(0, 0), (0, 5000), (5000, 5000), (5000, 80000), (80000, n)],
             [(0, n - 10), (n - 10, n - 3), (n - 3, n), (n, n)]]
    s2 = ref[2][0]
    for j in range(6):                   # share W starts 0..5 past the start of block 2 (the two-index edge)
        x = s2
        while x < n and w_at(P, x) < w_at(P, s2) + j:
            x += 1
        cases.append([(0, x // 3), (x // 3, x), (x, n)])
    runs = bytearray(data)               # a run straddling every seam
    bounds = even_bounds(n, 3)
    for a, _ in bounds[1:]:
        runs[a - 300: a + 700] = b"q" * 1000
    for bounds in cases:
        z, _ = _simulate(data, bounds, level, n)
        assert z == exp, bounds
    z, _ = _simulate(bytes(runs), bounds, level, n)
    assert z == bz2.compress(bytes(runs), level)
    assert bytes(Bzip2.decompressFile(z)) == bytes(runs)


def test_compress_file_sharded_single_rank_libbz2():
    from compressjs_b200 import sharded as S
    data = T.ascii_random(3 * 899981 // 2, 4)
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    assert bytes(S.compress_file_sharded(d, 9, flavor="libbz2").cpu().numpy().tobytes()) == bz2.compress(data, 9)
    assert bytes(S.compress_shares(d, len(data), 9, flavor="libbz2").cpu().numpy().tobytes()) == bz2.compress(data, 9)


def test_range_encode_never_takes_the_other_flavors_plan():
    """A libbz2 range encode after a compressjs plan of the same buffer (and the reverse) replans in its own flavor."""
    from compressjs_b200 import sharded as S
    from oracle import oracle as O
    L, nat = _lib()
    data = KINDS["maxdrift"](5 * 99981, 0) + T.texty(2 * 99981, 3)
    level = 1
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    for plan_flavor, enc_flavor, exp in ((0, "libbz2", bz2.compress(data, level)), (1, "compressjs", O.bzip2_compress(data, level))):
        total = C.c_size_t()
        assert L.b2_bzip2_plan_flavor(d.data_ptr(), len(data), level, C.byref(total), plan_flavor) == 0
        nb = len(M.cut(data, level)) if enc_flavor == "libbz2" else len(O.bzip2_compress(data, level, trace=True)[1])
        f, bits, cr = S._range_encoder(L, d, len(data), level, enc_flavor)(0, nb)
        assert bytes(S.assemble(level, [f], [bits], [cr], d.device).cpu().numpy().tobytes()) == exp


def test_short_halo_takes_the_fallback():
    """A halo shorter than a block of long runs: the chain is refused, and the fallback compress_shares takes (every
    rank gets the whole input and the exact plan) still writes libbz2's bytes."""
    from compressjs_b200 import sharded as S
    data = KINDS["runs"](3000000, 7)
    z, _ = _simulate(data, even_bounds(len(data), 3), 1, 20000)
    assert z is None
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    assert bytes(S.compress_file_sharded(d, 1, flavor="libbz2").cpu().numpy().tobytes()) == bz2.compress(data, 1)
    z, _ = _simulate(data, even_bounds(len(data), 3), 1, len(data))
    assert z == bz2.compress(data, 1)


def test_unknown_flavor_is_rejected():
    L, nat = _lib()
    d = torch.frombuffer(bytearray(T.texty(5000, 1)), dtype=torch.uint8).cuda()
    total = C.c_size_t()
    assert L.b2_bzip2_plan_flavor(d.data_ptr(), d.numel(), 1, C.byref(total), 7) == -101
    info = (C.c_uint64 * 6)()
    assert L.b2_bzip2_plan_share_flavor(d.data_ptr(), d.numel(), 1, 0, 0, 0, 1, 0, 2, info) == -101
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    bits = C.c_uint64()
    crcs = (C.c_uint32 * 4)()
    assert L.b2_bzip2_encode_range_dev_flavor(d.data_ptr(), d.numel(), 1, 0, 1, 0, out.data_ptr(), out.numel(), C.byref(bits), crcs, -1) == -101
    tab = (C.c_uint32 * 4)()
    assert L.b2_bzip2_share_cut_table(d.data_ptr(), d.numel(), 1, 0, 0, d.numel() + 1, 0, tab) == -101   # share past the buffer
