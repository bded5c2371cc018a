"""GPU sharded decode from sharded input (b2_dec_share_open / _export / _finish, sharded.decompress_shares).  Ranks are
simulated on one GPU: every rank's session is opened and exported, then reopened before its finish, as
test_gpu_decode_synthetic.py does for the whole-input sharded decode.  Every rank gets only its bytes [g0, g0 + hold)
of the stream, copied to a buffer of its own.  Every result, decoded bytes or error code, must be Bzip2.decompressFile's
and the whole-input sharded decode's (decompress_file_sharded, which the share decode falls back to when its rows cannot
settle the stream).  The share edges sit on every byte of every block magic and its CRC, the byte behind it, every byte
of every end-of-stream magic, its CRC and the next member's header, and the last byte of the stream."""
import ctypes as C

import pytest
import torch

from tests import bz2synth as W
from tests import synth_corpus as SC
from tests import util as T

pytestmark = pytest.mark.gpu

BAD_ARG = -101


def _S():
    from compressjs_b200 import sharded as S
    return S


def _call(fn):
    from compressjs_b200 import Bzip2Error
    try:
        return ("ok", bytes(fn()))
    except Bzip2Error as e:
        return ("err", e.errorCode)


def _expect(data, multistream):
    from compressjs_b200 import Bzip2
    return _call(lambda: Bzip2.decompressFile(data, None, multistream))


def _whole(d, world, multistream):
    """The whole-input sharded decode with `world` simulated ranks: ("ok", bytes) or ("err", code of the earliest error)."""
    from compressjs_b200 import _native
    S, L = _S(), _native.lib()
    try:
        rows = [S.decode_shard_rows(L, d, r, world)[1] for r in range(world)]
    except RuntimeError as e:   # a bad first header fails every rank's open alike
        return ("err", int(str(e).rsplit("code ", 1)[1].rstrip(")")))
    all_rows = torch.cat(rows)
    parts, errs = [], []
    for r in range(world):
        S.decode_shard_rows(L, d, r, world)
        o, res = S.decode_shard_finish(L, all_rows, multistream, d.device)
        if o is None:
            errs.append((res["err_idx"], res["err_code"]))
        else:
            parts.append((res["off"], o.cpu().numpy().tobytes()))
    if errs:
        return ("err", min(errs)[1])
    return ("ok", b"".join(p for _, p in sorted(parts)))


def _shares(d, edges, halo, multistream):
    """The share decode of device stream d with share edges `edges` (byte offsets, one rank per share): (result,
    unsettled), result ("ok", bytes) or ("err", code), or None when the rows do not settle the stream."""
    S = _S()
    total = d.numel()
    bounds = [0] + sorted(edges) + [total]
    g0s, lens = bounds[:-1], [bounds[i + 1] - bounds[i] for i in range(len(bounds) - 1)]
    holds = [min(total - g0, ln + halo) for g0, ln in zip(g0s, lens)]
    S.share_layout(list(zip(lens, holds)))
    bufs = [d[g0: g0 + h].clone() for g0, h in zip(g0s, holds)]
    opened = []
    for r in range(len(lens)):
        rows, rc, msg = S._share_open(bufs[r], lens[r], g0s[r], total)
        assert rc == 0, msg
        opened.append(rows)
    all_rows = torch.cat(opened)
    pieces, errs, flags = [], [], []
    for r in range(len(lens)):
        again, rc, msg = S._share_open(bufs[r], lens[r], g0s[r], total)
        assert rc == 0 and torch.equal(again, opened[r]), msg
        o, res = S._share_finish(all_rows, opened[r], multistream, d.device)
        flags.append(res["unsettled"])
        if res["unsettled"]:
            continue
        if o is None:
            errs.append((res["err_idx"], res["err_code"]))
        else:
            assert res["total"] >= res["off"] + o.numel()
            pieces.append((res["off"], o.cpu().numpy().tobytes(), res["total"]))
    assert len(set(flags)) == 1, flags          # every rank sees the same rows: all fall back or none
    if flags[0]:
        return None, True
    if errs:
        return ("err", min(errs)[1]), False
    # the pieces (what keep_sharded returns on every rank) tile the decoded stream
    out, at = b"", 0
    for off, p, tot in sorted(pieces):
        assert off == at or not p, (off, at)
        out += p
        at += len(p)
    assert all(tot == len(out) for _, _, tot in pieces)
    return ("ok", out), False


def _edges(data, multistream):
    """The byte offsets a share edge must sit on."""
    bm, em = W.magic_positions(data)
    out = {len(data) - 1, len(data)}
    for p in bm:
        out.update(range(p // 8, (p + 80) // 8 + 1))            # the magic, its CRC and the block's first bit behind them
    for p in em:
        b = (p + 80 + 7) // 8
        out.update(range(p // 8, b + 5))                          # the magic, the stream CRC, the next member's header
    return sorted(e for e in out if 0 < e <= len(data))


def _groups(edges, k):
    return [edges[i: i + k] for i in range(0, len(edges), k)]


def _check(data, multistream, edge_sets, halo):
    """Every edge set (k edges: k + 1 ranks) against decompressFile and the whole-input sharded decode at k + 1 ranks."""
    exp = _expect(data, multistream)
    d = torch.frombuffer(bytearray(data) or bytearray(1), dtype=torch.uint8).cuda()[: len(data)]
    whole = {}
    fell_back = 0
    for edges in edge_sets:
        world = len(edges) + 1
        if world not in whole:
            whole[world] = _whole(d, world, multistream) if data else exp
            assert whole[world] == exp, world
        got, unsettled = _shares(d, edges, halo, multistream)
        fell_back += unsettled
        assert unsettled or got == exp, (edges, halo, got[0], exp[0])
    return fell_back


def _edge_sets(data, multistream):
    """World 1; world 2 at every edge; worlds 3 and 8 with their edges in runs of 2 and 7; empty shares and shares shorter
    than a block."""
    e = _edges(data, multistream)
    n = len(data)
    sets = [[]] + [[x] for x in e] + _groups(e, 2) + _groups(e, 7)
    sets += [[n // 2] * 7, [0] * 7, [n] * 7, [min(n, 3 * i + 1) for i in range(7)], [n * i // 8 for i in range(1, 8)]]
    return sets


@pytest.mark.parametrize("name", sorted(SC.CASES))
def test_synthetic_case(name):
    f = SC.build(name).file
    for ms in ((False, True) if len(f.members) > 1 else (False,)):
        _check(f.data, ms, _edge_sets(f.data, ms), _S().DEC_HALO)


def test_synthetic_multistream():
    f = SC.multistream_file()
    for ms in (False, True):
        _check(f.data, ms, _edge_sets(f.data, ms), _S().DEC_HALO)


@pytest.mark.parametrize("k", range(5))
def test_sample_fixture(k):
    z = T.fixture("sample%d.bz2" % k)
    for ms in (False, True):
        _check(z, ms, _edge_sets(z, ms), _S().DEC_HALO)


def test_minimum_halo_and_fallback():
    """A halo of 14 bytes: a share edge more than 14 bytes before the end of an on-chain block leaves the block open at its
    owner, and the rows must not settle the stream; an edge within 14 bytes of the block's end settles it.  Every result
    is still the stream's."""
    from oracle import oracle as O
    S = _S()
    data = T.texty(250000, 3)
    z, tr = O.bzip2_compress(data, 1, trace=True)
    d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
    assert _whole(d, 2, False) == ("ok", data)
    for t in tr:
        start, end = t.bit_start, t.bit_start + t.bit_len
        for e in (start // 8 + 1, start // 8 + 20, (end + 7) // 8 - 15):       # the block runs past e + 14
            assert _shares(d, [e], S.DEC_HALO_MIN, False) == (None, True), (start, e)
        for e in ((end + 7) // 8 - 14, (end + 7) // 8 - 5):                   # it ends inside the halo
            assert _shares(d, [e], S.DEC_HALO_MIN, False) == (("ok", data), False), (start, e)
        assert _shares(d, [start // 8 + 20], S.DEC_HALO, False) == (("ok", data), False)
    # the minimum halo on the synthetic corpus and the fixtures: whatever settles is the stream's
    fell = 0
    for f in [SC.build(n).file for n in sorted(SC.CASES)] + [SC.multistream_file()]:
        e = _edges(f.data, True)
        fell += _check(f.data, True, _groups(e, 2), S.DEC_HALO_MIN)
    for k in range(5):
        z = T.fixture("sample%d.bz2" % k)
        fell += _check(z, True, _groups(_edges(z, True), 2), S.DEC_HALO_MIN)
    assert fell


def test_halo_of_13_bytes():
    """Every rank whose buffer does not end the stream refuses a 13-byte halo at open; decompress_shares refuses it on
    every rank (it checks every rank's halo)."""
    from compressjs_b200 import Bzip2, _native
    S, L = _S(), _native.lib()
    data = T.texty(300000, 5)
    z = Bzip2.compressFile(data, None, 1)
    d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
    n, world = len(z), 3
    info = (C.c_uint64 * 3)()
    sizes = []
    for r in range(world):
        g0, ln = r * n // world, (r + 1) * n // world - r * n // world
        hold = min(n - g0, ln + S.DEC_HALO_MIN - 1)
        sizes.append((ln, hold))
        buf = d[g0: g0 + hold].clone()
        torch.cuda.synchronize()
        rc = L.b2_dec_share_open(buf.data_ptr(), hold, g0, ln, n, info)
        assert rc == (BAD_ARG if g0 + hold < n else 0), (r, rc)
    with pytest.raises(ValueError):
        S.share_layout(sizes)
    with pytest.raises(ValueError):
        S.decompress_shares(d[: n // 2].clone(), n // 3)   # one rank: its buffer must be its share


def test_one_rank_through_the_public_call():
    from compressjs_b200 import Bzip2, Bzip2Error
    S = _S()
    data = T.texty(700000, 8)
    z = Bzip2.compressFile(data, None, 2)
    d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
    assert bytes(S.decompress_shares(d, len(z)).cpu().numpy().tobytes()) == data
    piece = S.decompress_shares(d, len(z), keep_sharded=True)
    assert (piece.offset, piece.total, bytes(piece.piece.cpu().numpy().tobytes())) == (0, len(data), data)
    bad = bytearray(z)
    bad[len(z) // 2] ^= 0x10
    with pytest.raises(Bzip2Error) as ei:
        S.decompress_shares(torch.frombuffer(bad, dtype=torch.uint8).cuda(), len(z))
    assert ei.value.errorCode == _expect(bytes(bad), False)[1]


def _big_streams():
    """64 MiB of ascii_random, texty and runs: at level 1, at level 9, and as a file of one-block level-9 members."""
    from compressjs_b200 import Bzip2
    third = (64 << 20) // 3
    data = T.ascii_random(third, 31) + T.texty(third, 32) + T.runs((64 << 20) - 2 * third, 33)
    members = b"".join(Bzip2.compressFile(data[i: i + 899000], None, 9) for i in range(0, len(data), 899000))
    return data, [("level1", Bzip2.compressFile(data, None, 1), False), ("level9", Bzip2.compressFile(data, None, 9), False),
                  ("members", members, True)]


def test_64mib_streams():
    data, streams = _big_streams()
    S = _S()
    for name, z, ms in streams:
        bm, em = W.magic_positions(z)
        n = len(z)
        # even shares at 1, 2, 3 and 8 ranks; 8 ranks with their edges on every byte of some blocks' magics and CRCs and
        # of end-of-stream magics, CRCs and headers; the last byte; empty shares
        sets = [[r * n // w for r in range(1, w)] for w in (1, 2, 3, 8)]
        e = set()
        for p in bm[1:3] + bm[len(bm) // 2: len(bm) // 2 + 2] + bm[-2:]:
            e.update(range(p // 8, (p + 80) // 8 + 1))
        for p in em[:2] + em[-2:]:
            e.update(range(p // 8, (p + 87) // 8 + 5))
        e = sorted(x for x in e if 0 < x <= n)
        sets += _groups(e, 7) + [[n - 1], [n // 3] * 3 + [n - 1] * 4]
        exp = ("ok", data)
        assert _expect(z, ms) == exp, name
        d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
        for w in (2, 8):
            assert _whole(d, w, ms) == exp, (name, w)
        for edges in sets:
            got, unsettled = _shares(d, edges, S.DEC_HALO, ms)
            assert not unsettled and got == exp, (name, edges)
