"""The libbz2 decoder flavor in the multi-GPU decodes (b2_dec_shard_open_flavor, b2_dec_share_open_flavor,
sharded.decompress_file_sharded / decompress_shares with flavor="libbz2") and in the device-resident decode
(b2_bzip2_decompress_dev_flavor), against the model of tests/libbz2_read_cases.py, which tests/golden/libbz2_read.json
pins to libbz2.  Ranks are simulated on one GPU as in test_gpu_decode_shares.py.  Every case, multistream on and off:
the whole-input decode at 1, 2, 3 and 8 ranks and the device decode give the model's bytes or code; the share decode
gives the same with its edges on every byte of every magic, its CRC and what follows it, on the last 11 bytes of the
stream (every R4 cut), on a tail (R5), with empty shares and final shares shorter than 10 bytes, under the default and
the minimum halo (which must fall back to the whole input at least once), with and without the count-byte classes kept
(B2_DEC_KEEP_CLS=0: randomised blocks classified again at expansion) and across batch seams (B2_DEC_BATCH).  The
default flavor's rows are unchanged; two large streams decode at 8 ranks."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import bz2synth as W
from tests import libbz2_read_cases as LC
from tests import synth_corpus as SC
from tests import util as T

pytestmark = pytest.mark.gpu

NAMES = sorted(LC.CASES)
BAD_ARG = -101
LB = "libbz2"


def _S():
    from compressjs_b200 import sharded as S
    return S


def _lib():
    from compressjs_b200 import _native
    return _native.lib()


def _call(fn):
    from compressjs_b200 import Bzip2Error
    try:
        out = fn()
        return ("ok", None if out is None else bytes(out.cpu().numpy().tobytes()))
    except Bzip2Error as e:
        return ("err", e.errorCode)


def _exp(c, ms):
    e = c.expect(ms)
    return e[:2]


def _dev(d, n, ms):
    """b2_bzip2_decompress_dev_flavor: ("ok", bytes) or ("err", code); the size-only call agrees, and a buffer one byte
    short is B2_ERR_BAD_ARG with the size needed."""
    L = _lib()
    torch.cuda.synchronize()
    need = C.c_size_t(0)
    rc = L.b2_bzip2_decompress_dev_flavor(d.data_ptr(), n, int(ms), None, 0, C.byref(need), 1)
    # on an error the walk goes on past data errors for the size: 16 MiB holds every case's blocks
    out = torch.empty(max(need.value, 1) if rc == 0 else 16 << 20, dtype=torch.uint8, device="cuda")
    got = C.c_size_t(0)
    rc2 = L.b2_bzip2_decompress_dev_flavor(d.data_ptr(), n, int(ms), out.data_ptr(), out.numel(), C.byref(got), 1)
    assert rc2 == rc, (rc, rc2)
    if rc:
        return ("err", rc)
    assert got.value == need.value
    if need.value:
        short = C.c_size_t(0)
        assert L.b2_bzip2_decompress_dev_flavor(d.data_ptr(), n, int(ms), out.data_ptr(), need.value - 1, C.byref(short), 1) == BAD_ARG
        assert short.value == need.value
    return ("ok", bytes(out[: got.value].cpu().numpy().tobytes()))


def _whole(d, world, ms, flavor=LB):
    """The whole-input sharded decode with `world` simulated ranks: ("ok", bytes) or ("err", earliest code)."""
    S, L = _S(), _lib()
    try:
        rows = [S.decode_shard_rows(L, d, r, world, flavor)[1] for r in range(world)]
    except RuntimeError as e:   # a bad first header fails every rank's open alike
        return ("err", int(str(e).rsplit("code ", 1)[1].rstrip(")")))
    all_rows = torch.cat(rows)
    parts, errs = [], []
    for r in range(world):
        S.decode_shard_rows(L, d, r, world, flavor)
        o, res = S.decode_shard_finish(L, all_rows, ms, d.device, flavor)
        if o is None:
            errs.append((res["err_idx"], res["err_code"]))
        else:
            parts.append((res["off"], o.cpu().numpy().tobytes()))
    if errs:
        return ("err", min(errs)[1])
    return ("ok", b"".join(p for _, p in sorted(parts)))


def _shares(d, edges, halo, ms, flavor=LB):
    """The share decode of device stream d with share edges `edges`: (result, unsettled), result ("ok", bytes) or
    ("err", code), or None when the rows do not settle the stream."""
    S = _S()
    total = d.numel()
    bounds = [0] + sorted(edges) + [total]
    g0s, lens = bounds[:-1], [bounds[i + 1] - bounds[i] for i in range(len(bounds) - 1)]
    holds = [min(total - g0, ln + halo) for g0, ln in zip(g0s, lens)]
    S.share_layout(list(zip(lens, holds)))
    bufs = [d[g0: g0 + h].clone() for g0, h in zip(g0s, holds)]
    opened = []
    for r in range(len(lens)):
        rows, rc, msg = S._share_open(bufs[r], lens[r], g0s[r], total, flavor)
        assert rc == 0, msg
        opened.append(rows)
    all_rows = torch.cat(opened)
    if flavor == LB:
        # the stream's last bytes travel in rows of kind 3 from every rank whose buffer ends the stream
        ends = [r for r in range(len(lens)) if g0s[r] + holds[r] == total]
        k3 = [int((opened[r][:, 1] == 3).sum()) for r in range(len(lens))]
        assert k3 == [int(r in ends) for r in range(len(lens))], (k3, ends)
        assert max(int(opened[r][-1, 2]) for r in ends) == min(10, total)
    pieces, errs, flags = [], [], []
    for r in range(len(lens)):
        S._share_open(bufs[r], lens[r], g0s[r], total, flavor)
        o, res = S._share_finish(all_rows, opened[r], ms, d.device, flavor)
        flags.append(res["unsettled"])
        if res["unsettled"]:
            continue
        if o is None:
            errs.append((res["err_idx"], res["err_code"]))
        else:
            pieces.append((res["off"], o.cpu().numpy().tobytes(), res["total"]))
    assert len(set(flags)) == 1, flags          # every rank sees the same rows: all fall back or none
    if flags[0]:
        return None, True
    if errs:
        return ("err", min(errs)[1]), False
    out, at = b"", 0
    for off, p, tot in sorted(pieces):
        assert off == at or not p, (off, at)
        out += p
        at += len(p)
    assert all(tot == len(out) for _, _, tot in pieces)
    return ("ok", out), False


def _edges(c):
    """The byte offsets a share edge must sit on: every byte of every block magic, its CRC and the byte behind; every
    byte of every end-of-stream magic, its CRC and the 4 header bytes behind; the last 11 bytes of the stream (every R4
    cut) and its end; the first 64 bytes of a tail (R5)."""
    data, f = c.data, c.f
    n = len(data)
    out = set(range(n - 11, n + 1))
    off = 0
    for m in f.members:
        for p in m.block_pos:
            p += 8 * off
            out.update(range(p // 8, (p + 80) // 8 + 1))
        e = 8 * off + m.eos_pos
        out.update(range(e // 8, (e + 80 + 7) // 8 + 5))
        off += len(m.data)
    out.update(range(len(f.data), len(f.data) + 64))
    return sorted(x for x in out if 0 < x <= n)


def _groups(edges, k):
    return [edges[i: i + k] for i in range(0, len(edges), k)]


def _special(n):
    """Empty shares, and final shares shorter than 10 bytes."""
    cl = lambda xs: sorted(min(n, max(0, x)) for x in xs)
    return [cl([0] * 7), cl([n] * 7), cl([n // 2] * 3 + [n] * 4), cl([n - 9]), cl([n - 5, n - 1]), cl([n - 9, n - 8, n - 3, n - 3]),
            cl([n - 12, n - 9, n - 6, n - 3, n - 1, n, n])]


def _check(c, ms, sets, halo, worlds, d=None):
    """Every edge set against the model, and the whole-input decode at `worlds` and at every edge set's world; returns
    how many edge sets fell back."""
    exp = _exp(c, ms)
    if d is None:
        d = torch.frombuffer(bytearray(c.data), dtype=torch.uint8).cuda()
    whole = {}
    for w in sorted(set(worlds) | {len(e) + 1 for e in sets}):
        whole[w] = _whole(d, w, ms)
        assert whole[w] == exp, (w, whole[w][0], exp)
    fell = 0
    for edges in sets:
        got, unsettled = _shares(d, edges, halo, ms)
        fell += unsettled
        assert unsettled or got == exp, (edges, halo, got if got is None else got[0], exp[0])
    return fell


@pytest.mark.parametrize("name", NAMES)
def test_case(name):
    """Default halo: world 2 at every edge (with multistream; the edges are the same without it), 3 and 8 at runs of
    them, the special sets; the device decode; the public calls at one rank, which raise on an error and deliver
    nothing."""
    S = _S()
    c = LC.build(name)
    n = len(c.data)
    d = torch.frombuffer(bytearray(c.data), dtype=torch.uint8).cuda()
    e = _edges(c)
    for ms in (True, False):
        exp = _exp(c, ms)
        assert _dev(d, n, ms) == exp, (name, ms)
        assert _call(lambda: S.decompress_file_sharded(d, ms, flavor=LB)) == exp, (name, ms)
        assert _call(lambda: S.decompress_shares(d, n, ms, flavor=LB)) == exp, (name, ms)
        sets = ([[]] + [[x] for x in e] if ms else []) + _groups(e, 2) + _groups(e, 7) + _special(n)
        _check(c, ms, sets, S.DEC_HALO, (1, 2, 3, 8), d)


def test_minimum_halo():
    """The 14-byte halo over every case: whatever settles is the model's, and the rest falls back to the whole-input
    decode, which gives the model's result at that world."""
    S = _S()
    fell = 0
    for name in NAMES:
        c = LC.build(name)
        e = _edges(c)
        for ms in (True, False):
            fell += _check(c, ms, _groups(e, 2) + _groups(e, 7) + _special(len(c.data)), S.DEC_HALO_MIN, ())
    assert fell


@pytest.mark.parametrize("env", [dict(B2_DEC_KEEP_CLS="0"), dict(B2_DEC_BATCH="1"), dict(B2_DEC_BATCH="7")],
                         ids=["keep_cls_0", "batch_1", "batch_7"])
def test_classes_dropped_and_batch_seams(env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    S = _S()
    fell = 0
    for name in NAMES:
        c = LC.build(name)
        n = len(c.data)
        d = torch.frombuffer(bytearray(c.data), dtype=torch.uint8).cuda()
        e = _edges(c)
        for ms in (True, False):
            assert _dev(d, n, ms) == _exp(c, ms), (name, ms)
            sets = _groups(e, 7) + _special(n)
            _check(c, ms, sets, S.DEC_HALO, (1, 2, 3), d)
            if ms:
                fell += _check(c, ms, sets, S.DEC_HALO_MIN, (), d)
    assert fell


def _raw_rows_shard(d, world, flavor):
    L = _lib()
    out = []
    for r in range(world):
        info = (C.c_uint64 * 3)()
        torch.cuda.synchronize()
        rc = (L.b2_dec_shard_open(d.data_ptr(), d.numel(), r, world, info) if flavor is None
              else L.b2_dec_shard_open_flavor(d.data_ptr(), d.numel(), r, world, info, flavor))
        if rc:
            out.append(rc)
            continue
        k = int(info[2]) - int(info[1])
        buf = (C.c_uint64 * (6 * max(k, 1)))()
        assert L.b2_dec_shard_export(buf) == 0
        rows = np.array(buf[: 6 * k], dtype=np.uint64).reshape(-1, 6)
        rows[rows[:, 0] == np.uint64(2 ** 64 - 7), 5] = 0   # an obsolete block's decode stops before origPtr: no value
        out.append((tuple(info), rows.tobytes()))
    return out


def _raw_rows_share(d, edges, flavor):
    L = _lib()
    total = d.numel()
    bounds = [0] + sorted(edges) + [total]
    out = []
    for g0, g1 in zip(bounds[:-1], bounds[1:]):
        hold = min(total - g0, g1 - g0 + _S().DEC_HALO)
        buf_in = d[g0: g0 + hold].clone()
        torch.cuda.synchronize()
        info = (C.c_uint64 * 3)()
        rc = (L.b2_dec_share_open(buf_in.data_ptr(), hold, g0, g1 - g0, total, info) if flavor is None
              else L.b2_dec_share_open_flavor(buf_in.data_ptr(), hold, g0, g1 - g0, total, info, flavor))
        assert rc == 0
        buf = (C.c_uint64 * (11 * max(int(info[0]), 1)))()
        assert L.b2_dec_share_export(buf) == 0
        out.append((tuple(info), tuple(buf[: 11 * int(info[0])])))
    return out


def test_default_flavor_rows_unchanged():
    """The open calls without a flavor and the _flavor opens with B2_BZ2_COMPRESSJS export the same rows, word for word,
    for the synthetic corpus and the sample*.bz2 fixtures (no run-of-four bit, no row of kind 3)."""
    streams = [SC.build(n).file.data for n in sorted(SC.CASES)] + [SC.multistream_file().data]
    streams += [T.fixture("sample%d.bz2" % k) for k in range(5)]
    for z in streams:
        if not z:
            continue
        d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
        n = len(z)
        for world in (1, 3):
            assert _raw_rows_shard(d, world, None) == _raw_rows_shard(d, world, 0)
        bm, em = W.magic_positions(z)
        for edges in ([], [n // 3, 2 * n // 3], sorted(min(n, p // 8 + 1) for p in (bm + em)[:7]), [n - 5]):
            old = _raw_rows_share(d, edges, None)
            assert old == _raw_rows_share(d, edges, 0)
            assert all(rows[1 + 11 * i] != 3 for _, rows in old for i in range(len(rows) // 11))


def test_unknown_flavor_is_bad_arg():
    L = _lib()
    z = bytes(LC.build("rand_short").data)
    d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
    torch.cuda.synchronize()
    info = (C.c_uint64 * 3)()
    n_out = C.c_size_t(0)
    out = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    for fl in (2, -1, 7):
        assert L.b2_dec_shard_open_flavor(d.data_ptr(), len(z), 0, 1, info, fl) == BAD_ARG
        assert L.b2_dec_share_open_flavor(d.data_ptr(), len(z), 0, len(z), len(z), info, fl) == BAD_ARG
        assert L.b2_bzip2_decompress_dev_flavor(d.data_ptr(), len(z), 1, out.data_ptr(), out.numel(), C.byref(n_out), fl) == BAD_ARG
    with pytest.raises(ValueError):
        _S().decompress_shares(d, len(z), flavor="bzip2")


def _even(n, world):
    return [r * n // world for r in range(1, world)]


def test_scale_256mib_randomised_members_on_8_ranks():
    """The file of test_gpu_libbz2_decode.py's 256 MiB scale test: one randomised 900 000-byte block per member."""
    members, outs = [], []
    for s in range(3):
        P = np.frombuffer(T.ascii_random(900000, 500 + s), np.uint8)
        members.append(W.Member([LC.rand_block(P)], 9).data)
        outs.append(W.model_rle1(P)[0].tobytes())
    k = (256 << 20) // 900000
    data = b"".join(members[i % 3] for i in range(k))
    exp = ("ok", b"".join(outs[i % 3] for i in range(k)))
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    assert _shares(d, _even(len(data), 8), _S().DEC_HALO, True) == (exp, False)
    assert _whole(d, 8, True) == exp


def test_scale_64mib_libbz2_stream_with_zero_padding_on_8_ranks():
    """A 64 MiB stream of the libbz2-flavor encoder followed by 1 MiB of zeros, which bzip2 -d ignores."""
    from compressjs_b200 import Bzip2
    half = 32 << 20
    data = T.ascii_random(half, 41) + T.runs(half, 42)
    z = bytes(Bzip2.compressFile(data, None, 9, flavor=LB)) + b"\0" * (1 << 20)
    d = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
    assert _shares(d, _even(len(z), 8), _S().DEC_HALO, True) == (("ok", data), False)
    assert _whole(d, 8, True) == ("ok", data)
