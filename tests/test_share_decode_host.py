"""CPU tests (gloo, world 2 and 3) of the exchange in compressjs_b200/sharded.py's decompress_shares: the halo check and
every rank's share offset and stream length, the rows padded and gathered in rank order, the earliest error across
ranks, placement on rank 0 and the keep_sharded pieces, and the fallback to the whole input, which every rank takes
together.  The two library stages and the whole-input decode are replaced by a toy codec whose decode is the identity:
one row per byte of the share (bit position, kind 1, the byte), byte 0xEE / 0xED fail the decode with -5 / -2 at their
position, 0xFF leaves the stream unsettled (as a block that runs past its owner's halo does), and 0xEF fails the open."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from compressjs_b200 import sharded as S
from tests import util as T

ERRS = {0xEE: -5, 0xED: -2}


def _first_error(stream):
    for i, b in enumerate(stream):
        if b in ERRS:
            return i, ERRS[b]
    return None


def _fake_stages(calls):
    def open_stage(d_buf, share_len, g0, total):
        calls.append(("open", g0, total, d_buf.numel()))
        share = d_buf[:share_len].tolist()
        if 0xEF in share:
            return torch.zeros((0, S.SHARE_ROW), dtype=torch.int64), -200, "toy open failed"
        rows = torch.zeros((share_len, S.SHARE_ROW), dtype=torch.int64)
        for i, b in enumerate(share):
            rows[i, 0], rows[i, 1], rows[i, 2] = 8 * (g0 + i), 1, b
        return rows, 0, ""

    def finish_stage(all_rows, own_rows, multistream, device):
        pos = [int(p) // 8 for p in all_rows[:, 0].tolist()]
        calls.append(("rows", pos == list(range(len(pos))) and bool((all_rows[:, 1] == 1).all()) and bool((all_rows[:, 3:] == 0).all())))
        stream = bytes(all_rows[:, 2].tolist())
        own = own_rows[:, 2].to(torch.uint8)
        off = int(own_rows[0, 0]) // 8 if own_rows.shape[0] else 0
        res = dict(off=off, len=own.numel(), total=len(stream), err_idx=-1, err_code=0, msg="", unsettled=0xFF in stream)
        err = _first_error(stream)
        if err is not None and off <= err[0] < off + own.numel():   # the owner of the failing byte reports it
            res.update(err_idx=err[0], err_code=err[1], msg="toy error at %d" % err[0])
            return None, res
        return own, res

    def whole_stage(stream_t, multistream, group):
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        stream = bytes(stream_t.tolist())
        calls.append(("whole", stream))
        a, b = rank * len(stream) // world, (rank + 1) * len(stream) // world
        res = dict(off=a, len=b - a, total=len(stream), err_idx=-1, err_code=0, msg="")
        err = _first_error(stream)
        if err is not None and a <= err[0] < b:
            res.update(err_idx=err[0], err_code=err[1], msg="toy error")
            return None, res
        return stream_t[a:b].clone(), res

    return open_stage, finish_stage, whole_stage


def _cases(world):
    """(name, stream, share lengths, halo, expected): expected is ("ok", None), ("err", code) or ("raise", type)."""
    g = T.rng(40 + world)
    base = bytes(int(v) for v in g.integers(0, 0xE0, size=157))
    n = len(base)
    even = [(r + 1) * n // world - r * n // world for r in range(world)]
    uneven = [0] + [n // (world - 1)] * (world - 2) + [n - (n // (world - 1)) * (world - 2)]
    ends_short = [n - 3 * (world - 1)] + [3] * (world - 1)   # shares shorter than the minimum halo
    err_late, err_early = bytearray(base), bytearray(base)
    err_late[n - 5] = 0xEE                                    # owned by the last rank
    err_early[n - 5] = 0xEE
    err_early[even[0] + 2] = 0xED                             # owned by rank 1: earlier, wins
    unsettled, unsettled_err = bytearray(base), bytearray(base)
    unsettled[even[0] - 1] = 0xFF
    unsettled_err[1] = 0xFF
    unsettled_err[n - 1] = 0xEE
    bad_open = bytearray(base)
    bad_open[n - 2] = 0xEF
    return [
        ("even", base, even, S.DEC_HALO, ("ok", None)),
        ("uneven_with_empty_share", base, uneven, 20, ("ok", None)),
        ("minimum_halo", base, even, S.DEC_HALO_MIN, ("ok", None)),
        ("shares_shorter_than_the_halo", base, ends_short, S.DEC_HALO_MIN, ("ok", None)),
        ("error_on_the_last_rank", bytes(err_late), even, 30, ("err", -5)),
        ("earliest_error_wins", bytes(err_early), even, 30, ("err", -2)),
        ("fallback", bytes(unsettled), even, 30, ("ok", None)),
        ("fallback_then_error", bytes(unsettled_err), uneven, 30, ("err", -5)),
        ("halo_of_13", base, even, S.DEC_HALO_MIN - 1, ("raise", ValueError)),
        ("open_fails_on_one_rank", bytes(bad_open), even, 30, ("raise", RuntimeError)),
    ]


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from compressjs_b200.bzip2 import Bzip2Error
    for name, stream, lens, halo, exp in _cases(world):
        g0 = sum(lens[:rank])
        hold = min(len(stream) - g0, lens[rank] + halo)
        d_buf = torch.frombuffer(bytearray(stream[g0: g0 + hold]) or bytearray(1), dtype=torch.uint8)[:hold]
        for keep in (False, True):
            calls = []
            stages = _fake_stages(calls)
            try:
                got = S._decompress_shares(d_buf, lens[rank], False, None, keep, *stages)
                if keep:
                    got = ("piece", got.offset, got.total, bytes(got.piece.tolist()))
                else:
                    got = ("ok", None if got is None else bytes(got.tolist()))
            except Bzip2Error as e:
                got = ("err", e.errorCode)
            except (ValueError, RuntimeError) as e:
                got = ("raise", type(e).__name__)
            q.put((name, keep, rank, got, calls, bool(S.PHASES.get("fallback_full_input"))))
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("world", [2, 3])
def test_share_decode_exchange(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    cases = _cases(world)
    got = {}
    for _ in range(len(cases) * 2 * world):
        name, keep, rank, res, calls, fell_back = q.get(timeout=300)
        got[(name, keep, rank)] = (res, calls, fell_back)
    for p in procs:
        p.join(timeout=60)
    for name, stream, lens, halo, exp in cases:
        for keep in (False, True):
            res = [got[(name, keep, r)] for r in range(world)]
            if exp[0] == "raise":
                assert all(x[0] == ("raise", exp[1].__name__) for x in res), (name, keep, res)
                continue
            if exp[0] == "err":
                assert all(x[0] == exp for x in res), (name, keep, res)
            elif keep:
                pieces = sorted((x[0][1], x[0][3]) for x in res)
                assert all(x[0][2] == len(stream) for x in res), name
                assert b"".join(p for _, p in pieces) == stream and all(o == sum(len(p) for _, p in pieces[:i]) for i, (o, _) in enumerate(pieces)), name
            else:
                assert res[0][0] == ("ok", stream), name
                assert all(x[0] == ("ok", None) for x in res[1:]), name
            # every rank opened at its share's first byte, with the stream's length, and saw every row once in order
            for r, (_, calls, fell_back) in enumerate(res):
                g0 = sum(lens[:r])
                assert calls[0] == ("open", g0, len(stream), min(len(stream) - g0, lens[r] + halo)), (name, r, calls[0])
                assert calls[1] == ("rows", True), (name, r)
                # the fallback: every rank or none, and then from the whole stream
                fb = 0xFF in stream
                assert fell_back == fb, (name, r)
                assert (len(calls) == 3 and calls[2] == ("whole", stream)) if fb else len(calls) == 2, (name, r)


def test_share_layout():
    assert S.share_layout([(10, 24), (5, 14), (9, 9)]) == ([0, 10, 15], 24)
    assert S.share_layout([(0, 14), (0, 14), (20, 20)]) == ([0, 0, 0], 20)
    assert S.share_layout([]) == ([], 0)
    assert S.share_layout([(5, 5), (0, 0)]) == ([0, 5], 5)          # the halo may stop at the end of the stream
    for bad in ([(10, 23), (14, 14)],    # halo of 13
                [(10, 9), (5, 5)],       # holds less than its share
                [(10, 30), (5, 5)]):     # holds more than the stream
        with pytest.raises(ValueError):
            S.share_layout(bad)
    assert S.DEC_HALO == 4 << 20 and S.DEC_HALO_MIN == 14


def test_single_rank_without_a_process_group():
    stream = bytes(range(100))
    calls = []
    stages = _fake_stages(calls)
    d_buf = torch.frombuffer(bytearray(stream), dtype=torch.uint8)
    out = S._decompress_shares(d_buf, len(stream), False, None, False, *stages)
    assert bytes(out.tolist()) == stream
    piece = S._decompress_shares(d_buf, len(stream), False, None, True, *stages)
    assert (piece.offset, piece.total, bytes(piece.piece.tolist())) == (0, len(stream), stream)
