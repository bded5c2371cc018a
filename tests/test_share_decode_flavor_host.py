"""CPU tests (gloo, world 2 and 3) of the decoder flavor in compressjs_b200/sharded.py's multi-GPU decodes: the flavor
that decompress_shares and decompress_file_sharded are given reaches the open, finish and whole-input stages on every
rank, the fallback to the whole input included; ranks that ask for different flavors all raise ValueError; an unknown
flavor raises ValueError before any collective.  The library stages are replaced by the toy codec of
test_share_decode_host.py (share decode) and by an identity codec of one candidate per byte (whole-input decode)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from compressjs_b200 import _native
from compressjs_b200 import sharded as S
from tests import util as T
from tests.test_share_decode_host import _fake_stages


def _install(calls):
    """Replaces the library stages of both paths with toys that record the flavor they are given."""
    open_t, finish_t, _ = _fake_stages([])   # the fallback runs the real _decode_whole_input over the toys below

    def share_open(d_buf, share_len, g0, total, flavor="compressjs"):
        calls.append(("open", flavor))
        return open_t(d_buf, share_len, g0, total)

    def share_finish(all_rows, own_rows, multistream, device, flavor="compressjs"):
        calls.append(("finish", flavor))
        return finish_t(all_rows, own_rows, multistream, device)

    held = {}

    def shard_rows(L, d_in, rank, world, flavor="compressjs"):
        calls.append(("shard_rows", flavor))
        n = d_in.numel()
        held.update(d=d_in, lo=rank * n // world, hi=(rank + 1) * n // world)
        rows = torch.zeros((held["hi"] - held["lo"], 6), dtype=torch.int64)
        rows[:, 4] = 1
        return (n, held["lo"], held["hi"]), rows

    def shard_finish(L, all_rows, multistream, device, flavor="compressjs"):
        calls.append(("shard_finish", flavor, all_rows.shape[0]))
        lo, hi, d = held["lo"], held["hi"], held["d"]
        return d[lo:hi].clone(), dict(off=lo, len=hi - lo, total=d.numel(), err_idx=-1, err_code=0, msg="")

    S._share_open, S._share_finish = share_open, share_finish
    S.decode_shard_rows, S.decode_shard_finish = shard_rows, shard_finish
    _native.lib = lambda: None


def _count_collectives(counter):
    real = dist.all_gather

    def all_gather(*a, **k):
        counter[0] += 1
        return real(*a, **k)
    dist.all_gather = all_gather


def _run(fn):
    from compressjs_b200.bzip2 import Bzip2Error
    try:
        got = fn()
        return ("ok", None if got is None else bytes(got.tolist()))
    except Bzip2Error as e:
        return ("err", e.errorCode)
    except (ValueError, RuntimeError) as e:
        return ("raise", type(e).__name__)


def _cases(world):
    g = T.rng(70 + world)
    base = bytes(int(v) for v in g.integers(0, 0xE0, size=131))
    n = len(base)
    even = [(r + 1) * n // world - r * n // world for r in range(world)]
    unsettled = bytearray(base)
    unsettled[even[0] - 1] = 0xFF
    return base, bytes(unsettled), even


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    calls, coll = [], [0]
    _install(calls)
    _count_collectives(coll)
    base, unsettled, even = _cases(world)
    g0 = sum(even[:rank])

    def share_buf(stream):
        hold = min(len(stream) - g0, even[rank] + 30)
        return torch.frombuffer(bytearray(stream[g0: g0 + hold]), dtype=torch.uint8)

    def record(name, fn):
        del calls[:]
        c0 = coll[0]
        got = _run(fn)
        q.put((name, rank, got, list(calls), coll[0] - c0, bool(S.PHASES.get("fallback_full_input"))))

    for fl in ("compressjs", "libbz2"):
        record("shares_" + fl, lambda: S.decompress_shares(share_buf(base), even[rank], flavor=fl))
        record("fallback_" + fl, lambda: S.decompress_shares(share_buf(unsettled), even[rank], flavor=fl))
        record("whole_" + fl, lambda: S.decompress_file_sharded(torch.frombuffer(bytearray(base), dtype=torch.uint8), flavor=fl))
    mixed = "libbz2" if rank == 0 else "compressjs"
    record("shares_mixed", lambda: S.decompress_shares(share_buf(base), even[rank], flavor=mixed))
    record("whole_mixed", lambda: S.decompress_file_sharded(torch.frombuffer(bytearray(base), dtype=torch.uint8), flavor=mixed))
    # an unknown flavor: raised where it is given, before any collective (here on every rank, each on its own)
    record("shares_unknown", lambda: S.decompress_shares(share_buf(base), even[rank], flavor="bzip2"))
    record("whole_unknown", lambda: S.decompress_file_sharded(torch.frombuffer(bytearray(base), dtype=torch.uint8), flavor=None))
    record("private_unknown", lambda: S._decompress_shares(share_buf(base), even[rank], False, None, False, S._share_open,
                                                             S._share_finish, S._decode_whole_input, flavor="LIBBZ2"))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


NAMES = ["shares_compressjs", "fallback_compressjs", "whole_compressjs", "shares_libbz2", "fallback_libbz2", "whole_libbz2",
         "shares_mixed", "whole_mixed", "shares_unknown", "whole_unknown", "private_unknown"]


@pytest.mark.parametrize("world", [2, 3])
def test_flavor_reaches_every_stage(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(len(NAMES) * world):
        name, rank, res, calls, colls, fell_back = q.get(timeout=300)
        got[(name, rank)] = (res, calls, colls, fell_back)
    for p in procs:
        p.join(timeout=60)
    base, unsettled, _ = _cases(world)
    for fl in ("compressjs", "libbz2"):
        for name, stream, fb in (("shares_" + fl, base, False), ("fallback_" + fl, unsettled, True), ("whole_" + fl, base, False)):
            for r in range(world):
                res, calls, _, fell_back = got[(name, r)]
                assert res == ("ok", stream if r == 0 else None), (name, r, res)
                kinds = [c[0] for c in calls]
                if name.startswith("whole"):
                    assert kinds == ["shard_rows", "shard_finish"], (name, r, calls)
                else:
                    assert fell_back == fb, (name, r)
                    assert kinds == ["open", "finish"] + (["shard_rows", "shard_finish"] if fb else []), (name, r, calls)
                # every stage, the fallback's included, on every rank, in the flavor asked for
                assert all(c[1] == fl for c in calls), (name, r, calls)
    for name in ("shares_mixed", "whole_mixed"):
        for r in range(world):
            res, calls, colls, _ = got[(name, r)]
            assert res == ("raise", "ValueError"), (name, r, res)
            # the share path raises at its first exchange, before any rank opens its share
            assert calls == [] if name == "shares_mixed" else [c[0] for c in calls] == ["shard_rows"], (name, r, calls)
            assert colls == 1, (name, r, colls)
    for name in ("shares_unknown", "whole_unknown", "private_unknown"):
        for r in range(world):
            res, calls, colls, _ = got[(name, r)]
            assert (res, calls, colls) == (("raise", "ValueError"), [], 0), (name, r, res, calls, colls)


def test_unknown_flavor_without_a_process_group():
    d = torch.zeros(20, dtype=torch.uint8)
    for fn in (lambda: S.decompress_shares(d, 20, flavor="bz2"), lambda: S.decompress_file_sharded(d, flavor="bz2"),
               lambda: S.decode_shard_rows(None, d, 0, 1, flavor="bz2"), lambda: S._share_open(d, 20, 0, 20, flavor="bz2"),
               lambda: S._decode_whole_input(d, flavor="bz2")):
        with pytest.raises(ValueError):
            fn()
