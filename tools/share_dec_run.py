"""The sharded decode from sharded input (sharded.decompress_shares) against the whole-input one (decompress_file_sharded).

The input is the config-2 stream: uniform ASCII (tests/util.py ascii_random, the generator bench.py uses for config 2),
1 GiB by default, compressed once on the GPU at level 9.  Eight ranks are simulated on one GPU, as the GPU tests do:
every rank's session is opened and exported, the rows are concatenated, then every rank's session is opened again and
finished.  Per rank the tool prints the bytes it uploads (whole input: the stream; shares: its share and a halo of
sharded.DEC_HALO, the last rank's share only), the time of its open (scan, decode and export) and of its finish (walk,
expand and CRC check).  Each time is the host wall clock of one call, which ends in a device synchronise; one warm-up
round runs first.  The ranks' outputs are placed at their offsets and compared with the input, for both paths.

When the box has several GPUs, the same comparison then runs on real ranks (one process per GPU, NCCL): every rank
uploads its bytes and times the whole call of each path (decompress_file_sharded, decompress_shares), the decoded
stream assembled on rank 0, which checks it against the input.

The card's name and power limit, read in the same run, head the output.

    python tools/share_dec_run.py [GiB] [ranks]      (default 1 GiB, 8 simulated ranks)
"""
import json
import os
import socket
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()
    except Exception as e:
        return ["nvidia-smi failed: %r" % e]


def stream(gib):
    from compressjs_b200 import Bzip2
    from tests import util as T
    data = T.ascii_random(int(gib * (1 << 30)))
    return data, bytes(Bzip2.compressFile(data, None, 9))


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def simulated(z, data_dev, world):
    """Both paths with `world` ranks simulated on this GPU: per rank (bytes uploaded, open ms, finish ms); checks both
    outputs against the input."""
    from compressjs_b200 import sharded as S, _native
    L = _native.lib()
    n = len(z)
    host = torch.frombuffer(bytearray(z), dtype=torch.uint8).pin_memory()
    res = {}
    # whole input: every rank uploads the stream and scans all of it
    d_in = host.cuda()
    rows, t_open = [], []
    for r in range(world):
        (info, rw), ms = timed(lambda: S.decode_shard_rows(L, d_in, r, world))
        rows.append(rw)
        t_open.append(ms)
    all_rows = torch.cat(rows)
    pieces, t_fin = [], []
    for r in range(world):
        S.decode_shard_rows(L, d_in, r, world)
        (o, info), ms = timed(lambda: S.decode_shard_finish(L, all_rows, False, d_in.device))
        assert o is not None, info
        pieces.append((info["off"], o))
        t_fin.append(ms)
    res["whole_input"] = dict(uploaded=[n] * world, open_ms=t_open, finish_ms=t_fin, identical=placed(pieces, data_dev))
    del d_in, pieces
    # shares: every rank uploads its share and a halo, scans and decodes its own candidates
    g0s = [r * n // world for r in range(world)]
    lens = [(r + 1) * n // world - g0s[r] for r in range(world)]
    holds = [min(n - g0, ln + S.DEC_HALO) for g0, ln in zip(g0s, lens)]
    bufs = [host[g0: g0 + h].cuda() for g0, h in zip(g0s, holds)]
    rows, t_open = [], []
    for r in range(world):
        (rw, rc, msg), ms = timed(lambda: S._share_open(bufs[r], lens[r], g0s[r], n))
        assert rc == 0, msg
        rows.append(rw)
        t_open.append(ms)
    all_rows = torch.cat(rows)
    pieces, t_fin = [], []
    for r in range(world):
        S._share_open(bufs[r], lens[r], g0s[r], n)
        (o, info), ms = timed(lambda: S._share_finish(all_rows, rows[r], False, bufs[r].device))
        assert o is not None and not info["unsettled"], info
        pieces.append((info["off"], o))
        t_fin.append(ms)
    res["shares"] = dict(uploaded=holds, open_ms=t_open, finish_ms=t_fin, identical=placed(pieces, data_dev))
    return res


def placed(pieces, data_dev):
    out = torch.empty_like(data_dev)
    at = 0
    for off, p in sorted(pieces, key=lambda x: x[0]):
        if not p.numel():
            continue
        assert off == at, (off, at)
        out[off: off + p.numel()] = p
        at += p.numel()
    return at == data_dev.numel() and bool(torch.equal(out, data_dev))


def _rank(rank, world, port, z, data, q):
    import torch.distributed as dist
    from compressjs_b200 import sharded as S, _native
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    assert _native.lib().b2_init(rank) == 0, _native.last_error()
    dist.init_process_group("nccl", rank=rank, world_size=world)
    n = len(z)
    g0, g1 = rank * n // world, (rank + 1) * n // world
    hold = min(n, g1 + S.DEC_HALO) - g0
    host = torch.frombuffer(bytearray(z), dtype=torch.uint8)
    out = {}
    for rep in range(2):   # the first round is the warm-up
        d_in, t_up_whole = timed(lambda: host.cuda())
        full, t_whole = timed(lambda: S.decompress_file_sharded(d_in))
        ok_whole = rank != 0 or bytes(full.cpu().numpy().tobytes()) == data
        del d_in, full
        d_buf, t_up_share = timed(lambda: host[g0: g0 + hold].cuda())
        full, t_share = timed(lambda: S.decompress_shares(d_buf, g1 - g0))
        ok_share = rank != 0 or bytes(full.cpu().numpy().tobytes()) == data
        del d_buf, full
        out = dict(rank=rank, uploaded_whole=n, uploaded_shares=hold, upload_ms_whole=t_up_whole, upload_ms_shares=t_up_share,
                   call_ms_whole=t_whole, call_ms_shares=t_share, identical_whole=ok_whole, identical_shares=ok_share,
                   fallback=bool(S.PHASES.get("fallback_full_input")))
    q.put(out)
    dist.destroy_process_group()


def real_ranks(z, data, world):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, world, port, z, data, q)) for r in range(world)]
    for p in procs:
        p.start()
    rows = sorted((q.get(timeout=1800) for _ in range(world)), key=lambda x: x["rank"])
    for p in procs:
        p.join(timeout=120)
    return rows


def main():
    gib = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    world = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    if not torch.cuda.is_available():
        raise SystemExit("share_dec_run: no CUDA device")
    for line in card():
        print("card:", line)
    data, z = stream(gib)
    print("config-2 bytes: %d, level-9 stream: %d bytes" % (len(data), len(z)))
    data_dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    simulated(z, data_dev, world)   # warm-up
    res = simulated(z, data_dev, world)
    for path, r in res.items():
        print("%s (%d simulated ranks): output identical to the input: %s" % (path, world, r["identical"]))
        for k in range(world):
            print("  rank %d: uploaded %11d bytes, open %8.1f ms, finish %7.1f ms" % (k, r["uploaded"][k], r["open_ms"][k], r["finish_ms"][k]))
        print("  sum: uploaded %d bytes, open %.1f ms, finish %.1f ms; slowest rank: open %.1f ms, finish %.1f ms"
              % (sum(r["uploaded"]), sum(r["open_ms"]), sum(r["finish_ms"]), max(r["open_ms"]), max(r["finish_ms"])))
    print(json.dumps({"simulated_ranks": world, **res}))
    ngpu = torch.cuda.device_count()
    if ngpu > 1:
        del data_dev
        rows = real_ranks(z, data, ngpu)
        for r in rows:
            print(json.dumps(r))
    else:
        print("real ranks: not measured (%d GPU on this box)" % ngpu)


if __name__ == "__main__":
    main()
