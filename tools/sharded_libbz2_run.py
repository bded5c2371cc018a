"""Cost of the libbz2 flavor's sharded encode: simulates the ranks of an 8 x 1 GiB config-2 job on one GPU (rank r's
share is bench.py's gen_ascii(1 GiB, SEED + r), followed by a 4 MiB halo of the next share, as bench.py holds them).
All eight share summaries are computed first; then, per rank, the cut table (b2_bzip2_share_cut_table), the share
plan (b2_bzip2_plan_share_flavor) and the range encode (b2_bzip2_encode_range_dev_flavor) are timed with CUDA events
around each call (the share plan reuses the scan and piece bitmap of the table call before it); the host side of the
table exchange (the gathered tables from the device and the chain) is timed with a wall clock; and for the last rank the compressjs flavor's share plan and range encode beside them.  The
assembled stream is compared with b2_bzip2_compress_dev_flavor of the concatenated input (its SHA-256 is reported),
and a 64 MiB prefix with bz2.compress.  Prints one JSON line (also written to DIR/sharded_libbz2_run.json with --out).

    python tools/sharded_libbz2_run.py [--world 8] [--mib 1024] [--out DIR]
"""
import argparse
import bz2
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    rc = fn()
    b.record()
    b.synchronize()
    return rc, a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--halo-mib", type=int, default=4)
    ap.add_argument("--check-mib", type=int, default=64)
    ap.add_argument("--level", type=int, default=9)
    ap.add_argument("--out")
    a = ap.parse_args()
    import numpy as np
    import torch
    from bench import SEED, gen_ascii
    from compressjs_b200 import _native, sharded as S
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    L = _native.lib()
    level, world, shard, halo = a.level, a.world, a.mib << 20, a.halo_mib << 20

    def err(name):
        raise RuntimeError(name + ": " + _native.last_error())

    full = torch.empty(world * shard, dtype=torch.uint8, device="cuda")
    for r in range(world):
        full[r * shard:(r + 1) * shard] = torch.from_numpy(gen_ascii(shard, SEED + r)).cuda()
    torch.cuda.synchronize()
    bufs = [full[r * shard: min(world * shard, (r + 1) * shard + halo)] for r in range(world)]   # share + halo
    summaries = []
    for r in range(world):
        sm = (C.c_uint64 * 4)()
        if L.b2_bzip2_share_summary(bufs[r].data_ptr(), shard, sm):
            err("b2_bzip2_share_summary")
        summaries.append(tuple(int(v) for v in sm))
    ins, _, w_total = S.share_plan_inputs(summaries, level)
    tables, ranks = [], []
    warm = (C.c_uint32 * 4)()   # the first call of the process sets up the library: keep it out of the timings
    L.b2_bzip2_share_cut_table(bufs[0].data_ptr(), bufs[0].numel(), level, ins[0][0], ins[0][1], shard, 0, warm)
    for r in range(world):
        dmax = S.share_drift_bound(ins[r][1], level)
        tab = (C.c_uint32 * (4 * (dmax + 1)))()
        rc, ms = timed(lambda: L.b2_bzip2_share_cut_table(bufs[r].data_ptr(), bufs[r].numel(), level, ins[r][0], ins[r][1], shard, dmax, tab))
        if rc:
            err("b2_bzip2_share_cut_table")
        tables.append(np.frombuffer(tab, dtype=np.int32).reshape(-1, 4).copy())
        ranks.append({"rank": r, "candidates": dmax + 1, "table_bytes": 16 * (dmax + 1), "ms_table": round(ms, 3)})
    # the host side of the exchange on every rank: the all-gathered tables (padded to the longest, as compress_shares
    # sends them) come back from the device and are chained
    longest = max(t.shape[0] for t in tables)
    gathered = torch.zeros((world, longest, 4), dtype=torch.int32, device="cuda")
    for r, t in enumerate(tables):
        gathered[r, : t.shape[0]] = torch.from_numpy(t).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host = [gathered[r][: tables[r].shape[0]].cpu().numpy() for r in range(world)]
    chain = S.libbz2_share_chain(ins, w_total, host, level, [r == world - 1 for r in range(world)])
    ms_chain = (time.perf_counter() - t0) * 1e3
    del gathered
    if chain is None:
        raise SystemExit("the chain was refused: the halo is too short for this input")
    res, total = chain
    frags, bits, crcs = [], [], []
    for r in range(world):
        first, drift, count = res[r]
        # as on rank r of compress_shares, the share plan follows the rank's own table call and takes over its scan and
        # piece bitmap (the table is rebuilt here, untimed, because the loop above ran every rank's table first)
        dmax = S.share_drift_bound(ins[r][1], level)
        tab = (C.c_uint32 * (4 * (dmax + 1)))()
        L.b2_bzip2_share_cut_table(bufs[r].data_ptr(), bufs[r].numel(), level, ins[r][0], ins[r][1], shard, dmax, tab)
        info = (C.c_uint64 * 6)()
        rc, ms_plan = timed(lambda: L.b2_bzip2_plan_share_flavor(bufs[r].data_ptr(), bufs[r].numel(), level, ins[r][0], ins[r][1], first, count,
                                                                  drift, 1, info))
        if rc or int(info[4]) != count:
            err("b2_bzip2_plan_share_flavor")
        cap = count * 1400000 + 4096
        out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        nb = C.c_uint64()
        cr = (C.c_uint32 * max(count, 1))()
        rc, ms_enc = timed(lambda: L.b2_bzip2_encode_range_dev_flavor(bufs[r].data_ptr(), bufs[r].numel(), level, first, count, 0, out.data_ptr(),
                                                                       cap, C.byref(nb), cr, 1))
        if rc:
            err("b2_bzip2_encode_range_dev_flavor")
        frags.append(out); bits.append(int(nb.value)); crcs.append(list(cr)[:count])
        ranks[r].update({"first": first, "drift": drift, "blocks": count, "ms_plan": round(ms_plan, 3), "ms_encode": round(ms_enc, 3)})
    # the compressjs flavor's share path of the last rank, beside it
    r = world - 1
    cj_ins, cj_total, _ = S.share_plan_inputs(summaries, level)
    info = (C.c_uint64 * 6)()
    rc, cj_plan = timed(lambda: L.b2_bzip2_plan_share(bufs[r].data_ptr(), bufs[r].numel(), level, cj_ins[r][0], cj_ins[r][1], cj_ins[r][2],
                                                       cj_ins[r][3], info))
    cnt = int(info[4])
    cap = cnt * 1400000 + 4096
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    nb = C.c_uint64()
    cr = (C.c_uint32 * max(cnt, 1))()
    rc2, cj_enc = timed(lambda: L.b2_bzip2_encode_range_dev(bufs[r].data_ptr(), bufs[r].numel(), level, cj_ins[r][2], cnt, 0, out.data_ptr(), cap,
                                                             C.byref(nb), cr))
    del out
    if rc or rc2:
        err("compressjs share path")
    # the assembled stream against one call over the whole input
    sh, o = [], 32
    for f, n_ in zip(frags, bits):
        sh.append(S.shift_right_bits(f, n_, o % 8))
        o += n_
    del frags
    got = S.assemble(level, sh, bits, crcs, full.device)
    del sh
    ref = torch.empty(L.b2_bzip2_bound(full.numel()), dtype=torch.uint8, device="cuda")
    on = C.c_size_t()
    if L.b2_bzip2_compress_dev_flavor(full.data_ptr(), full.numel(), level, ref.data_ptr(), ref.numel(), C.byref(on), 1):
        err("b2_bzip2_compress_dev_flavor")
    same = got.numel() == on.value and bool(torch.equal(got, ref[: on.value]))
    sha = hashlib.sha256(got.cpu().numpy().tobytes()).hexdigest()
    del ref, got
    pre = full[: a.check_mib << 20].cpu().numpy().tobytes()
    po, pn = C.POINTER(C.c_uint8)(), C.c_size_t()
    if L.b2_bzip2_compress_flavor(pre, len(pre), level, C.byref(po), C.byref(pn), 1):
        err("b2_bzip2_compress_flavor")
    prefix_ok = C.string_at(po, pn.value) == bz2.compress(pre, level)
    L.b2_free(po)
    res = {"card": card(), "world": world, "share_mib": a.mib, "halo_mib": a.halo_mib, "level": level, "blocks": total,
           "gathered_table_bytes_per_rank": world * 16 * longest, "ms_host_gathered_tables_to_chain": round(ms_chain, 3),
           "stream_equals_single_call": same, "stream_sha256": sha, "prefix_mib_equals_bz2": a.check_mib if prefix_ok else False,
           "ranks": ranks, "compressjs_last_rank": {"ms_plan": round(cj_plan, 3), "ms_encode": round(cj_enc, 3), "blocks": cnt}}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sharded_libbz2_run.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
