"""The encoder's RLE1 block cut and CRCs against the oracle at every tile, scan-group and block seam.

The corpus of tests/rle1_cases.py runs through the encoder in several configurations, each in a child process because
the library reads its settings once per process:
- default: Bzip2.compressFile (a), b2_bzip2_compress_dev at pointer skews 0, 1 and 255 (e: a skew that is not 0 mod 16
  turns the tile fast path off and moves the CRC pieces), and simulated ranks that hold only their share of the input
  through b2_bzip2_share_summary / b2_bzip2_plan_share, with share edges inside planted runs (f);
- B2_RLE_SCAN_GROUPS=1: the multi-CTA tile scan on the 8-40 MiB cases (b), and the simulated ranks again;
- B2_H2D_CHUNK: a pinned input uploaded in chunks that end on a tile edge, one byte past it, or inside a run (c);
- B2_STREAM_WINDOW: a streaming window that ends inside a long run or on a block boundary (d).
For every case the test checks:
- the per-block trace (raw_start, raw_len, n, crc) equals the oracle's rle1_split (the first differing block and
  field is reported);
- the stream equals the oracle's byte for byte (for f: whenever the ranks' pieces chain up, which the model predicts
  for every share job);
- decompressFile gives the input back, and libbz2 decodes the stream when it is in its language;
- the path counters of b2_stats equal the model's prediction.  Pinned uploads are the exception: how many chunks have
  landed when a prefix is planned depends on timing, so only their trace and stream are checked.
"""
import bz2
import json
import os
import subprocess
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import oracle as O
from tests import rle1_cases as RC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTERS = ("rle_group_scans", "rle_walk_parallel", "rle_walk_serial")

_CHILD = r"""
import ctypes as C, json, sys
sys.path.insert(0, %(root)r)
import numpy as np, torch
from compressjs_b200 import Bzip2, _native, sharded as S
from tests import rle1_cases as RC
jobs = json.loads(sys.argv[1])
L = _native.lib()
out = {}

def counters():
    st = _native.stats()
    return np.array([st[f] for f in %(counters)r], dtype=np.int64)

def trace():
    return np.array([(t.raw_start, t.raw_len, t.n, t.crc) for t in _native.last_trace()], dtype=np.int64).reshape(-1, 4)

for j, job in enumerate(jobs):
    try:
        c = RC.case(job["case"])
        data, level, mode, key = c.data, job["level"], job["mode"], "j%%d_" %% j
        if mode == "file":
            z = Bzip2.compressFile(data, None, level)
            out[key + "stats"], out[key + "trace"] = counters(), trace()
        elif mode == "pinned":
            src = torch.frombuffer(bytearray(data), dtype=torch.uint8).pin_memory()
            o, n = C.POINTER(C.c_uint8)(), C.c_size_t()
            assert L.b2_bzip2_compress(src.data_ptr(), len(data), level, C.byref(o), C.byref(n)) == 0, _native.last_error()
            z = C.string_at(o, n.value)
            L.b2_free(o)
            out[key + "stats"], out[key + "trace"] = counters(), trace()
        elif mode == "dev":
            skew = job["skew"]
            buf = torch.zeros(len(data) + 512, dtype=torch.uint8, device="cuda")
            buf[skew:skew + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            cap = L.b2_bzip2_bound(len(data))
            d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
            n = C.c_size_t()
            torch.cuda.synchronize()
            assert L.b2_bzip2_compress_dev(buf.data_ptr() + skew, len(data), level, d_out.data_ptr(), cap, C.byref(n)) == 0, _native.last_error()
            out[key + "stats"], out[key + "trace"] = counters(), trace()
            z = bytes(d_out[:n.value].cpu().numpy().tobytes())
        else:   # shares
            world, halo = job["world"], job["halo"]
            edges = RC.share_edges(c, world)
            n_all = len(data)
            bufs, summaries, st_sum = [], [], []
            for r in range(world):
                g0, g1 = edges[r], edges[r + 1]
                hold = min(n_all, g1 + halo) - g0
                d = torch.frombuffer(bytearray(data[g0:g0 + hold]), dtype=torch.uint8).cuda()
                torch.cuda.synchronize()
                sm = (C.c_uint64 * 4)()
                assert L.b2_bzip2_share_summary(d.data_ptr(), g1 - g0, sm) == 0, _native.last_error()
                st_sum.append(counters())
                bufs.append((d, g0))
                summaries.append(tuple(int(v) for v in sm))
            plan, total, _ = S.share_plan_inputs(summaries, level)
            infos, rows, st_plan, frags, bits, crcs = [], [], [], [], [], []
            for r in range(world):
                d, g0 = bufs[r]
                st_in, w_in, first, count, _ = plan[r]
                info = (C.c_uint64 * 6)()
                assert L.b2_bzip2_plan_share(d.data_ptr(), d.numel(), level, st_in, w_in, first, count, info) == 0, _native.last_error()
                st_plan.append(counters())
                row = [int(v) for v in info]
                rows.append(row)
                infos.append((row[0] + g0, row[1] + g0, row[2], row[3], row[4], total))
                f, nb, cr = S._range_encoder(L, d, d.numel(), level)(first, row[4])
                frags.append(f); bits.append(nb); crcs.append(cr)
            ok = S.spec_plan_ok(infos, n_all)
            z = b""
            if ok:
                sh, o = [], 32
                for f, nb in zip(frags, bits):
                    sh.append(S.shift_right_bits(f, nb, o %% 8))
                    o += nb
                z = bytes(S.assemble(level, sh, bits, crcs, frags[0].device).cpu().numpy().tobytes())
            out[key + "summaries"] = np.array([[np.uint64(v) for v in s] for s in summaries], dtype=np.uint64)
            out[key + "plan"] = np.array([[np.uint64(v) for v in p[:4]] for p in plan], dtype=np.uint64)
            out[key + "rows"] = np.array(rows, dtype=np.uint64)
            out[key + "st_sum"], out[key + "st_plan"] = np.array(st_sum), np.array(st_plan)
            out[key + "ok"] = np.array(ok)
        out[key + "z"] = np.frombuffer(z, dtype=np.uint8)
        out[key + "back"] = np.array(bool(z) and Bzip2.decompressFile(z) == data)
    except Exception as ex:   # reported by the parent with the job it belongs to
        out["j%%d_err" %% j] = np.array(repr(ex))
np.savez(sys.argv[2], **out)
"""


def _configs():
    """{name: (env, [job])}."""
    cs = RC.cases()
    cfg = {"default": ({}, []), "groups": ({"B2_RLE_SCAN_GROUPS": "1"}, [])}
    for c in cs:
        for lv in c.levels:
            cfg["default"][1].append(dict(case=c.name, level=lv, mode="file"))
            if c.groups_hook:
                cfg["groups"][1].append(dict(case=c.name, level=lv, mode="file"))
            for world, halo in c.shares:
                job = dict(case=c.name, level=lv, mode="shares", world=world, halo=halo)
                cfg["default"][1].append(job)
                if c.groups_hook:
                    cfg["groups"][1].append(job)
            if c.skew:
                cfg["default"][1].extend(dict(case=c.name, level=lv, mode="dev", skew=s) for s in (0, 1, 255))
            for ch in c.chunk:
                cfg.setdefault("chunk_%d" % ch, ({"B2_H2D_CHUNK": str(ch)}, []))[1].append(dict(case=c.name, level=lv, mode="pinned"))
        for w in c.window:
            win = RC.window_bytes(c, w)
            cfg.setdefault("window_%s_%d" % (c.name, win), ({"B2_STREAM_WINDOW": str(win)}, []))[1].append(
                dict(case=c.name, level=c.levels[0], mode="file", window=win))
    return cfg


CONFIGS = _configs()


@pytest.fixture(scope="module")
def gpu_runs(tmp_path_factory):
    """One child process per configuration, started in the background while the oracle runs."""
    tmp = tmp_path_factory.mktemp("rle1_seams")
    results = {}

    def run_all():
        for name, (env, jobs) in CONFIGS.items():
            out = tmp / ("%s.npz" % name)
            e = {k: v for k, v in os.environ.items() if k not in ("B2_RLE_SCAN_GROUPS", "B2_H2D_CHUNK", "B2_STREAM_WINDOW")}
            e.update(env)
            r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT, "counters": COUNTERS}, json.dumps(jobs), str(out)],
                               env=e, capture_output=True, text=True, timeout=1800)
            results[name] = (r, out)

    th = threading.Thread(target=run_all)
    th.start()
    return th, results


@pytest.fixture(scope="module")
def oracle():
    """(case, level) -> (rle1_split, stream)."""
    keys = sorted({(j["case"], j["level"]) for _, jobs in CONFIGS.values() for j in jobs})
    threads = min(os.cpu_count() or 1, 16)

    def one(k):
        data = RC.case(k[0]).data
        return k, (O.rle1_split(data, k[1])[:3], O.bzip2_compress(data, k[1], threads=threads))

    with ThreadPoolExecutor(max_workers=2) as ex:
        return dict(ex.map(one, keys))


def _trace_diff(tr, split, n):
    starts, lens, crcs = split
    exp = np.stack([starts.astype(np.int64), np.diff(np.append(starts.astype(np.int64), n)), lens.astype(np.int64),
                    crcs.astype(np.int64)], axis=1) if len(starts) else np.zeros((0, 4), dtype=np.int64)
    if tr.shape == exp.shape and np.array_equal(tr, exp):
        return None
    for k in range(min(len(tr), len(exp))):
        for f, name in enumerate(("raw_start", "raw_len", "n", "crc")):
            if tr[k, f] != exp[k, f]:
                return "block %d: %s %d, oracle %d" % (k, name, tr[k, f], exp[k, f])
    return "%d blocks, oracle %d" % (len(tr), len(exp))


@pytest.mark.parametrize("config", list(CONFIGS))
def test_rle1_cut_matches_oracle_and_model(config, gpu_runs, oracle):
    th, results = gpu_runs
    th.join()
    r, out = results[config]
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(out)
    env, jobs = CONFIGS[config]
    hook = "B2_RLE_SCAN_GROUPS" in env
    failures = []
    for j, job in enumerate(jobs):
        c, lv, mode, key = RC.case(job["case"]), job["level"], job["mode"], "j%d_" % j
        m = RC.model(c.name)
        split, stream = oracle[(c.name, lv)]
        tag = "%s level %d %s%s" % (c.name, lv, mode, " skew %d" % job["skew"] if mode == "dev" else "")
        if key + "err" in got:
            failures.append("%s: %s" % (tag, got[key + "err"]))
            continue
        z = got[key + "z"].tobytes()
        if mode == "shares":
            tag += " world %d" % job["world"]
            ranks, want_ok = RC.share_plan(c, lv, job["world"], job["halo"], hook)
            summ = [tuple(int(v) for v in s) for s in got[key + "summaries"]]
            want = [tuple(int(v) for v in rk["summary"]) for rk in ranks]
            if summ != want:
                failures.append("%s: share summaries %s, model %s" % (tag, summ, want))
            for r, rk in enumerate(ranks):
                if tuple(got[key + "st_sum"][r]) != rk["sum_counters"]:
                    failures.append("%s rank %d: summary counters %s, model %s" % (tag, r, tuple(got[key + "st_sum"][r]), rk["sum_counters"]))
                first, count = (int(v) for v in got[key + "plan"][r][2:4])
                if (first, count) != (rk["first"], rk["count"]):
                    failures.append("%s rank %d: blocks [%d, +%d) planned, model [%d, +%d)" % (tag, r, first, count, rk["first"], rk["count"]))
                blocks, cnt = rk["blocks"], rk["counters"]
                have = tuple(int(v) for v in got[key + "st_plan"][r])
                row = [int(v) for v in got[key + "rows"][r]]
                if have != cnt or row[4] != len(blocks) or (blocks and (row[0], row[1]) != (blocks[0].s, blocks[-1].e)):
                    failures.append("%s rank %d: counters %s, %d blocks [%d, %d); model %s, %d blocks %s" % (
                        tag, r, have, row[4], row[0], row[1], cnt, len(blocks), (blocks[0].s, blocks[-1].e) if blocks else ()))
            if bool(got[key + "ok"]) != want_ok:
                failures.append("%s: the ranks' pieces chain up: %s, model %s" % (tag, bool(got[key + "ok"]), want_ok))
            if bool(got[key + "ok"]) and z != stream:
                failures.append("%s: the assembled stream differs from the oracle's" % tag)
            if bool(got[key + "ok"]) and not bool(got[key + "back"]):
                failures.append("%s: decompressFile does not give the input back" % tag)
            continue
        d = _trace_diff(got[key + "trace"], split, m.n)
        if d:
            failures.append("%s: trace differs: %s" % (tag, d))
        if z != stream:
            failures.append("%s: stream differs from the oracle's (%d vs %d bytes)" % (tag, len(z), len(stream)))
        if not bool(got[key + "back"]):
            failures.append("%s: decompressFile does not give the input back" % tag)
        if mode != "pinned":
            want = RC.window_counters(c.data, lv, job["window"], hook) if "window" in job else m.counters(lv, hook)
            have = tuple(int(v) for v in got[key + "stats"])
            if have != tuple(want):
                failures.append("%s: counters %s, model %s" % (tag, dict(zip(COUNTERS, have)), dict(zip(COUNTERS, want))))
        if mode == "file" and "window" not in job and m.libbz2(lv) and bz2.decompress(z) != c.data:
            failures.append("%s: libbz2 does not decode the stream" % tag)
    assert not failures, "%s:\n" % config + "\n".join(failures)


def test_corpus_counters_cover_every_path(gpu_runs):
    """What the GPU reported across the corpus: the group scan with and without the hook, and both walks."""
    th, results = gpu_runs
    th.join()
    tot = {}
    for config in ("default", "groups"):
        r, out = results[config]
        assert r.returncode == 0, r.stderr[-4000:]
        got = np.load(out)
        tot[config] = sum(got["j%d_stats" % j] for j, job in enumerate(CONFIGS[config][1]) if job["mode"] == "file")
    assert tot["default"][0] > 0 and tot["groups"][0] > tot["default"][0]
    assert tot["default"][1] > 0 and tot["default"][2] > 0
