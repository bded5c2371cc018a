"""bzip2 -9 decode (b2_bzip2_decompress, host in, host out) of a large config-2-style buffer, default input window
against a small one ($B2_DEC_WINDOW).

The input is uniform ASCII (tests/util.py ascii_random, the generator bench.py uses for config 2), compressed once at
level 9.  Each window runs in a child process of its own: one warm-up call, then REPS timed calls; it prints the median
host wall clock (the call ends in a device synchronise), dev_peak_bytes of the last call, and checks the output
against the input ($B2_LIB picks another build of the library).  The card's name and power limit, read in the same run, head the output.

    python tools/dec_window_run.py [GiB [REPS [WINDOW ...]]]      (default: 4 GiB, 3 calls, windows default and 256 MiB)
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np


def child(zpath, reps, want, want_n):
    import ctypes as C
    from compressjs_b200 import _native
    L = _native.lib()
    z = np.fromfile(zpath, dtype=np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    times = []
    for i in range(reps + 1):   # warm-up, then the timed calls
        t0 = time.perf_counter()
        rc = L.b2_bzip2_decompress(z.ctypes.data, z.size, 0, C.byref(out), C.byref(n))
        dt = time.perf_counter() - t0
        assert rc == 0, _native.last_error()
        st = _native.stats()
        got = np.ctypeslib.as_array(out, (n.value,))   # (ctypes.string_at takes no size past 2^31)
        if i == reps and hashlib.sha256(got).hexdigest() != want:
            from tests import util as T
            ref = np.frombuffer(T.ascii_random(int(want_n)), np.uint8)
            m = min(ref.size, got.size)
            bad = np.flatnonzero(ref[:m] != got[:m])
            raise SystemExit("output differs: %d bytes for %d, first difference at %s" % (got.size, ref.size, bad[:1]))
        L.b2_free(out)
        if i:
            times.append(1e3 * dt)
    print(json.dumps({"ms_median": float(np.median(times)), "ms": times, "dev_peak_bytes": st["dev_peak_bytes"],
                      "bytes": n.value}))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return "nvidia-smi failed: %r" % e


def main():
    gib = float(sys.argv[1]) if len(sys.argv) > 1 else 4
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    windows = sys.argv[3:] or ["default", str(256 << 20)]
    from tests import util as T
    from compressjs_b200 import Bzip2
    print("card:", card(), flush=True)
    data = T.ascii_random(int(gib * (1 << 30)))
    t0 = time.perf_counter()
    z = Bzip2.compressFile(data, None, 9)
    print("input %.2f GiB -> %d bytes bzip2 -9 (encode %.1f s)" % (gib, len(z), time.perf_counter() - t0), flush=True)
    want, n = hashlib.sha256(data).hexdigest(), len(data)
    del data
    with tempfile.TemporaryDirectory() as tmp:
        zpath = os.path.join(tmp, "z.bz2")
        with open(zpath, "wb") as f:
            f.write(z)
        del z
        for w in windows:
            env = dict(os.environ)
            env.pop("B2_DEC_WINDOW", None)
            if w != "default":
                env["B2_DEC_WINDOW"] = w
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", zpath, str(reps), want, str(n)], env=env,
                               capture_output=True, text=True, timeout=3600)
            if r.returncode:
                print("window %s: FAILED %s" % (w, (r.stdout + r.stderr)[-600:]), flush=True)
                continue
            res = json.loads(r.stdout.strip().splitlines()[-1])
            print("window %s: %s" % (w, json.dumps(res)), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        child(sys.argv[2], int(sys.argv[3]), sys.argv[4], sys.argv[5])
    else:
        main()
