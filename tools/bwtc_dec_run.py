"""BWTC -9 decode (b2_bwtc_decompress) of the bench's bwtc workload, two builds of the library side by side.

The input is the first MiB of the config-2 buffer (uniform ASCII, tests/util.py ascii_random, the generator bench.py
uses), compressed once at level 9.  Every library in LIBS decodes it in a child process of its own ($B2_LIB), one
warm-up call and then one timed call; the children alternate between the libraries, REPS rounds.  Per library it
prints the median and range of ms_total (host wall clock around the call, which ends in a device synchronise),
ms_hdec (the serial decoder) and ms_ibwt (inverse BWT) from the library's CUDA-event stage timers, and checks that
every library returns the same bytes as the input.  The card's name and power limit head the output.

    python tools/bwtc_dec_run.py MiB REPS LIB [LIB ...]

The serial decoder runs at about 0.6 MB/s on an H100, so one call on 64 MiB takes about two minutes.
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


def child(zpath):
    import ctypes as C
    from compressjs_b200._native import Stats
    L = C.CDLL(os.environ["B2_LIB"])   # only the calls used here: an older library lacks some of today's symbols
    L.b2_bwtc_decompress.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
    L.b2_free.argtypes = [C.c_void_p]
    L.b2_get_stats.argtypes = [C.POINTER(Stats)]
    L.b2_last_error.restype = C.c_char_p
    z = np.fromfile(zpath, dtype=np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    res = None
    for _ in range(2):   # warm-up, then the timed call
        t0 = time.perf_counter()
        rc = L.b2_bwtc_decompress(z.ctypes.data, z.size, C.byref(out), C.byref(n))
        dt = time.perf_counter() - t0
        assert rc == 0, L.b2_last_error()
        s = Stats()
        L.b2_get_stats(C.byref(s))
        st = s.as_dict()
        digest = hashlib.sha256(C.string_at(out, n.value)).hexdigest()
        L.b2_free(out)
        res = {"ms_total": 1e3 * dt, "ms_hdec": st["ms_hdec"], "ms_ibwt": st["ms_ibwt"], "bytes": n.value, "sha256": digest}
    print(json.dumps(res))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return "nvidia-smi failed: %r" % e


def main():
    mb, reps, libs = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3:]
    from tests import util as T
    from compressjs_b200 import BWTC
    print("card:", card())
    data = T.ascii_random(mb << 20)
    z = BWTC.compressFile(data, None, 9)
    want = hashlib.sha256(data).hexdigest()
    print("input %d MiB -> %d bytes BWTC -9" % (mb, len(z)), flush=True)
    runs = {lib: [] for lib in libs}
    with tempfile.TemporaryDirectory() as tmp:
        zpath = os.path.join(tmp, "z.bwtc")
        with open(zpath, "wb") as f:
            f.write(z)
        for _ in range(reps):
            for lib in libs:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", zpath], env=dict(os.environ, B2_LIB=lib),
                                   capture_output=True, text=True, timeout=3600)
                assert r.returncode == 0, r.stdout + r.stderr
                res = json.loads(r.stdout.strip().splitlines()[-1])
                assert res["sha256"] == want and res["bytes"] == len(data), (lib, res)
                runs[lib].append(res)
                print(lib, json.dumps(res), flush=True)
    for lib, rs in runs.items():
        summary = {k: "%.1f (%.1f-%.1f)" % (np.median([r[k] for r in rs]), min(r[k] for r in rs), max(r[k] for r in rs))
                   for k in ("ms_total", "ms_hdec", "ms_ibwt")}
        print("median of %d: %s %s" % (len(rs), lib, json.dumps(summary)))
    print("outputs identical to the input for every library")


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        child(sys.argv[2])
    else:
        main()
