"""Block recovery (b2_bzip2_recover) of a config-2 1 GiB buffer at level 9, undamaged and with every 64th block's data
damaged, against b2_bzip2_decompress of the undamaged stream.

The input is uniform ASCII (tests/util.py ascii_random, the generator bench.py uses for config 2), compressed once on the
GPU at level 9.  The damaged copy has one byte flipped in the middle of every 64th block.  After one warm-up call of
each, the calls run alternately, three times each; each time is the host wall clock of one call, which ends in a device
synchronise, and the median is printed with dev_peak_bytes of the call.  The outputs are checked: the recovered bytes of
the undamaged stream equal the input, and the repaired streams decode to the recovered bytes.  Then one repair call runs
under torch.profiler for the time of the splice kernel alone (k_splice).  The card's name and power limit, read in the
same run, head the output.

    python tools/recover_run.py [GiB]      (default 1)
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:
        return "nvidia-smi failed: %r" % e


def main():
    from compressjs_b200 import Bzip2, _native
    from tests import util as T
    L = _native.lib()
    gib = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    print("card:", card())
    data = T.ascii_random(int(gib * (1 << 30)))
    z = Bzip2.compressFile(data, None, 9)
    starts = [t.bit_start for t in _native.last_trace()]
    bad = bytearray(z)
    for k in range(0, len(starts) - 1, 64):
        bad[(starts[k] + starts[k + 1]) // 16] ^= 0x5A
    bad = bytes(bad)
    za, ba = np.frombuffer(z, np.uint8), np.frombuffer(bad, np.uint8)
    print("blocks:", len(starts), "damaged:", len(range(0, len(starts) - 1, 64)), "compressed bytes:", len(z))

    def recover(a, mode):
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        rows, cnt = C.POINTER(_native.RecoveredBlock)(), C.c_size_t()
        rc = L.b2_bzip2_recover(a.ctypes.data, a.size, mode, C.byref(out), C.byref(n), C.byref(rows), C.byref(cnt))
        assert rc == 0, _native.last_error()
        intact = sum(rows[i].status == 0 for i in range(cnt.value))
        return out, n.value, rows, cnt.value, intact

    def decompress(a):
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        rc = L.b2_bzip2_decompress(a.ctypes.data, a.size, 0, C.byref(out), C.byref(n))
        assert rc == 0, _native.last_error()
        return out, n.value

    calls = {
        "decompress_undamaged": lambda: decompress(za),
        "recover_bytes_undamaged": lambda: recover(za, 0),
        "recover_bz2_undamaged": lambda: recover(za, 1),
        "recover_bytes_damaged": lambda: recover(ba, 0),
        "recover_bz2_damaged": lambda: recover(ba, 1),
    }
    times = {k: [] for k in calls}
    peak = {}
    for rep in range(4):   # the first round is the warm-up
        for name, fn in calls.items():
            t0 = time.perf_counter()
            r = fn()
            dt = time.perf_counter() - t0
            peak[name] = _native.stats()["dev_peak_bytes"]
            if rep == 3:   # check the outputs once
                if name.startswith("recover"):
                    out, n, rows, cnt, intact = r
                    got = np.ctypeslib.as_array(out, (n,)).tobytes()
                    if name == "recover_bytes_undamaged":
                        assert got == data and intact == cnt == len(starts)
                    if name.startswith("recover_bz2"):
                        ref = recover(za if "undamaged" in name else ba, 0)
                        want = np.ctypeslib.as_array(ref[0], (ref[1],)).tobytes()
                        assert Bzip2.decompressFile(got) == want
                        L.b2_free(ref[0]); L.b2_free(ref[2])
                        print(name, "intact:", intact, "of", cnt, "repaired stream bytes:", n)
                else:
                    assert np.ctypeslib.as_array(r[0], (r[1],)).tobytes() == data
            L.b2_free(r[0])
            if name.startswith("recover"):
                L.b2_free(r[2])
            if rep:
                times[name].append(1e3 * dt)
    for name in calls:
        print(json.dumps({"call": name, "ms_median": float(np.median(times[name])), "ms": times[name],
                          "dev_peak_bytes": peak[name]}))
    # the splice kernel alone, from the profiler's kernel records of one repair call
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = recover(ba, 1)
    L.b2_free(r[0]); L.b2_free(r[2])
    ks = [e for e in prof.events() if e.name.startswith("k_splice") or "k_splice" in e.name]
    us = sum(e.device_time for e in ks) if ks and hasattr(ks[0], "device_time") else sum(e.cuda_time for e in ks)
    print(json.dumps({"kernel": "k_splice", "launches": len(ks), "ms_total": us / 1e3,
                      "bits_spliced": len(bad) * 8, "call": "recover_bz2_damaged"}))


if __name__ == "__main__":
    main()
