"""The libbz2 decoder flavor against the default one, and its derandomise kernel.

1. The config-2 stream: uniform ASCII (tests/util.py ascii_random, the generator bench.py uses for config 2), 1 GiB by
   default, compressed once on the GPU at level 9, decoded through b2_bzip2_decompress and through
   b2_bzip2_decompress_flavor(B2_BZ2_LIBBZ2).  Both outputs must equal the input.
2. A multistream file of randomised 900 000-byte blocks, about 256 MB: three distinct one-block members written with
   tests/bz2synth.py (tests/libbz2_read_cases.py rand_block), repeated.  Decoded through the libbz2 flavor; the output is
   checked against the model.
After one warm-up call of each, the calls run alternately, three times each; each time is the host wall clock of one
call, which ends in a device synchronise, and the median is printed.  Then, in a run of its own, one decode of the
randomised file runs under torch.profiler for the time of the derandomise kernel alone (k_derand).  The card's name and
power limit, read in the same run, head the output.

    python tools/libbz2_dec_run.py [GiB]      (default 1)
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


def randomised_file(target=256 << 20):
    from tests import bz2synth as W
    from tests import libbz2_read_cases as LC
    from tests import util as T
    members, outs = [], []
    for s in range(3):
        P = np.frombuffer(T.ascii_random(900000, 500 + s), np.uint8)
        members.append(W.Member([LC.rand_block(P)], 9).data)
        outs.append(W.model_rle1(P)[0].tobytes())
    n = target // 900000
    return b"".join(members[i % 3] for i in range(n)), b"".join(outs[i % 3] for i in range(n)), n


def main():
    from compressjs_b200 import Bzip2, _native
    from tests import util as T
    L = _native.lib()
    gib = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    print("card:", card())
    data = T.ascii_random(int(gib * (1 << 30)))
    z = np.frombuffer(bytes(Bzip2.compressFile(data, None, 9)), np.uint8)
    rz, rexp, nm = randomised_file()
    ra = np.frombuffer(rz, np.uint8)
    print("config-2 bytes:", len(data), "compressed:", z.size, "| randomised members:", nm, "compressed:", ra.size,
          "decoded:", len(rexp))

    def dec(a, ms, flavor):
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        rc = L.b2_bzip2_decompress_flavor(a.ctypes.data, a.size, ms, C.byref(out), C.byref(n), flavor)
        assert rc == 0, _native.last_error()
        return out, n.value

    calls = {
        "config2_default": (lambda: dec(z, 0, 0), data),
        "config2_libbz2": (lambda: dec(z, 0, 1), data),
        "randomised_libbz2": (lambda: dec(ra, 1, 1), rexp),
    }
    times = {k: [] for k in calls}
    for rep in range(4):   # the first round is the warm-up
        for name, (fn, want) in calls.items():
            t0 = time.perf_counter()
            out, n = fn()
            dt = time.perf_counter() - t0
            if rep == 3:
                assert np.ctypeslib.as_array(out, (n,)).tobytes() == want, name
            L.b2_free(out)
            if rep:
                times[name].append(1e3 * dt)
    for name, (_, want) in calls.items():
        med = float(np.median(times[name]))
        print(json.dumps({"call": name, "ms_median": med, "ms": times[name], "decoded_bytes": len(want),
                          "GB_per_s": len(want) / med / 1e6}))
    d, l = np.median(times["config2_default"]), np.median(times["config2_libbz2"])
    print(json.dumps({"libbz2_over_default": float(l / d)}))


def profile_derand():
    from compressjs_b200 import _native
    import torch
    from torch.profiler import ProfilerActivity, profile
    L = _native.lib()
    rz, rexp, nm = randomised_file()
    ra = np.frombuffer(rz, np.uint8)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    assert L.b2_bzip2_decompress_flavor(ra.ctypes.data, ra.size, 1, C.byref(out), C.byref(n), 1) == 0
    L.b2_free(out)
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert L.b2_bzip2_decompress_flavor(ra.ctypes.data, ra.size, 1, C.byref(out), C.byref(n), 1) == 0
    L.b2_free(out)
    ks = [e for e in prof.events() if "k_derand" in e.name]
    us = sum(e.device_time for e in ks) if ks and hasattr(ks[0], "device_time") else sum(e.cuda_time for e in ks)
    print(json.dumps({"kernel": "k_derand", "launches": len(ks), "ms_total": us / 1e3, "blocks": nm,
                      "us_per_block": us / max(nm, 1)}))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--profile":
        profile_derand()
    else:
        main()
