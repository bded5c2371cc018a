"""Small driver for profiling: one bzip2 -9 encode + one decode of MB MiB of a chosen workload.

    python tools/prof_run.py [MB] [ascii|enwik|text] [both|enc|dec] [--kernels [TRACE_DIR]]

--kernels runs one more encode under torch.profiler (CUDA activities) and prints the GPU time of every kernel name,
summed over its launches, largest first; with TRACE_DIR it also writes the Chrome trace there.  The profiled encode is
a run of its own, after the timed ones, so the stage timers printed above it are not slowed by tracing.
"""
import ctypes as C
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from compressjs_b200 import _native
from tests import util as T

argv = [a for a in sys.argv[1:]]
kernels, trace_dir = False, None
if "--kernels" in argv:
    i = argv.index("--kernels")
    kernels = True
    if i + 1 < len(argv):
        trace_dir = argv.pop(i + 1)
    argv.pop(i)
mb = int(argv[0]) if len(argv) > 0 else 64
kind = argv[1] if len(argv) > 1 else "ascii"
mode = argv[2] if len(argv) > 2 else "both"
n = mb << 20
if kind == "ascii":
    data = T.ascii_random(n)
elif kind == "enwik":
    from tools.workloads import enwik_like
    n = mb * 1000000
    data = enwik_like(n).tobytes()
else:
    data = (T.texty(min(n, 8 << 20), 3) * (n // (8 << 20) + 1))[:n]
L = _native.lib()
L.b2_init(0)
d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
cap = L.b2_bzip2_bound(n)
d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
out_n = C.c_size_t()


def encode():
    rc = L.b2_bzip2_compress_dev(d_in.data_ptr(), n, 9, d_out.data_ptr(), cap, C.byref(out_n))
    assert rc == 0, _native.last_error()


reps = 2 if mode != "dec" else 1
for _ in range(reps):
    encode()
print("enc", {k: round(v, 3) if isinstance(v, float) else v for k, v in _native.stats().items()})
if mode != "enc":
    d_dec = torch.empty(n, dtype=torch.uint8, device="cuda")
    dn = C.c_size_t()
    rc = L.b2_bzip2_decompress_dev(d_out.data_ptr(), out_n.value, 0, d_dec.data_ptr(), n, C.byref(dn))
    assert rc == 0 and dn.value == n and torch.equal(d_dec, d_in), _native.last_error()
    print("dec", {k: round(v, 3) if isinstance(v, float) else v for k, v in _native.stats().items()})
if kernels:
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        encode()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.split("(")[0].split("<")[0]
            t, k = tot.get(name, (0.0, 0))
            tot[name] = (t + e.device_time_total / 1000.0, k + 1)
    print("kernels of one encode of %d MiB (%s), GPU ms summed over launches, and ms per GiB of input:" % (mb, kind))
    print("%-36s %10s %8s %10s" % ("kernel", "ms", "launches", "ms/GiB"))
    for name, (t, k) in sorted(tot.items(), key=lambda x: -x[1][0]):
        print("%-36s %10.3f %8d %10.3f" % (name[:36], t, k, t * (1 << 30) / n))
    print("%-36s %10.3f" % ("total", sum(t for t, _ in tot.values())))
    if trace_dir:
        os.makedirs(trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(trace_dir, "encode_%dMiB_%s.pt.trace.json" % (mb, kind)))
