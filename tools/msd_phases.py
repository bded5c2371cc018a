"""Cycles per phase of the forward BWT's bucket sort (k_msd_bucket), from its clock64() probe.

    python tools/msd_phases.py [MB] [REPS]

Builds a copy of libb2bz.so with bwt_msd.cu compiled under -DB2_MSD_PROBE (in a temporary directory; the other
objects are the ones build() left under build/), encodes MB MiB of config-2 ASCII at level 9 REPS times after one
warm-up, and prints, per phase, the cycles thread 0 of a CTA spent from one phase boundary to the next, averaged over
every bucket of the timed encodes.  The probe keeps its sums in shared memory, so the probe build has the default
build's registers and no spills; each stamp still adds a clock read and a shared-memory update to thread 0's path, so
the probe build's kernel times are not the library's.
"""
import ctypes as C
import glob
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402

PHASES = ["wait + load", "histogram", "scan + queue", "scatter", "ordering", "write-out"]


def build_probe(tmp):
    objdirs = glob.glob(os.path.join(ROOT, "build", "obj-*"))
    if len(objdirs) != 1:
        raise RuntimeError("run build() first (expected one object directory under build/, found %d)" % len(objdirs))
    objs = [os.path.join(objdirs[0], s[:-3] + ".o") for s in G.SRCS if s != "bwt_msd.cu"]
    probe_obj = os.path.join(tmp, "bwt_msd_probe.o")
    nvcc = G._nvcc()
    subprocess.check_call([nvcc] + G.NVCC_FLAGS + ["-DB2_MSD_PROBE", "-c", os.path.join(G.CSRC, "bwt_msd.cu"), "-o", probe_obj], cwd=G.CSRC)
    lib = os.path.join(tmp, "libb2bz.so")
    subprocess.check_call([nvcc] + G.ARCH + ["-shared", "-o", lib] + objs + [probe_obj, "-cudart", "static"])
    return lib


def main():
    mb = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["B2_LIB"] = build_probe(tmp)
        import torch
        from compressjs_b200 import _native
        from tests import util as T
        L = _native.lib()
        L.b2_msd_probe.argtypes = [C.POINTER(C.c_ulonglong)]
        assert L.b2_init(0) == 0, _native.last_error()
        n = mb << 20
        d_in = torch.frombuffer(bytearray(T.ascii_random(n)), dtype=torch.uint8).cuda()
        cap = L.b2_bzip2_bound(n)
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        out_n = C.c_size_t()
        acc = (C.c_ulonglong * (len(PHASES) + 1))()
        for r in range(reps + 1):
            rc = L.b2_bzip2_compress_dev(d_in.data_ptr(), n, 9, d_out.data_ptr(), cap, C.byref(out_n))
            assert rc == 0, _native.last_error()
            assert L.b2_msd_probe(acc) == len(PHASES)
            if r == 0:  # warm-up
                tot = [0] * (len(PHASES) + 1)
                continue
            tot = [t + a for t, a in zip(tot, acc)]
        buckets = tot[-1]
        assert buckets, "no bucket went through k_msd_bucket (the batch took the LSD path)"
        cyc = [t / buckets for t in tot[:-1]]
        print("k_msd_bucket phases, %d MiB ascii, %d encodes, %d buckets each; cycles of thread 0 per bucket:" % (mb, reps, buckets // reps))
        for name, c in zip(PHASES, cyc):
            print("  %-14s %8.0f  %5.1f %%" % (name, c, 100.0 * c / sum(cyc)))
        print("  %-14s %8.0f" % ("total", sum(cyc)))


if __name__ == "__main__":
    main()
