"""Encode time of the two bzip2 flavors on the 1 GiB config-2 input (ASCII random, level 9) with the input in HBM, and
the libbz2 flavor's bytes against bz2.compress on a 64 MiB prefix.  Runs the flavors alternately, three times each,
and reports medians of the call time (CUDA events around b2_bzip2_compress_dev_flavor) and of the RLE1 and Huffman
stage times (b2_get_stats).  Prints one JSON line (also written to DIR/libbz2_run.json when --out is given).

    python tools/libbz2_run.py [--mib 1024] [--runs 3] [--out DIR]
"""
import argparse
import bz2
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--check-mib", type=int, default=64)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from compressjs_b200 import _native
    from tests.util import ascii_random
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    L = _native.lib()
    n = a.mib << 20
    data = ascii_random(n)
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = L.b2_bzip2_bound(n)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    out_n = C.c_size_t()

    def one(flavor):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        rc = L.b2_bzip2_compress_dev_flavor(d_in.data_ptr(), n, 9, d_out.data_ptr(), cap, C.byref(out_n), flavor)
        e1.record()
        torch.cuda.synchronize()
        if rc:
            raise RuntimeError(_native.last_error())
        st = _native.stats()
        return {"ms": e0.elapsed_time(e1), "ms_rle1": st["ms_rle1"], "ms_bwt": st["ms_bwt"], "ms_mtf": st["ms_mtf"],
                "ms_huff": st["ms_huff"], "ms_pack": st["ms_pack"], "bytes": out_n.value, "blocks": st["blocks"]}

    one(0), one(1)  # warm-up of both flavors' kernels and the memory pool
    res = {0: [], 1: []}
    for _ in range(a.runs):
        for fl in (0, 1):
            res[fl].append(one(fl))
    med = {name: {k: statistics.median(r[k] for r in res[fl]) for k in res[fl][0]} for fl, name in ((0, "compressjs"), (1, "libbz2"))}
    for name in med:
        med[name]["gb_per_s"] = n / med[name]["ms"] / 1e6
    # bytes of the libbz2 flavor on a prefix, against the host's libbz2
    m = a.check_mib << 20
    rc = L.b2_bzip2_compress_dev_flavor(d_in.data_ptr(), m, 9, d_out.data_ptr(), cap, C.byref(out_n), 1)
    torch.cuda.synchronize()
    assert rc == 0, _native.last_error()
    got = d_out[:out_n.value].cpu().numpy().tobytes()
    line = {"card": card(), "input": "config-2 ascii_random %d MiB, level 9, input in HBM" % a.mib, "runs": a.runs,
            "median": med, "libbz2_prefix_mib": a.check_mib, "libbz2_prefix_equals_bz2": got == bz2.compress(data[:m], 9)}
    print(json.dumps(line))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "libbz2_run.json"), "w") as f:
            json.dump(line, f, indent=1)
    if not line["libbz2_prefix_equals_bz2"]:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
