"""Stream entry points against the whole-buffer ones, and the command line before and after it became a pipe filter.

    python tools/stream_run.py [MiB=1024] [reps=3] [out.json]

On MiB of BASELINE config-2 input (uniform printable ASCII, level 9), the median wall time of
  - b2_bzip2_compress (pageable input) against b2_bzip2_compress_stream (callbacks over the same bytes), and
    b2_bzip2_decompress against b2_bzip2_decompress_stream;
  - `python -m compressjs_b200 -z / -d -t bzip2` as it is (streams), and as it was (read_input + run: the whole input,
    then the whole output), each from a regular file and from a pipe, into /dev/null.
The card's name and power limit, read in the same run, head the output; the result is printed as JSON (and written to
out.json if given)."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from compressjs_b200 import _native  # noqa: E402
from tests import util as T  # noqa: E402

OLD_CLI = """
import os, sys
sys.path.insert(0, %r)
from compressjs_b200 import cli
data, size = cli.read_input(0)
out, err = cli.run("bzip2", %s, 9, -1, data, size)
sys.stdout.buffer.write(out)
"""


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return "nvidia-smi failed: %r" % e


def med(f, reps):
    f()   # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), (min(ts), max(ts))


def main():
    mb = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    n = mb << 20
    L = _native.lib()
    L.b2_init(0)
    data = T.ascii_random(n)
    a = np.frombuffer(data, np.uint8)
    res = {"card": card(), "mib": mb, "reps": reps}

    def one_shot_z():
        out, on = C.POINTER(C.c_uint8)(), C.c_size_t()
        assert L.b2_bzip2_compress(a.ctypes.data, n, 9, C.byref(out), C.byref(on)) == 0, _native.last_error()
        z = C.string_at(out, on.value)
        L.b2_free(out)
        return z

    z = one_shot_z()
    za = np.frombuffer(z, np.uint8)

    def one_shot_d():
        out, on = C.POINTER(C.c_uint8)(), C.c_size_t()
        assert L.b2_bzip2_decompress(za.ctypes.data, za.size, 0, C.byref(out), C.byref(on)) == 0, _native.last_error()
        assert on.value == n
        L.b2_free(out)

    def streamed(call, src, arg, expect_len):
        base = np.frombuffer(src, np.uint8).ctypes.data
        pos, got = [0], [0]

        def rd(user, buf, cap):
            k = min(cap, len(src) - pos[0])
            if k:
                C.memmove(buf, base + pos[0], k)
            pos[0] += k
            return k

        def wr(user, buf, k):
            got[0] += k
            return 0

        def run():
            pos[0] = got[0] = 0
            assert call(_native.READ_FN(rd), _native.WRITE_FN(wr), None, arg) == 0, _native.last_error()
            assert got[0] == expect_len
        return run

    res["compress_one_shot_s"], res["compress_one_shot_range"] = med(one_shot_z, reps)
    res["compress_stream_s"], res["compress_stream_range"] = med(streamed(L.b2_bzip2_compress_stream, data, 9, len(z)), reps)
    res["decompress_one_shot_s"], res["decompress_one_shot_range"] = med(one_shot_d, reps)
    res["decompress_stream_s"], res["decompress_stream_range"] = med(streamed(L.b2_bzip2_decompress_stream, z, 0, n), reps)
    print({k: v for k, v in res.items() if k.endswith("_s") or k == "card"}, file=sys.stderr, flush=True)

    with tempfile.TemporaryDirectory() as td:
        raw, comp = os.path.join(td, "raw"), os.path.join(td, "raw.bz2")
        with open(raw, "wb") as f:
            f.write(data)
        with open(comp, "wb") as f:
            f.write(z)
        for d, src in ((False, raw), (True, comp)):
            flag = "-d" if d else "-z"
            new = "%s -m compressjs_b200 %s -t bzip2 %s" % (sys.executable, flag, "" if d else "-9")
            old_py = os.path.join(td, "old_cli_%s.py" % flag[1])
            with open(old_py, "w") as f:
                f.write(OLD_CLI % (ROOT, d))
            old = "%s %s" % (sys.executable, old_py)
            for name, cmd in (("new", new), ("old", old)):
                for how, sh in (("file", "%s < %s > /dev/null" % (cmd, src)), ("pipe", "cat %s | %s > /dev/null" % (src, cmd))):
                    key = "cli_%s_%s_%s" % ("d" if d else "z", name, how)
                    res[key + "_s"], res[key + "_range"] = med(
                        lambda sh=sh: subprocess.run(["bash", "-c", "set -o pipefail; " + sh], cwd=ROOT, check=True), reps)
                    print(key, res[key + "_s"], file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 3:
        with open(sys.argv[3], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
