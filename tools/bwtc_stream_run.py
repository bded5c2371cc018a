"""Wall clock and device peak of the BWTC stream calls against the buffer calls, and the peak resident memory of the
command line's BWTC pipeline.

    python tools/bwtc_stream_run.py [--mb 128] [--dec-mb 2] [--pipe-mb 8] [--out DIR]

- compress: BWTC -9 of the first --mb MiB of the config-2 buffer (bench.py's generator) through b2_bwtc_compress and
  through b2_bwtc_compress_stream (4 MiB reads, size given); the two outputs must be equal;
- decompress: the stream of the first --dec-mb MiB through b2_bwtc_decompress and b2_bwtc_decompress_stream (the
  decoder is one serial thread, a few MiB are enough);
- the command line: `-z -t bwtc -1 | -d -t bwtc` as separate processes on --pipe-mb MiB, with the peak RSS of each.
One warm-up call of each kind first; the card's name and power limit go with the numbers.  Prints one JSON line (also
written to DIR/bwtc_stream_run.json when --out is given)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

READ = 4 << 20


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=60).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:   # noqa: BLE001 -- reported, not fatal
        return {"error": repr(e)}


class Calls:
    def __init__(self, N, data):
        self.data, self.pos, self.out = data, 0, []
        self.rd, self.wr = N.READ_FN(self._read), N.WRITE_FN(self._write)

    def _read(self, user, buf, cap):
        k = min(cap, READ, len(self.data) - self.pos)
        if k:
            C.memmove(buf, self.data[self.pos:self.pos + k], k)
        self.pos += k
        return k

    def _write(self, user, buf, n):
        self.out.append(C.string_at(buf, n))
        return 0


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=128)
    ap.add_argument("--dec-mb", type=int, default=2)
    ap.add_argument("--pipe-mb", type=int, default=8)
    ap.add_argument("--out")
    a = ap.parse_args()
    import bench
    from compressjs_b200 import _native as N
    L = N.lib()
    host = bench.gen_ascii(a.mb << 20, bench.SEED)
    data = host.tobytes()

    def buf_c(d):
        arr = np.frombuffer(d, np.uint8)
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        assert L.b2_bwtc_compress(arr.ctypes.data, arr.size, 9, C.byref(out), C.byref(n)) == 0, N.last_error()
        z = C.string_at(out, n.value)
        L.b2_free(out)
        return z

    def stream_c(d):
        cb = Calls(N, d)
        assert L.b2_bwtc_compress_stream(cb.rd, cb.wr, None, 9, len(d)) == 0, N.last_error()
        return b"".join(cb.out)

    def buf_d(z):
        arr = np.frombuffer(z, np.uint8)
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        assert L.b2_bwtc_decompress(arr.ctypes.data, arr.size, C.byref(out), C.byref(n)) == 0, N.last_error()
        d = C.string_at(out, n.value)
        L.b2_free(out)
        return d

    def stream_d(z):
        cb = Calls(N, z)
        assert L.b2_bwtc_decompress_stream(cb.rd, cb.wr, None) == 0, N.last_error()
        return b"".join(cb.out)

    res = {"gpu": gpu_info(), "compress_bytes": len(data)}
    small = data[:1 << 20]
    buf_c(small), stream_c(small)   # warm-up
    z1, t = timed(lambda: buf_c(data))
    res["compress_buffer"] = {"s": round(t, 3), "MBps": round(len(data) / t / 1e6, 2), "dev_peak_bytes": N.stats()["dev_peak_bytes"]}
    z2, t = timed(lambda: stream_c(data))
    res["compress_stream"] = {"s": round(t, 3), "MBps": round(len(data) / t / 1e6, 2), "dev_peak_bytes": N.stats()["dev_peak_bytes"]}
    res["compress_equal"] = z1 == z2
    res["compressed_bytes"] = len(z1)
    dd = data[:a.dec_mb << 20]
    zd = buf_c(dd)
    zs = buf_c(small)
    buf_d(zs), stream_d(zs)   # warm-up
    back1, t = timed(lambda: buf_d(zd))
    res["decompress_buffer"] = {"bytes": len(dd), "s": round(t, 3), "MBps": round(len(dd) / t / 1e6, 3), "dev_peak_bytes": N.stats()["dev_peak_bytes"]}
    back2, t = timed(lambda: stream_d(zd))
    res["decompress_stream"] = {"bytes": len(dd), "s": round(t, 3), "MBps": round(len(dd) / t / 1e6, 3), "dev_peak_bytes": N.stats()["dev_peak_bytes"]}
    res["decompress_equal"] = back1 == back2 == dd

    # the command line, as separate processes; the peak RSS of each from its wrapper
    wrapper = ("import resource, subprocess, sys\nrc = subprocess.call(sys.argv[2:])\n"
               "open(sys.argv[1], 'w').write(str(resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss * 1024))\nsys.exit(rc)\n")
    with tempfile.TemporaryDirectory() as t:
        w = os.path.join(t, "wrapper.py")
        open(w, "w").write(wrapper)
        src = os.path.join(t, "in")
        open(src, "wb").write(data[:a.pipe_mb << 20])
        py = sys.executable
        cmd = ("set -o pipefail; cat %(src)s | %(py)s %(w)s %(t)s/rss_z %(py)s -m compressjs_b200 -z -t bwtc -1 | "
               "%(py)s %(w)s %(t)s/rss_d %(py)s -m compressjs_b200 -d -t bwtc | cmp - %(src)s") % dict(src=src, py=py, w=w, t=t)
        env = dict(os.environ, B2_BWT_BATCH="2", B2_BWTC_DEC_BATCH="2", B2_DEC_WINDOW=str(64 << 10))
        r, dt = timed(lambda: subprocess.run(["bash", "-c", cmd], cwd=ROOT, env=env, capture_output=True, text=True))
        res["cli_pipeline"] = {"bytes": a.pipe_mb << 20, "level": 1, "ok": r.returncode == 0, "s": round(dt, 2),
                               "knobs": "B2_BWT_BATCH=2 B2_BWTC_DEC_BATCH=2 B2_DEC_WINDOW=65536",
                               "rss_z": int(open(os.path.join(t, "rss_z")).read()) if r.returncode == 0 else None,
                               "rss_d": int(open(os.path.join(t, "rss_d")).read()) if r.returncode == 0 else None,
                               "stderr": r.stderr[-500:]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "bwtc_stream_run.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
