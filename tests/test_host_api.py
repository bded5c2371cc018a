"""CPU tests of the host layer: the C-ABI library loads and exports every symbol of include/b2bz.h,
fails loudly without a GPU (no CPU fallback), and the stream coercion rules of lib/Util.js:9-101."""
import os
import re

import numpy as np
import pytest

from tests import util as T

ROOT = T.ROOT


def test_library_exports_every_declared_symbol():
    from compressjs_b200 import _native
    L = _native.lib()
    hdr = open(os.path.join(ROOT, "include", "b2bz.h")).read()
    declared = set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", hdr))
    assert declared and declared == set(_native.EXPORTS)
    for name in declared:
        assert hasattr(L, name), name


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from compressjs_b200 import Bzip2
    with pytest.raises(RuntimeError) as e:
        Bzip2.compressFile(b"hello", None, 9)
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under compressjs_b200/ may import, link or call it."""
    pkg = os.path.join(ROOT, "compressjs_b200")
    pat = re.compile(r"(from\s+oracle|import\s+oracle|liboracle|\borc_[a-z0-9_]+\s*\()")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc", ".js")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not pat.search(src), f


def test_level_validation_matches_reference():
    from compressjs_b200 import Bzip2
    for bad in (0, 10, -1):
        with pytest.raises(ValueError):  # `throw new Error('Invalid block size multiplier')` lib/Bzip2.js:888-890
            Bzip2.compressFile(b"x", None, bad)


def test_stream_coercion():
    from compressjs_b200 import _streams as S

    class In:
        def __init__(self, b):
            self.b, self.i = b, 0

        def readByte(self):
            if self.i >= len(self.b):
                return -1
            self.i += 1
            return self.b[self.i - 1]

    class Out:
        def __init__(self):
            self.buf = bytearray()

        def writeByte(self, b):
            self.buf.append(b)

    assert S.coerce_input(In(b"abc")).tobytes() == b"abc"
    assert S.coerce_input([1, 2, 3]).tobytes() == b"\x01\x02\x03"
    assert S.coerce_input(bytearray(b"xy")).tobytes() == b"xy"
    data = np.frombuffer(b"hello", dtype=np.uint8)
    assert S.deliver_output(None, data) == b"hello"
    o = Out()
    assert S.deliver_output(o, data) is o and bytes(o.buf) == b"hello"
    assert S.deliver_output(5, data) == b"hello"
    with pytest.raises(TypeError):
        S.deliver_output(4, data)
    buf = bytearray(5)
    assert S.deliver_output(buf, data) is buf and bytes(buf) == b"hello"
    with pytest.raises(TypeError):
        S.deliver_output(bytearray(6), data)


def test_device_allocator_port_matches_kats(tmp_path):
    """compressjs_b200/csrc/huffalloc.cuh compiled for the host == test/huffman.js known answers."""
    import ctypes as C
    import subprocess
    so = str(tmp_path / "libha_test.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-x", "c", os.path.join(ROOT, "tests", "host", "huffalloc_host.c"), "-o", so])
    L = C.CDLL(so)
    fib = [0, 1]
    while len(fib) < 36:
        fib.append(fib[-1] + fib[-2])

    def f(a, ml):
        arr = np.array(a, dtype=np.int32)
        L.host_ha_allocate(arr.ctypes.data, arr.size, ml)
        return arr.tolist()
    assert f([1] * 5, 32) == [3, 3, 2, 2, 2]
    assert f([0, 0, 1, 1, 1, 1], 3) == [3, 3, 3, 3, 2, 2]
    assert f(fib[:36], 20) == [20] * 16 + [19, 19, 18, 17, 16, 16, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1]
    assert f(fib[:36], 6) == [6] * 30 + [5, 5, 5, 4, 3, 2]
    from oracle import oracle as O
    g = T.rng(5)
    for _ in range(300):
        n = int(g.integers(3, 259))
        fr = np.sort(g.integers(0, 900000, size=n)).astype(np.int32)
        assert f(fr, 20) == O.huffman_code_lengths(fr.tolist(), 20)


def test_bwtc_core_matches_oracle(tmp_path):
    """compressjs_b200/csrc/bwtc_core.cuh (the serial model + range coder that bwtc.cu runs on the GPU) built for the
    host: container bytes and decoded L columns must equal the oracle's for every level family."""
    import ctypes as C
    import subprocess
    from oracle import oracle as O
    so = str(tmp_path / "libbwtc_host_test.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-x", "c", os.path.join(ROOT, "tests", "host", "bwtc_host.c"), "-o", so])
    L = C.CDLL(so)
    L.host_bwtc_encode.restype = C.c_size_t
    L.host_bwtc_encode.argtypes = [C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t]
    L.host_bwtc_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]

    def enc(data, level):
        bs = level * 100000
        blocks = [data[i:i + bs] for i in range(0, len(data), bs)]
        pairs = [O.bwt_sentinel(b) for b in blocks]
        lens = np.array([len(b) for b in blocks], dtype=np.uint32)
        pp = np.array([p for _, p in pairs], dtype=np.uint32)
        U = np.frombuffer(b"".join(u for u, _ in pairs) or b"\0", dtype=np.uint8).copy()
        cap = len(data) * 2 + 4096
        out = np.zeros(cap, dtype=np.uint8)
        n = L.host_bwtc_encode(level, len(blocks), lens.ctypes.data, pp.ctypes.data, U.ctypes.data, len(data), out.ctypes.data, cap)
        return bytes(out[:n])

    def dec(z, n):
        Lout = np.zeros(max(n, 1), dtype=np.uint8)
        lens = np.zeros(64, dtype=np.uint32)
        pp = np.zeros(64, dtype=np.uint32)
        fs = C.c_uint64()
        a = np.frombuffer(z, dtype=np.uint8).copy()
        nb = L.host_bwtc_decode(a.ctypes.data, a.size, Lout.ctypes.data, Lout.size, lens.ctypes.data, pp.ctypes.data, 64, C.byref(fs))
        assert nb >= 0 and fs.value == n + 1
        out, off = b"", 0
        for k in range(nb):
            ln = int(lens[k])
            out += O.unbwt_sentinel(bytes(Lout[off:off + ln]), int(pp[k]))
            off += ln
        return out

    cases = [T.fixture("sample0.ref"), T.fixture("sample2.ref"), T.fixture("sample5.ref")[:450001], b"", b"a", b"\x00" * 5000,
             T.ascii_random(250001, 3) + T.runs(60000, 4)]
    for d in cases:
        for level in (1, 2, 5, 6, 9):
            ref = O.bwtc_compress(d, level)
            assert enc(d, level) == ref
            assert dec(ref, len(d)) == d


def test_napi_addon_type_checks_against_the_napi_surface():
    """The N-API addon cannot be built here (no node, no node-gyp); it must at least compile as C++ against the
    declarations of the N-API calls it makes (tests/host/node_api_stub) and its build recipe must be present."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    napi = os.path.join(root, "compressjs_b200", "napi")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I" + os.path.join(root, "tests", "host", "node_api_stub"),
                        os.path.join(napi, "addon.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert os.path.exists(os.path.join(napi, "binding.gyp"))
    pkg = json.load(open(os.path.join(napi, "package.json")))
    assert pkg["main"] == "index.js" and pkg["gypfile"] is True
