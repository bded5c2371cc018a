"""ctypes loader for libb2bz.so (the C ABI of include/b2bz.h).

Fails loudly: if the shared library is missing, or no CUDA device is usable, every call
raises -- there is no CPU fallback in the product path.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2_LIB") or os.path.join(_HERE, "libb2bz.so")
_LIB = None

EXPORTS = [
    "b2_init", "b2_shutdown", "b2_last_error", "b2_free",
    "b2_bzip2_compress", "b2_bzip2_decompress", "b2_bzip2_decompress_block", "b2_bzip2_table",
    "b2_bzip2_decompress_partial", "b2_bzip2_decompress_block_partial", "b2_bzip2_table_partial", "b2_bzip2_decompress_blocks",
    "b2_bwt_cyclic", "b2_bwt_cyclic_batch", "b2_suffixsort", "b2_bwt_sentinel", "b2_bwt_inverse", "b2_bwtc_compress", "b2_bwtc_compress_unsized", "b2_bwtc_decompress", "b2_crc32_bzip2",
    "b2_bzip2_bound", "b2_bzip2_compress_dev", "b2_bzip2_decompress_dev",
    "b2_bzip2_plan", "b2_bzip2_plan_spec", "b2_bzip2_share_summary", "b2_bzip2_plan_share", "b2_bitshift_dev", "b2_dec_shard_open", "b2_dec_shard_export", "b2_dec_shard_finish", "b2_bzip2_encode_range_dev", "b2_get_stats", "b2_last_trace",
]


class Stats(C.Structure):
    _fields_ = [(n, C.c_float) for n in
                ("ms_total", "ms_h2d", "ms_d2h", "ms_rle1", "ms_bwt", "ms_mtf", "ms_huff", "ms_pack",
                 "ms_scan", "ms_hdec", "ms_unmtf", "ms_ibwt", "ms_unrle", "ms_radix")] + \
               [(n, C.c_uint64) for n in
                ("radix_launches", "radix_bytes", "bwt_bytes", "bwt_rounds", "kernel_launches", "blocks",
                 "raw_bytes", "comp_bytes", "msd_launches", "msd_scatter_bytes", "msd_bucket_bytes")] + \
               [(n, C.c_float) for n in ("ms_msd_scatter", "ms_msd_bucket")] + \
               [(n, C.c_uint64) for n in
                ("bwt_msd_done", "bwt_direct_done", "bwt_rounds_batches", "bwt_wide_batches",
                 "bwt_msd_fallback_why", "bwt_direct_fallback_why", "dev_peak_bytes",
                 "rle_group_scans", "rle_walk_parallel", "rle_walk_serial")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class BlockTrace(C.Structure):
    _fields_ = [("n", C.c_int32), ("pidx", C.c_int32), ("m", C.c_int32), ("alpha", C.c_int32),
                ("ngroups", C.c_int32), ("nsel", C.c_int32), ("crc", C.c_uint32), ("pad", C.c_uint32),
                ("raw_start", C.c_uint64), ("raw_len", C.c_uint64), ("bit_start", C.c_uint64),
                ("bit_len", C.c_uint64)]


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "compressjs_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    u8pp, szp = C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)
    L.b2_init.argtypes = [C.c_int]
    L.b2_last_error.restype = C.c_char_p
    L.b2_free.argtypes = [C.c_void_p]
    L.b2_bzip2_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, u8pp, szp]
    for sfx in ("", "_partial"):
        getattr(L, "b2_bzip2_decompress" + sfx).argtypes = [C.c_void_p, C.c_size_t, C.c_int, u8pp, szp]
        getattr(L, "b2_bzip2_decompress_block" + sfx).argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, u8pp, szp]
        getattr(L, "b2_bzip2_table" + sfx).argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.POINTER(C.c_uint64)),
                                                      C.POINTER(C.POINTER(C.c_uint32)), szp]
    L.b2_bzip2_decompress_blocks.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, u8pp, szp,
                                             C.POINTER(C.POINTER(C.c_uint64)), szp]
    L.b2_bwt_cyclic.restype = C.c_int32
    L.b2_bwt_cyclic.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.b2_bwt_cyclic_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.b2_suffixsort.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.b2_bwt_sentinel.restype = C.c_int32
    L.b2_bwt_sentinel.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.b2_bwt_inverse.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
    L.b2_bwtc_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, u8pp, szp]
    L.b2_bwtc_compress_unsized.argtypes = [C.c_void_p, C.c_size_t, C.c_int, u8pp, szp]
    L.b2_bwtc_decompress.argtypes = [C.c_void_p, C.c_size_t, u8pp, szp]
    L.b2_crc32_bzip2.restype = C.c_uint32
    L.b2_crc32_bzip2.argtypes = [C.c_void_p, C.c_size_t]
    L.b2_bzip2_bound.restype = C.c_size_t
    L.b2_bzip2_bound.argtypes = [C.c_size_t]
    L.b2_bzip2_compress_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, szp]
    L.b2_bzip2_decompress_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, szp]
    L.b2_bzip2_plan.argtypes = [C.c_void_p, C.c_size_t, C.c_int, szp]
    L.b2_bzip2_plan_spec.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.b2_bzip2_share_summary.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
    L.b2_bzip2_plan_share.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_uint64, C.c_uint64, C.c_size_t, C.c_size_t, C.POINTER(C.c_uint64)]
    L.b2_dec_shard_open.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.b2_dec_shard_export.argtypes = [C.c_void_p]
    L.b2_dec_shard_finish.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
    L.b2_bitshift_dev.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    L.b2_bzip2_encode_range_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_size_t, C.c_size_t, C.c_int,
                                            C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p]
    L.b2_get_stats.argtypes = [C.POINTER(Stats)]
    L.b2_last_trace.restype = C.c_size_t
    L.b2_last_trace.argtypes = [C.c_void_p, C.c_size_t]
    _LIB = L
    return L


def last_error():
    return lib().b2_last_error().decode("utf-8", "replace")


def stats():
    s = Stats()
    lib().b2_get_stats(C.byref(s))
    return s.as_dict()


def last_trace():
    L = lib()
    n = L.b2_last_trace(None, 0)
    arr = (BlockTrace * max(n, 1))()
    L.b2_last_trace(arr, n)
    return [arr[i] for i in range(n)]
