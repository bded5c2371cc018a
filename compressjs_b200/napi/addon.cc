// addon.cc -- Node N-API veneer over include/b2bz.h (cannot be built in the graft image: no node
// headers).  It only marshals Buffers; every byte of work happens behind the C ABI.
// Build (where node-gyp exists): node-gyp configure build  with libraries: ["-lb2bz"].
#include <node_api.h>
#include <stdint.h>
#include "../../include/b2bz.h"

static void fin(napi_env, void* data, void*) { b2_free(data); }

// `prop` / `val`, `prop2` / `val2`: what a failed decode had delivered (a Buffer, the table rows, end offsets), attached
// to the error for the shim
static napi_value fail(napi_env env, int rc, const char* prop = nullptr, napi_value val = nullptr, const char* prop2 = nullptr,
                       napi_value val2 = nullptr) {
  napi_value msg, err, code;
  napi_create_string_utf8(env, b2_last_error(), NAPI_AUTO_LENGTH, &msg);
  if (rc == B2_ERR_BAD_LEVEL) napi_create_error(env, nullptr, msg, &err);        // `new Error(...)` lib/Bzip2.js:888-890
  else napi_create_type_error(env, nullptr, msg, &err);                            // `new TypeError(...)` lib/Bzip2.js:82-88
  napi_create_int32(env, rc, &code);
  napi_set_named_property(env, err, "errorCode", code);
  if (prop && val) napi_set_named_property(env, err, prop, val);
  if (prop2 && val2) napi_set_named_property(env, err, prop2, val2);
  napi_throw(env, err);
  return nullptr;
}

static bool buf_arg(napi_env env, napi_value v, const uint8_t** p, size_t* n) {
  void* d = nullptr;
  if (napi_get_buffer_info(env, v, &d, n) != napi_ok) return false;
  *p = (const uint8_t*)d;
  return true;
}

// compressFile(buffer, level, flavor) -> Buffer    (Bzip2.compressFile, lib/Bzip2.js:879; flavor: B2_BZ2_*, default 0)
static napi_value CompressFile(napi_env env, napi_callback_info info) {
  size_t argc = 3; napi_value argv[3];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n; int32_t level = 9, flavor = B2_BZ2_COMPRESSJS;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  napi_get_value_int32(env, argv[1], &level);
  if (argc > 2) napi_get_value_int32(env, argv[2], &flavor);
  uint8_t* out; size_t out_n;
  int rc = b2_bzip2_compress_flavor(in, n, level, &out, &out_n, flavor);
  if (rc) return fail(env, rc);
  napi_value buf; napi_create_external_buffer(env, out_n, out, fin, nullptr, &buf);
  return buf;
}
// result of a b2_bzip2_decompress*_partial call: the Buffer, or the error with the bytes decoded before it as .partial
static napi_value decoded(napi_env env, int rc, uint8_t* out, size_t out_n) {
  napi_value buf = nullptr;
  if (out) napi_create_external_buffer(env, out_n, out, fin, nullptr, &buf);
  if (rc) return fail(env, rc, "partial", buf);
  return buf;
}
// decompressFile(buffer, multistream, flavor) -> Buffer    (Bunzip.decode, lib/Bzip2.js:454; flavor: B2_BZ2_*, default 0)
static napi_value DecompressFile(napi_env env, napi_callback_info info) {
  size_t argc = 3; napi_value argv[3];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n; bool ms = false; int32_t flavor = B2_BZ2_COMPRESSJS;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  if (argc > 1) napi_get_value_bool(env, argv[1], &ms);
  if (argc > 2) napi_get_value_int32(env, argv[2], &flavor);
  uint8_t* out = nullptr; size_t out_n = 0;
  int rc = b2_bzip2_decompress_partial_flavor(in, n, ms ? 1 : 0, &out, &out_n, flavor);
  return decoded(env, rc, out, out_n);
}
// decompressBlock(buffer, bitpos) -> Buffer        (Bunzip.decodeBlock, lib/Bzip2.js:482)
static napi_value DecompressBlock(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n; double pos = 0;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  napi_get_value_double(env, argv[1], &pos);
  uint8_t* out = nullptr; size_t out_n = 0;
  int rc = b2_bzip2_decompress_block_partial(in, n, (uint64_t)pos, &out, &out_n);
  return decoded(env, rc, out, out_n);
}
// decompressBlocks(buffer, positions /* Float64Array */) -> [Buffer, [end offset of each position's bytes]]
// (decompressBlock at every position, one GPU pass); on a decode error the bytes delivered before it go with the error as
// .partial and the end offsets of the positions delivered in full as .ends
static napi_value DecompressBlocks(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n;
  napi_typedarray_type ty; size_t count = 0; void* pv = nullptr; napi_value ab; size_t off;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  if (argc < 2 || napi_get_typedarray_info(env, argv[1], &ty, &count, &pv, &ab, &off) != napi_ok || ty != napi_float64_array)
    return fail(env, B2_ERR_BAD_ARG);
  uint64_t* pos = new uint64_t[count + 1];
  for (size_t i = 0; i < count; i++) pos[i] = (uint64_t)((const double*)pv)[i];
  uint8_t* out = nullptr; size_t out_n = 0; uint64_t* ends = nullptr; size_t done = 0;
  int rc = b2_bzip2_decompress_blocks(in, n, pos, count, &out, &out_n, &ends, &done);
  delete[] pos;
  if (rc && !out) return fail(env, rc);
  napi_value buf, e;
  napi_create_external_buffer(env, out_n, out, fin, nullptr, &buf);
  napi_create_array_with_length(env, done, &e);
  for (size_t i = 0; i < done; i++) {
    napi_value v;
    napi_create_double(env, (double)ends[i], &v);
    napi_set_element(env, e, (uint32_t)i, v);
  }
  b2_free(ends);
  if (rc) return fail(env, rc, "partial", buf, "ends", e);
  napi_value r; napi_create_array_with_length(env, 2, &r);
  napi_set_element(env, r, 0, buf); napi_set_element(env, r, 1, e);
  return r;
}
// integer argument that must be a JS number; false (and B2_ERR_BAD_ARG thrown by the caller) otherwise
static bool int_arg(napi_env env, napi_value v, int32_t* out) {
  napi_valuetype ty;
  if (napi_typeof(env, v, &ty) != napi_ok || ty != napi_number) return false;
  return napi_get_value_int32(env, v, out) == napi_ok;
}
// n bytes must exist in both the source and the destination view
static bool len_ok(int32_t n, size_t a, size_t b) { return n >= 0 && (size_t)n <= a && (size_t)n <= b; }

// table(buffer, multistream) -> [[bitpos, size], ...]   (Bunzip.table, lib/Bzip2.js:508); on a decode error the rows
// of the blocks before it go with the error as .rows
static napi_value Table(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n; bool ms = false;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  if (argc > 1) napi_get_value_bool(env, argv[1], &ms);
  uint64_t* bp = nullptr; uint32_t* sz = nullptr; size_t cnt = 0;
  int rc = b2_bzip2_table_partial(in, n, ms ? 1 : 0, &bp, &sz, &cnt);
  if (rc && !bp) return fail(env, rc);
  napi_value arr; napi_create_array_with_length(env, cnt, &arr);
  for (size_t i = 0; i < cnt; i++) {
    napi_value row, a, b;
    napi_create_array_with_length(env, 2, &row);
    napi_create_double(env, (double)bp[i], &a); napi_create_uint32(env, sz[i], &b);
    napi_set_element(env, row, 0, a); napi_set_element(env, row, 1, b);
    napi_set_element(env, arr, (uint32_t)i, row);
  }
  b2_free(bp); b2_free(sz);
  if (rc) return fail(env, rc, "rows", arr);
  return arr;
}
// recover(buffer, repair) -> [Buffer, [[bitpos, endbit, out_off, size, crc, got, status], ...]]   (b2_bzip2_recover:
// the intact blocks' bytes, or with repair the repaired stream, and one row per block magic; status is B2_REC_*)
static napi_value Recover(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n; bool repair = false;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  if (argc > 1) napi_get_value_bool(env, argv[1], &repair);
  uint8_t* out = nullptr; size_t out_n = 0; b2_recovered_block* rows = nullptr; size_t cnt = 0;
  int rc = b2_bzip2_recover(in, n, repair ? B2_RECOVER_BZ2 : B2_RECOVER_BYTES, &out, &out_n, &rows, &cnt);
  if (rc) return fail(env, rc);
  napi_value buf, arr;
  napi_create_external_buffer(env, out_n, out, fin, nullptr, &buf);
  napi_create_array_with_length(env, cnt, &arr);
  for (size_t i = 0; i < cnt; i++) {
    const b2_recovered_block& r = rows[i];
    const double f[7] = {(double)r.bitpos, (double)r.endbit, (double)r.out_off, (double)r.size, (double)r.crc, (double)r.got,
                         (double)r.status};
    napi_value o;
    napi_create_array_with_length(env, 7, &o);
    for (uint32_t k = 0; k < 7; k++) { napi_value v; napi_create_double(env, f[k], &v); napi_set_element(env, o, k, v); }
    napi_set_element(env, arr, (uint32_t)i, o);
  }
  b2_free(rows);
  napi_value res; napi_create_array_with_length(env, 2, &res);
  napi_set_element(env, res, 0, buf); napi_set_element(env, res, 1, arr);
  return res;
}
// bwtransform2(T, U, n) -> pidx                     (BWT.bwtransform2, lib/BWT.js:372)
static napi_value Bwtransform2(napi_env env, napi_callback_info info) {
  size_t argc = 3; napi_value argv[3];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t *T, *U; size_t tn, un; int32_t n = 0;
  if (!buf_arg(env, argv[0], &T, &tn) || !buf_arg(env, argv[1], &U, &un)) return fail(env, B2_ERR_BAD_ARG);
  if (argc < 3 || !int_arg(env, argv[2], &n) || !len_ok(n, tn, un)) return fail(env, B2_ERR_BAD_ARG);
  int32_t p = b2_bwt_cyclic(T, (uint8_t*)U, n);
  if (p < 0) return fail(env, p);
  napi_value r; napi_create_int32(env, p, &r);
  return r;
}

// bwtcCompressFile(buffer, level) -> Buffer        (BWTC.compressFile, lib/BWTC.js:12)
static napi_value BwtcCompressFile(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n; int32_t level = 9;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  if (argc > 1) napi_get_value_int32(env, argv[1], &level);
  uint8_t* out; size_t out_n;
  int rc = b2_bwtc_compress(in, n, level, &out, &out_n);
  if (rc) return fail(env, rc);
  napi_value buf; napi_create_external_buffer(env, out_n, out, fin, nullptr, &buf);
  return buf;
}
// bwtcDecompressFile(buffer) -> Buffer              (BWTC.decompressFile, lib/BWTC.js:141)
static napi_value BwtcDecompressFile(napi_env env, napi_callback_info info) {
  size_t argc = 1; napi_value argv[1];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* in; size_t n;
  if (!buf_arg(env, argv[0], &in, &n)) return fail(env, B2_ERR_BAD_ARG);
  uint8_t* out; size_t out_n;
  int rc = b2_bwtc_decompress(in, n, &out, &out_n);
  if (rc == B2_ERR_BAD_MAGIC) { napi_throw_error(env, nullptr, "Bad magic"); return nullptr; }   // lib/Util.js:151-153
  if (rc) return fail(env, rc);
  napi_value buf; napi_create_external_buffer(env, out_n, out, fin, nullptr, &buf);
  return buf;
}
// suffixsort(T, SA /* Int32Array */, n) -> 0        (BWT.suffixsort, lib/BWT.js:305)
static napi_value Suffixsort(napi_env env, napi_callback_info info) {
  size_t argc = 3; napi_value argv[3];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t* T; size_t tn; int32_t n = 0;
  napi_typedarray_type ty; size_t len; void* sa; napi_value ab; size_t off;
  if (!buf_arg(env, argv[0], &T, &tn)) return fail(env, B2_ERR_BAD_ARG);
  if (napi_get_typedarray_info(env, argv[1], &ty, &len, &sa, &ab, &off) != napi_ok || ty != napi_int32_array) return fail(env, B2_ERR_BAD_ARG);
  if (argc < 3 || !int_arg(env, argv[2], &n) || !len_ok(n, tn, len)) return fail(env, B2_ERR_BAD_ARG);
  int rc = b2_suffixsort(T, (int32_t*)sa, n);
  if (rc < 0) return fail(env, rc);
  napi_value r; napi_create_int32(env, 0, &r);
  return r;
}
// bwtransform(T, U, n) -> pidx + 1                   (BWT.bwtransform, lib/BWT.js:328; A is scratch, dropped)
static napi_value Bwtransform(napi_env env, napi_callback_info info) {
  size_t argc = 3; napi_value argv[3];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t *T, *U; size_t tn, un; int32_t n = 0;
  if (!buf_arg(env, argv[0], &T, &tn) || !buf_arg(env, argv[1], &U, &un)) return fail(env, B2_ERR_BAD_ARG);
  if (argc < 3 || !int_arg(env, argv[2], &n) || !len_ok(n, tn, un)) return fail(env, B2_ERR_BAD_ARG);
  int32_t p = b2_bwt_sentinel(T, (uint8_t*)U, n);
  if (p < 0) return fail(env, p);
  napi_value r; napi_create_int32(env, p, &r);
  return r;
}
// unbwtransform(T, U, n, pidx)                       (BWT.unbwtransform, lib/BWT.js:352; LF is scratch, dropped)
static napi_value Unbwtransform(napi_env env, napi_callback_info info) {
  size_t argc = 4; napi_value argv[4];
  napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr);
  const uint8_t *T, *U; size_t tn, un; int32_t n = 0, pidx = 0;
  if (!buf_arg(env, argv[0], &T, &tn) || !buf_arg(env, argv[1], &U, &un)) return fail(env, B2_ERR_BAD_ARG);
  if (argc < 4 || !int_arg(env, argv[2], &n) || !int_arg(env, argv[3], &pidx) || !len_ok(n, tn, un) || pidx < 0 || pidx > n)
    return fail(env, B2_ERR_BAD_ARG);
  int rc = b2_bwt_inverse(T, (uint8_t*)U, n, pidx);
  if (rc < 0) return fail(env, rc);
  return nullptr;
}

static napi_value Init(napi_env env, napi_value exports) {
  napi_property_descriptor d[] = {
      {"compressFile", nullptr, CompressFile, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"decompressFile", nullptr, DecompressFile, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"decompressBlock", nullptr, DecompressBlock, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"decompressBlocks", nullptr, DecompressBlocks, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"recover", nullptr, Recover, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"table", nullptr, Table, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"bwtransform2", nullptr, Bwtransform2, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"suffixsort", nullptr, Suffixsort, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"bwtransform", nullptr, Bwtransform, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"unbwtransform", nullptr, Unbwtransform, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"bwtcCompressFile", nullptr, BwtcCompressFile, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"bwtcDecompressFile", nullptr, BwtcDecompressFile, nullptr, nullptr, nullptr, napi_default, nullptr},
  };
  napi_define_properties(env, exports, sizeof d / sizeof d[0], d);
  return exports;
}
NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
