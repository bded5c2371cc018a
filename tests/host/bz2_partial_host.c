/* bz2_partial_host.c -- the CPU oracle's decoder (oracle/bz2_oracle.c, included as it is) with what it had written when
 * it fails handed back: the reference writes every decoded byte to its output stream as it goes (lib/Bzip2.js:405-448)
 * and calls table's callback once per good block (:508-548), so when it throws, the blocks in front of the error are
 * out, and so are the bytes of a block whose CRC fails.  Test infrastructure only (tests/partial_cases.py builds it).
 * Every function returns the oracle's code; *out / the row arrays are set on every return and freed by the caller. */
#include "../../oracle/bz2_oracle.c"

/* Bzip2.decompressFile (lib/Bzip2.js:454-481) */
ORC_EXPORT int part_bzip2_decompress(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n) {
  obuf_t o = {0, 0, 0};
  int rc = decode_impl(in, n, multistream, &o, 0, NULL, NULL, NULL);
  *out = o.buf ? o.buf : (uint8_t*)malloc(1); *out_n = o.len;
  return rc;
}

/* Bzip2.decodeBlock (lib/Bzip2.js:482-503) */
ORC_EXPORT int part_bzip2_decompress_block(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n) {
  crc_init();
  bunzip_t bz; memset(&bz, 0, sizeof bz);
  br_init(&bz.rd, in, n);
  obuf_t o = {0, 0, 0};
  int rc = start_bunzip(&bz);
  if (!rc) {
    br_seekbit(&bz.rd, bitpos);
    rc = get_next_block(&bz);
    if (rc == 1) rc = read_bunzip(&bz, &o);
  }
  free(bz.dbuf);
  *out = o.buf ? o.buf : (uint8_t*)malloc(1); *out_n = o.len;
  return rc;
}

/* Bzip2.table (lib/Bzip2.js:508-548): the loop of decode_impl's table mode, with the row count kept on an error */
ORC_EXPORT int part_bzip2_table(const uint8_t* in, size_t n, int multistream, uint64_t** bitpos, uint32_t** sizes, size_t* count) {
  crc_init();
  bunzip_t bz; memset(&bz, 0, sizeof bz);
  br_init(&bz.rd, in, n);
  obuf_t o = {0, 0, 0};
  size_t cap = 64;
  *bitpos = (uint64_t*)malloc(cap * 8); *sizes = (uint32_t*)malloc(cap * 4); *count = 0;
  int rc = start_bunzip(&bz);
  while (!rc && !br_stream_eof(&bz.rd)) {
    uint64_t position = br_tellbit(&bz.rd);
    rc = get_next_block(&bz);
    if (rc == 1) {
      o.len = 0;
      rc = read_bunzip(&bz, &o);
      if (rc) break;
      if (*count >= cap) { cap *= 2; *bitpos = (uint64_t*)realloc(*bitpos, cap * 8); *sizes = (uint32_t*)realloc(*sizes, cap * 4); }
      (*bitpos)[*count] = position; (*sizes)[*count] = (uint32_t)o.len; ++*count;
    } else if (rc == 0) {
      br_bits(&bz.rd, 32); /* the stream CRC, ignored */
      if (!multistream || br_stream_eof(&bz.rd)) break;
      rc = start_bunzip(&bz);
    }
  }
  free(bz.dbuf); free(o.buf);
  return rc;
}
