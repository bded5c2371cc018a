/* bz2_recover_host.c -- the CPU oracle's decodeBlock (oracle/bz2_oracle.c, included as it is) with what block recovery
 * needs of it: the bit behind the block's end-of-block code and the CRC of the bytes it decoded.  Test infrastructure
 * only (tests/recover_model.py builds it). */
#include "../../oracle/bz2_oracle.c"

/* Bzip2.decodeBlock (lib/Bzip2.js:482-503) at bitpos.  Returns the oracle's code and sets *out / *out_n on every return
 * (freed by the caller): the block's bytes when it decoded up to its CRC check, whether that passed or not.  *endbit and
 * *got (the CRC of those bytes) are set then too, and are 0 otherwise. */
ORC_EXPORT int rec_bzip2_decompress_block(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n,
                                          uint64_t* endbit, uint32_t* got) {
  crc_init();
  bunzip_t bz; memset(&bz, 0, sizeof bz);
  br_init(&bz.rd, in, n);
  obuf_t o = {0, 0, 0};
  *endbit = 0; *got = 0;
  int rc = start_bunzip(&bz);
  if (!rc) {
    br_seekbit(&bz.rd, bitpos);
    rc = get_next_block(&bz);
    if (rc == 1) {
      *endbit = br_tellbit(&bz.rd);
      rc = read_bunzip(&bz, &o);
      *got = orc_crc32(o.buf, o.len);
    }
  }
  free(bz.dbuf);
  *out = o.buf ? o.buf : (uint8_t*)malloc(1); *out_n = o.len;
  return rc;
}
