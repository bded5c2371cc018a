/*
 * b2bz.h -- C ABI of libb2bz.so, the GPU-native (H100) bzip2 / BWT block pipeline.
 *
 * This is the drop-in boundary for compressjs' bzip2 hot path.  Every entry point
 * below replaces one JavaScript function of the reference (file:line in
 * cscott/compressjs); a Node N-API addon (compressjs_b200/napi/addon.cc), or any other
 * FFI, binds exactly these symbols.  Plain pointers and sizes only.
 *
 * Conventions
 *   - return value 0 = OK; negative = the reference's Bunzip.Err code
 *     (lib/Bzip2.js:62-72: -2 NOT_BZIP_DATA, -5 DATA_ERROR, -7 OBSOLETE_INPUT) or
 *     B2_ERR_* below.  b2_last_error() returns the reference's message text.
 *   - inputs are borrowed for the duration of the call; outputs are allocated by the
 *     library in pinned host memory and released with b2_free().
 *   - all work runs on the GPU selected by b2_init(); there is NO CPU fallback: if no
 *     CUDA device is usable every call fails with B2_ERR_CUDA.
 *   - calls are synchronous and serialised by an internal mutex.  A call made from inside a stream callback (below)
 *     fails with B2_ERR_BAD_ARG instead of waiting for that mutex.
 */
#ifndef B2BZ_H
#define B2BZ_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_OK 0
#define B2_ERR_NOT_BZIP_DATA (-2) /* lib/Bzip2.js:66 */
#define B2_ERR_DATA_ERROR (-5)    /* lib/Bzip2.js:69 */
#define B2_ERR_OBSOLETE_INPUT (-7) /* lib/Bzip2.js:71 */
#define B2_ERR_BAD_LEVEL (-100)   /* lib/Bzip2.js:888-890 "Invalid block size multiplier" */
#define B2_ERR_BAD_ARG (-101)
#define B2_ERR_BAD_MAGIC (-102)   /* lib/Util.js:151-153 Error("Bad magic") of the BWTC container */
#define B2_ERR_STREAM (-103)      /* a read or write callback of a stream call asked to abort */
#define B2_ERR_CUDA (-200)        /* CUDA runtime failure or no device: never falls back to CPU */

/* Select the CUDA device (ordinal) used by this process and create the context.
 * Called implicitly with device 0 (or $B2_DEVICE / $LOCAL_RANK) by the first call. */
int b2_init(int device);
void b2_shutdown(void);
const char* b2_last_error(void);
void b2_free(void* p);

/* ---- compressjs.Bzip2 (lib/Bzip2.js) -------------------------------------------- */
/* Bzip2.compressFile(input, output, level)            lib/Bzip2.js:879-929 */
int b2_bzip2_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n);
/* Bzip2.decompressFile(input, output, multistream)    lib/Bzip2.js:454-481
 * Members of a multistream file may have different levels.  On an error nothing is returned and nothing needs freeing.
 * Device memory does not grow with the file: the input goes to the device a window of W bytes at a time
 * ($B2_DEC_WINDOW, default 4 GiB), its blocks are decoded B at a time ($B2_DEC_BATCH, default 2048; B counts only the
 * blocks of the largest batch), and the decoded bytes leave through a staging buffer of at most max(W, one block) bytes.
 * A window grows past W only for a block longer than W.  For W >= 64 KiB, one call of this family (table and
 * decompress_block[s] too; b2_bzip2_decompress_dev has no staging buffer) keeps at most
 *     2 * max(W, 48 MiB) + B * 24 MiB + 16 bytes per magic in a window
 * on the device (b2_stats.dev_peak_bytes).  A position list keeps the whole input on the device instead of a window. */
int b2_bzip2_decompress(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n);
/* Bzip2.decompressBlock(input, bitPos, output)        lib/Bzip2.js:482-503 */
int b2_bzip2_decompress_block(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n);
/* Bzip2.table(input, callback, multistream)           lib/Bzip2.js:508-548
 * (the callback is replayed by the host shim from the two arrays) */
int b2_bzip2_table(const uint8_t* in, size_t n, int multistream, uint64_t** bitpos, uint32_t** sizes, size_t* count);
/* The same three calls with the reference's output on error: it writes every decoded byte to its output stream as it
 * goes (lib/Bzip2.js:405-448) and calls table's callback once per good block, so the bytes and blocks in front of an
 * error are already out when it throws.  On a decode error (-2 / -5 / -7) these return that code and the message of
 * the calls above, and *out / *out_n (the row arrays and *count) hold that prefix, to be released with b2_free():
 *   - a block whose CRC fails: the blocks before it and all of its own bytes (they are written before the check);
 *   - any other error inside a block, a bad magic, truncation: the blocks before it;
 *   - a bad stream CRC: every block of the member; a bad header of a later member: all earlier members;
 *   - table: the rows of the blocks before the failing one (the stream CRC is not checked, as there).
 * On any other error (CUDA failure, bad argument) nothing is returned.  On success they equal the calls above. */
int b2_bzip2_decompress_partial(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n);
int b2_bzip2_decompress_block_partial(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n);
int b2_bzip2_table_partial(const uint8_t* in, size_t n, int multistream, uint64_t** bitpos, uint32_t** sizes, size_t* count);
/* GPU extension: Bzip2.decompressBlock at every position of a list, in one pass (the input is uploaded once and only
 * the given positions are tested for a magic).  The result equals b2_bzip2_decompress_block_partial called once per
 * position, in list order, until the first error: positions may repeat and come in any order, an end-of-stream magic
 * gives 0 bytes, a position without a magic fails with -2 "Not bzip data", and every block is held to the dbufSize of
 * the file's first header.  *out holds the positions' bytes back to back; ends[k] is the end offset of position k's.
 *   - success: 0, *done == count, ends has count entries;
 *   - decode error (-2 / -5 / -7): the first failing position's code and message; *done = the positions delivered in
 *     full before it, ends has *done entries, and *out_n also counts the failing position's own bytes when only its CRC
 *     failed (b2_bzip2_decompress_block_partial);
 *   - count == 0: 0 and nothing decoded, whatever the input holds;  count > 0 with bitpos == NULL: B2_ERR_BAD_ARG.
 * *out and *ends are released with b2_free(); on any other error nothing is returned. */
int b2_bzip2_decompress_blocks(const uint8_t* in, size_t n, const uint64_t* bitpos, size_t count, uint8_t** out, size_t* out_n,
                               uint64_t** ends, size_t* done);

/* ---- streams: Bzip2.compressFile / decompressFile over readByte / writeByte streams (lib/Bzip2.js:405-448, 879-929) ----
 * The input is pulled through a read callback and the output pushed through a write callback as the call goes, so host
 * memory does not grow with the stream.  Both callbacks run on the calling thread, in stream order.
 *   read:  puts 1..cap bytes into buf and returns how many; 0 = end of input; < 0 = abort.  A short read is not the end:
 *          only a read that returns 0 ends the input.  Returning more than cap fails the call with B2_ERR_BAD_ARG.
 *   write: takes n > 0 bytes of output; returns 0 to go on, anything else to abort.
 * After an abort no further callback runs and the call returns B2_ERR_STREAM, with a message naming the callback.  Any
 * call of this library made from inside a callback fails with B2_ERR_BAD_ARG ("called from inside a stream callback";
 * b2_crc32_bzip2 returns (uint32_t)B2_ERR_BAD_ARG there, and b2_free, b2_get_stats, b2_last_trace and b2_shutdown do
 * nothing). */
typedef int64_t (*b2_read_fn)(void* user, uint8_t* buf, size_t cap);
typedef int (*b2_write_fn)(void* user, const uint8_t* buf, size_t n);
/* Compress: everything passed to write, concatenated, is the *out of b2_bzip2_compress on everything read returned, at
 * the same level, however the input is split into reads; b2_last_trace and b2_get_stats report the call as they do
 * there.  An empty input gives the 14-byte file.  A bad level returns B2_ERR_BAD_LEVEL before any callback runs.  The
 * input goes through the device in the windows of b2_bzip2_compress (W = $B2_STREAM_WINDOW): the same device memory. */
int b2_bzip2_compress_stream(b2_read_fn rd, b2_write_fn wr, void* user, int level);
/* Decompress: the bytes passed to write, the return code and b2_last_error() are those of b2_bzip2_decompress_partial on
 * the same input (data errors, CRC failures, truncation, bad members, "Not bzip data"): no byte past the prefix that
 * call returns is ever written, because a block's bytes are written only once the blocks and stream CRCs in front of
 * them have checked out.  The input is read only as far as the decode needs (a member's trailer ends a stream read
 * without multistream).  Device memory is that of b2_bzip2_decompress ($B2_DEC_WINDOW, $B2_DEC_BATCH, the formula
 * above).
 * Host memory: a stream call holds one input buffer, which starts at 64 KiB and doubles as data arrives, and one pinned
 * output buffer (compress: b2_bzip2_bound of the first window's input; decompress: the most bytes written at once).
 * The input buffer is freed when the call returns, the output buffer goes back to the pinned buffers the library
 * recycles (as b2_free does).  Whatever the stream's length, they stay within
 *     compress:    W + 1 bytes of input and b2_bzip2_bound(W) + 64 of output: under 3 W + 1 MiB in all;
 *     decompress:  the input window plus 5 bytes, and max(W, 48 MiB) of output: under 3 max(W, 48 MiB) in all
 * (the input window is W, wider only for a block longer than W, as in b2_bzip2_decompress; a compressed block is
 * under 2 MiB). */
int b2_bzip2_decompress_stream(b2_read_fn rd, b2_write_fn wr, void* user, int multistream);

/* ---- compressjs.BWT (lib/BWT.js) ------------------------------------------------- */
/* BWT.bwtransform2(T, U, n, 256) -> pidx  (cyclic)    lib/BWT.js:372-417
 * n is limited to 900 000 (the largest bzip2 block; the reference has no limit): longer strings return B2_ERR_BAD_ARG. */
int32_t b2_bwt_cyclic(const uint8_t* T, uint8_t* U, int32_t n);
/* many independent blocks at once (what compressFile does per block, batched):
 * block k is T + offs[k], length lens[k] (each <= 900000); U gets the same layout;
 * pidx[k] receives each block's primary index. */
int b2_bwt_cyclic_batch(const uint8_t* T, uint8_t* U, const uint64_t* offs, const int32_t* lens, int32_t* pidx, size_t nblocks);
/* The sentinel ("string is terminated by EOF") family used by the reference's BWTC container.  One string of
 * at most 2^20 - 2 = 1 048 574 bytes per call (the slot size of the block pipeline; BWTC blocks are <= 900 000).
 * BWT.suffixsort(T, SA, n)                            lib/BWT.js:305-321 ; returns 0 */
int b2_suffixsort(const uint8_t* T, int32_t* SA, int32_t n);
/* BWT.bwtransform(T, U, A, n) -> pidx + 1             lib/BWT.js:328-350 (A is scratch in the reference) */
int32_t b2_bwt_sentinel(const uint8_t* T, uint8_t* U, int32_t n);
/* BWT.unbwtransform(T, U, LF, n, pidx)                lib/BWT.js:352-363 (L = the transformed string, pidx as
 * returned by bwtransform; LF is scratch in the reference) */
int b2_bwt_inverse(const uint8_t* L, uint8_t* out, int32_t n, int32_t pidx);
/* ---- compressjs.BWTC (lib/BWTC.js) -- new, bound by one serial coder thread: see compressjs_b200/csrc/bwtc.cu -----
 * BWTC.compressFile(input, output, level)             lib/BWTC.js:12-139 (level outside 1..9 means 9, as there) */
int b2_bwtc_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n);
/* BWTC.compressFile of an input stream without a size  lib/Util.js:119-124: the header's size field is "unknown" (the
 * single byte 0x80, which the range coder takes as its first byte); everything else is b2_bwtc_compress.  This is what
 * the compressjs command line writes for a pipe or an empty file. */
int b2_bwtc_compress_unsized(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n);
/* BWTC.decompressFile(input, output)                  lib/BWTC.js:141-231, for streams with a size field and for
 * streams of unknown size (decoded up to the "no more blocks" marker).  Blocks are decoded a batch at a time
 * ($B2_BWTC_DEC_BATCH, default two per SM) and each batch goes to the host, so device memory is bounded by one batch
 * (about 17 MiB per block) for any file size.  A stream whose blocks exceed its size field fails as soon as they do.
 * On an error nothing is returned. */
int b2_bwtc_decompress(const uint8_t* in, size_t n, uint8_t** out, size_t* out_n);
/* ---- BWTC over read / write callbacks (b2_read_fn / b2_write_fn and their rules as for the bzip2 stream calls above) --
 * BWTC.compressFile over a read callback (lib/BWTC.js:12-139, lib/Util.js:104-142).  size >= 0 is written as the
 * header's size field (what the reference takes from inStream.size); size == -1 writes "size unknown"; any other size is
 * B2_ERR_BAD_ARG before a callback runs.  The blocks are those of every byte read, as in the reference: a size that
 * differs from the bytes read is written as given (the stream then fails the size check when decoded, as it does
 * there).  Level outside 1..9 means 9.
 * Everything passed to write, concatenated, is the *out of b2_bwtc_compress on everything read when size is their
 * count, and of b2_bwtc_compress_unsized when size == -1, however the input is split into reads and whatever
 * $B2_BWT_BATCH is; b2_get_stats reports raw_bytes, comp_bytes and blocks as those calls do. */
int b2_bwtc_compress_stream(b2_read_fn rd, b2_write_fn wr, void* user, int level, int64_t size);
/* BWTC.decompressFile over a read callback (lib/BWTC.js:141-231).  The return code and b2_last_error() are those of
 * b2_bwtc_decompress on the same bytes.  On success the bytes written are its result.  On a data error (-5) they are
 * exactly the blocks decoded in full before the failing check, in stream order, as the reference has written them when
 * it throws (lib/BWTC.js:228): a block that passes the size field is not among them, and a size field larger than the
 * blocks has every block written.  "Bad magic" (B2_ERR_BAD_MAGIC) and a bad header write nothing.  All of this holds
 * however the input is split into reads, and whatever $B2_DEC_WINDOW and $B2_BWTC_DEC_BATCH are.  The input is read only
 * as far as the decode needs (bytes behind the "no more blocks" marker may stay unread).
 *
 * Memory of every BWTC call (b2_stats.dev_peak_bytes for the device), whatever the size of the input:
 *   compress, device:    B * 96 MiB + 8 MiB, B = $B2_BWT_BATCH blocks (default two per SM): per block the forward BWT
 *                        (at most 58.5 MiB), the slots, symbols and frequency triples of the model (21 MiB at level 9)
 *                        and two output windows of the coder's worst case on one batch (each 3 n, or 2 n at levels
 *                        1..5, + n / 64 + 1 KiB for a block of n raw bytes: 5.2 MiB for both at level 9).  The input is
 *                        never on the device as a whole: it goes to the batch's slots a batch at a time.
 *   decompress, device:  W' + B * 17 MiB + 8 MiB, B = $B2_BWTC_DEC_BATCH blocks (default two per SM): per block the L
 *                        column, the decoded bytes and the inverse BWT (16.4 MiB).  W' is the window of coded bytes,
 *                        W = $B2_DEC_WINDOW (default 4 GiB, at least 64 KiB), or less for a shorter input; it widens
 *                        only for a block whose coded bytes do not fit in it, to under twice that block's coded bytes (a
 *                        coded block is under 2.72 MB; the worst one built so far, tests/bwtc_cases.py, has 1.03 MB).
 *   compress, host:      one batch of raw input (B * level * 100 000 bytes) and one pinned output buffer, which starts at
 *                        the usual coded size of a batch (B * 1.02 MB at level 9) and grows to a batch's coded bytes
 *                        only when they are more (B * 2.72 MB at level 9 in the worst case).
 *   decompress, host:    the input window (W' + 1 bytes) and one pinned batch of decoded bytes (B * 900 000 bytes). */
int b2_bwtc_decompress_stream(b2_read_fn rd, b2_write_fn wr, void* user);
/* CRC32 helper object of lib/CRC32.js:72-103 (bzip2 polynomial, MSB first) */
uint32_t b2_crc32_bzip2(const uint8_t* p, size_t n);

/* ---- device-resident entry points (buffers already in HBM) ----------------------- */
/* Same semantics as b2_bzip2_compress, but `d_in` / `d_out` are device pointers on the
 * b2_init() device (e.g. torch tensors' data_ptr()).  out_cap must be >= b2_bzip2_bound(n).
 * Used by bench.py for the HBM-resident `value` and by the multi-GPU host layer. */
size_t b2_bzip2_bound(size_t n);
int b2_bzip2_compress_dev(const void* d_in, size_t n, int level, void* d_out, size_t out_cap, size_t* out_n);
/* Decode with device buffers; *out_n receives the decoded size; fails with
 * B2_ERR_BAD_ARG (and the needed size in *out_n) if out_cap is too small. */
int b2_bzip2_decompress_dev(const void* d_in, size_t n, int multistream, void* d_out, size_t out_cap, size_t* out_n);

/* ---- block-range encode for multi-GPU sharding (SURVEY.md section 8e) ------------- */
/* Plan cache: b2_bzip2_plan, _plan_spec and _plan_share keep their plan, replacing the one kept before.  The next
 * b2_bzip2_encode_range_dev takes it if it names the same (buffer, n, level), else plans the buffer exactly; either way
 * the cache is empty afterwards.  b2_bzip2_compress_dev empties it, no other call touches it.  The buffer must not
 * change in between. */
/* Exact plan of the whole buffer; total_blocks receives the number of blocks in the file. */
int b2_bzip2_plan(const void* d_in, size_t n, int level, size_t* total_blocks);
/* Speculative range plan for rank `rank` of `world`: cuts only this rank's share of the blocks, starting from
 * the boundary implied by W-space arithmetic (exact unless a run-phase slip happened earlier in the file).
 * info[0..5] = raw start, raw end, first block, planned count, blocks actually cut, total block guess.
 * The ranks must verify end(r) == start(r+1), start(0) == 0, end(last) == n and cut == planned on every rank
 * (compressjs_b200/sharded.py does); otherwise fall back to b2_bzip2_plan. */
int b2_bzip2_plan_spec(const void* d_in, size_t n, int level, int rank, int world, uint64_t* info);
/* Sharded input: every rank holds only a contiguous share of the input (followed by a halo: the first bytes of the
 * next share, so that a block that starts in the share can be finished).
 * summary[0..3] = {aggregate RLE1 run state of the share (packed, opaque), length of its leading run, RLE1 bytes of the
 * share when no run enters it, share length}; the host layer combines the summaries of all ranks in order
 * (compressjs_b200/sharded.py: share_plan_inputs) into the run state / RLE1 output in front of every share. */
int b2_bzip2_share_summary(const void* d_share, size_t n, uint64_t* summary);
/* Cuts blocks [first, first+count) of the whole input inside the buffer d_buf[0, n) = share + halo, given the run state
 * and RLE1 output in front of it.  Speculative like b2_bzip2_plan_spec (same checks by the caller); info[0..5] = raw
 * start, raw end (offsets inside d_buf), first, planned, blocks cut, RLE1 output up to the end of the buffer. */
int b2_bzip2_plan_share(const void* d_buf, size_t n, int level, uint64_t state_in, uint64_t w_in, size_t first, size_t count, uint64_t* info);
/* dst := the first nbits of src moved to start at bit `phase` (0..7, MSB first), zero outside; dst must hold
 * ceil((phase+nbits)/32)*4 bytes and may not overlap src.  Used to align a fragment to its global bit offset. */
int b2_bitshift_dev(const void* d_src, uint64_t nbits, int phase, void* d_dst);
/* Encodes blocks [first, first+count) of the stream that b2_bzip2_compress would produce for (d_in, n, level)
 * WITHOUT file header/trailer: the fragment starts at bit offset bit_phase (0..7, chosen by the caller = global bit
 * offset mod 8) inside d_out (4-byte aligned, >= 32 bytes, zeroed first) and is *out_bits long (0 without blocks).
 * block_crcs (host, one entry per block) receives the per-block CRCs so the caller can fold the stream CRC. */
int b2_bzip2_encode_range_dev(const void* d_in, size_t n, int level, size_t first, size_t count, int bit_phase,
                              void* d_out, size_t out_cap, uint64_t* out_bits, uint32_t* block_crcs);

/* ---- sharded decode (SURVEY.md section 8e; BASELINE config 5) ----------------------------------- */
/* Every rank holds the compressed stream.  open: scan the magics and decode this rank's share of the
 * candidate blocks; info = {block candidates in the file, first, one-past-last of the own share}.
 * export: 6 x uint64 per own candidate (status, detail, end bit, block length, decoded length, 0).
 * finish: `all` = the exported rows of ALL candidates in order (all-gathered by the caller); walks the
 * block chain, expands and CRC-checks the own blocks into d_out; res = {offset of the own output in the
 * decoded stream, its length, total decoded length, index of the first failing event or -1, its code}. */
int b2_dec_shard_open(const void* d_in, size_t n, int rank, int world, uint64_t* info);
int b2_dec_shard_export(uint64_t* buf);
int b2_dec_shard_finish(const uint64_t* all, int multistream, void* d_out, size_t out_cap, uint64_t* res);

/* ---- instrumentation -------------------------------------------------------------- */
typedef struct b2_stats {
  /* GPU milliseconds of the last call, from CUDA events on the library's stream */
  float ms_total, ms_h2d, ms_d2h;
  float ms_rle1, ms_bwt, ms_mtf, ms_huff, ms_pack;          /* encode stages */
  float ms_scan, ms_hdec, ms_unmtf, ms_ibwt, ms_unrle;      /* decode stages */
  float ms_radix;            /* time inside the radix-sort pass kernel (dominant BWT kernel) */
  uint64_t radix_launches;   /* pass-kernel launches in the last call */
  uint64_t radix_bytes;      /* algorithmic bytes moved by those launches (read+written) */
  uint64_t bwt_bytes;        /* algorithmic bytes of the whole BWT stage (all its kernels) */
  uint64_t bwt_rounds;       /* prefix-doubling rounds executed (max over batches) */
  uint64_t kernel_launches;  /* all kernels launched by the last call */
  uint64_t blocks;           /* bzip2 blocks processed */
  uint64_t raw_bytes, comp_bytes;
  /* MSD path of the forward BWT (bwt_msd.cu): one scatter pass + one shared-memory bucket sort per batch */
  uint64_t msd_launches;       /* batches that took the path (one launch of each of the two kernels) */
  uint64_t msd_scatter_bytes;  /* algorithmic bytes of k_msd_scatter (text in, records out) */
  uint64_t msd_bucket_bytes;   /* algorithmic bytes of k_msd_bucket (records in, column out) */
  float ms_msd_scatter, ms_msd_bucket;
  /* How each forward-BWT batch finished (bwt.cu).  Every non-empty batch counts in exactly one of the first three. */
  uint64_t bwt_msd_done;             /* finished by the MSD path (5-byte ties ordered directly) */
  uint64_t bwt_direct_done;          /* finished by the 4-byte LSD sort + direct tie resolve */
  uint64_t bwt_rounds_batches;       /* finished by the rank-based prefix-doubling rounds (sentinel calls included) */
  uint64_t bwt_wide_batches;         /* sorted on 8-byte prefixes first (text-like mode) */
  uint64_t bwt_msd_fallback_why;     /* OR over batches of why the MSD path gave up: 1 = bucket > MB_CAP, 2 = cell >
                                        MB_MAXCELL, 4 = tie list > n/8, 8 = tie group > 16, 16 = tie deeper than the resolver */
  uint64_t bwt_direct_fallback_why;  /* the same bits 4 / 8 / 16 for the LSD direct resolve */
  uint64_t dev_peak_bytes;           /* high-water mark of the library's device allocations during the last call */
  /* How the RLE1 stage (rle1.cu) planned, summed over the plans of the last call */
  uint64_t rle_group_scans;    /* plans whose tile scan ran as the multi-CTA group scan (> 8192 tiles, or B2_RLE_SCAN_GROUPS) */
  uint64_t rle_walk_parallel;  /* speculative parallel block walks that chained up and were accepted */
  uint64_t rle_walk_serial;    /* single-CTA block walks: the fallback of a rejected parallel walk, or the only walk */
} b2_stats;
void b2_get_stats(b2_stats* s);

/* Per-block trace of the last compress call (for stage-by-stage parity tests). */
typedef struct b2_block_trace {
  int32_t n, pidx, m, alpha, ngroups, nsel;
  uint32_t crc, pad;
  uint64_t raw_start, raw_len, bit_start, bit_len;
} b2_block_trace;
size_t b2_last_trace(b2_block_trace* out, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* B2BZ_H */
