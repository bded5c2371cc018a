// enc.h -- shared declarations of the encode stages.
#pragma once
#include "ctx.h"

// One bzip2 block as cut by the RLE1 stage (lib/Bzip2.js:636-667 readBlock).
struct BlkInfo {
  u64 s;    // first raw byte
  u64 e;    // one past the last raw byte consumed
  u64 b;    // end of the (re-phased) run the block starts in; == s when the block starts on a run start
  u64 Wb;   // RLE1 output bytes produced by raw[0,b) under maximal-run phases
  u32 ofs;  // RLE1 bytes produced by raw[s,b) with a fresh run state at s
  u32 n;    // post-RLE1 length of the block (<= blockSize)
};

inline u32 rle1_block_size(int level) { return (u32)level * 100000 - 19; }  // lib/Bzip2.js:892-900

struct Rle1Plan {
  DBuf<u32> tile_carry;   // per raw tile: length (mod 255) of the run entering the tile
  DBuf<u64> tile_prefix;  // per raw tile: W(tile start)
  DBuf<u8> tile_plain;    // per raw tile: 1 = no four equal bytes in a row in or into the tile (RLE1 copies it byte for byte)
  DBuf<BlkInfo> blocks;   // device block table
  std::vector<BlkInfo> h_blocks;
  size_t nblocks = 0;      // entries of h_blocks
  size_t first_index = 0;  // global block index of h_blocks[0] (range plans)
  u64 w_total = 0;         // W at the end of the buffer (RLE1 bytes of the whole input up to there); total_guess = ceil(W / BS)
  size_t total_guess(int level) const { return (size_t)((w_total + rle1_block_size(level) - 1) / rle1_block_size(level)); }
};

#define RLE_TILE 4096

// Tile scan (tile_*, w_total).  st0 / W0: run state and RLE1 output in front of the buffer when it is a share of a larger
// input; summary (host, optional): receives the aggregate run state of the buffer and the length of its leading run.
void rle1_scan_tiles(Ctx& c, const u8* d_in, size_t n, Rle1Plan& plan, u64 st0 = 0, u64 W0 = 0, u64* summary = nullptr);
// Cut of blocks [first, first+count) of the whole input from the speculative boundary W = first * blockSize, over a
// plan whose tiles are scanned (exact unless a run-phase slip happened earlier in the input).
void rle1_cut_range(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan, size_t first, size_t count);
// libbz2 flavor over a share buffer d_buf[0, n) = share + halo entered with run state st0 and W base W0
// (b2_bzip2_share_cut_table / b2_bzip2_plan_share_flavor): the cut table of every entry drift 0..dmax into h_table
// (4 u32 per row), and the cut of the blocks [first, first + count) whose first block starts at W = first * blockSize +
// drift.  The table call keeps its tile scan and piece bitmap for the cut that follows on the same buffer and entry
// state; rle1_release_share_probe drops them.
void rle1_share_cut_table(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t share_len, u64 dmax, u32* h_table);
void rle1_cut_share_libbz2(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t first, u64 drift, size_t count,
                           Rle1Plan& plan);
void rle1_release_share_probe();
// Tile scan and exact cut of every block of d_in[0, n) (the flavor of c.bz_flavor).
void rle1_plan(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan);
// materialise blocks [first, first+count) of the plan into the slot layout at d_T (u8[count<<20]);
// d_n receives their lengths, d_crc their CRCs.
void rle1_materialize(Ctx& c, const u8* d_in, size_t n, const Rle1Plan& plan, size_t first, size_t count, u8* d_T, u32* d_n, u32* d_crc);

#define HUFF_MAXSYM 258
#define HUFF_MAXGROUPS 6
#define HUFF_GROUP 50
#define SEL_STRIDE 18432  // per-block stride of the per-group arrays (>= 900001 / 50 + 1)

// The zero-run coder's symbols (0..257) in one byte each.  Only symbol 256 (MTF rank 255) and 257 (the end of
// block in a block that uses 255 or 256 byte values) do not fit; they are rare and go to a bit mask per group.
// `hi` and `any_hi` are zeroed once when they are allocated; every batch then clears the masks of the slots whose
// flag the batch before set (no other slot has a mask bit), so ASCII and text batches clear nothing.
struct NarrowSyms {
  u8* lo;                      // [nblk << SEG_SHIFT] low byte of every symbol (slot layout)
  unsigned long long* hi;      // [nblk][SEL_STRIDE] bit j of word g: symbol 50 g + j is >= 256
  u32* any_hi;                 // [nblk] the block has a symbol >= 256 (most have none, and skip the masks)
};

// MTF + RLE2 (lib/Bzip2.js:743-815): U (slot layout) -> symbols (slot layout), m, freq, used map
void mtf_rle2_batch(Ctx& c, const u8* d_T, const u8* d_U, const u32* d_n, const u32* h_n, u32 nblk, const NarrowSyms& sym, u32* d_m,
                    u32* d_freq /*[nblk][258]*/, u32* d_used /*[nblk][8]*/,
                    const u32* d_bytehist = nullptr /*[nblk][256] byte histograms of the blocks, if known*/);

// per-block result of the Huffman stage
struct HuffBlk {
  u32 ngroups, nsel, alpha, m;
  u64 body_bits;  // bits of the block from the 48-bit magic through the last Huffman code
  u8 len[HUFF_MAXGROUPS][HUFF_MAXSYM + 6];
};
// Table optimisation (lib/Bzip2.js:671-733, 826-843 + HuffmanAllocator.js): selectors u8 (stride SEL_STRIDE), and
// d_goff[blk * SEL_STRIDE + g] = bit offset of group g's codes inside the block's code section (g <= nsel: the last
// entry is the length of the section)
void huffman_batch(Ctx& c, const NarrowSyms& sym, const u32* d_m, const u32* d_freq, const u32* d_used, u32 nblk, u8* d_sel, u8* d_selmtf,
                   HuffBlk* d_hb, u32* d_goff);
// bit packing of blocks at their final bit offsets (lib/Bzip2.js:740-741,749-758,847-874)
void pack_batch(Ctx& c, const NarrowSyms& sym, const u8* d_sel, const u8* d_selmtf, const HuffBlk* d_hb, const u32* d_goff, const u32* d_used,
                const u32* d_pidx, const u32* d_crc, const u64* d_bitoff, const u32* d_flag, u32 nblk, u32 max_m, u32* d_out_words);

#include <vector>
void crc_ranges(Ctx& c, const u8* d_data, const BlkInfo* d_ranges, const std::vector<BlkInfo>& h_ranges, u32* d_crc_out);
u32 crc32_device(Ctx& c, const u8* d_p, size_t n);
void bwt_forward_batch(Ctx& c, const u8* d_T, u8* d_U, const u32* d_n, const u32* h_n, u32 nblk, u32* d_pidx, bool sentinel = false,
                       u32* d_sa_out = nullptr, u32* d_hist_out = nullptr);

// ---- the host-side input and output of the host entry points (implemented in api.cu) ----
// The input: the stream's bytes [base, base + have) in a host buffer.  From a read callback (b2_bzip2_*_stream) the
// buffer doubles as data arrives; over a caller's buffer (the host-buffer calls) every byte is there from the start and
// the buffer is only read.  A callback that aborts throws B2Error{B2_ERR_STREAM}.
struct StreamIn {
  b2_read_fn rd = nullptr; void* user = nullptr;  // null rd: buf is the caller's, borrowed for the call
  cudaStream_t busy = nullptr;  // copies out of buf may be queued here: they are waited for before buf changes
  u8* buf = nullptr;
  size_t cap = 0, base = 0, have = 0;
  bool eof = false;   // read returned 0: the stream is base + have bytes long
  StreamIn(b2_read_fn rd_, void* user_, cudaStream_t busy_) : rd(rd_), user(user_), busy(busy_) {}
  // never written: without rd nothing reads into buf
  StreamIn(const u8* p, size_t n) : buf(const_cast<u8*>(p)), cap(n), have(n), eof(true) {}
  StreamIn(const StreamIn&) = delete;
  ~StreamIn();
  size_t fill(size_t end);  // read until the bytes in front of `end` are here or the input ends; returns base + have
  void drop(size_t pos);    // forget the bytes in front of pos
  const u8* at(size_t pos) const { return buf + (pos - base); }
};
// The output, in pinned buffers of the library's pool (a buffer still held when the sink is destroyed goes back to it).
// With a write callback (b2_bzip2_*_stream) buf stages the pieces, and put() hands each one to the callback once the
// copies into buf on `busy` have landed.  Without one (the host-buffer calls) buf is the result: pieces go at its end,
// put() only counts them, and take() hands the buffer to the caller.
struct StreamOut {
  b2_write_fn wr = nullptr; void* user = nullptr;
  cudaStream_t busy;  // copies into buf are queued here
  u8* buf = nullptr;
  size_t cap = 0;
  u64 written = 0;    // bytes handed over
  StreamOut(b2_write_fn wr_, void* user_, cudaStream_t busy_) : wr(wr_), user(user_), busy(busy_) {}
  explicit StreamOut(cudaStream_t busy_) : busy(busy_) {}
  StreamOut(const StreamOut&) = delete;
  ~StreamOut();
  u8* next() const { return wr ? buf : buf + written; }  // where the next piece's bytes go
  // next() has room for `bytes`.  buf doubles, or takes exactly what is needed when `last` says it will not grow again.
  // A staging buffer drops its contents and doubles no further than `limit`; the result keeps its contents.
  void reserve(size_t bytes, bool last = false, size_t limit = SIZE_MAX);
  void put(const u8* p, size_t n);  // hand over the n bytes at p, which follow those handed over before
  u8* take();                       // the result, never null (also for 0 bytes); released with b2_free
};

// ---- bzip2 encode drivers (encode.cu), one per entry point of include/b2bz.h ----
void bzip2_compress_dev(Ctx& c, const u8* d_in, size_t n, int level, u8* d_out, size_t out_cap, size_t* out_n);
// b2_bzip2_compress and b2_bzip2_compress_stream: the input comes from `in`, the output goes to `out`, which has room for
// out_cap bytes at out.next()
void bzip2_compress_host(Ctx& c, StreamIn& in, int level, u8* d_in, size_t win, u8* d_out, size_t out_cap, StreamOut& out,
                         size_t* out_n, bool pinned_in);
size_t bzip2_plan(Ctx& c, const u8* d_in, size_t n, int level);
void bzip2_plan_spec(Ctx& c, const u8* d_in, size_t n, int level, int rank, int world, u64* info);
void bzip2_share_summary(Ctx& c, const u8* d_in, size_t n, u64* out);
void bzip2_plan_share(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t first, size_t count, u64* info);
void bzip2_share_cut_table(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t share_len, u64 dmax, u32* table);
void bzip2_plan_share_flavor(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t first, size_t count, u64 drift, u64* info);
void bzip2_encode_range(Ctx& c, const u8* d_in, size_t n, int level, size_t first, size_t count, int bit_phase, u8* d_out, size_t out_cap,
                        u64* out_bits, u32* block_crcs);
void bitshift_device(Ctx& c, const void* src, u64 nbits, int phase, void* dst);
void bzip2_release_plan();  // the plan kept for b2_bzip2_encode_range_dev

// Bytes of compressed input on the device at a time in the bzip2 and BWTC decoders, which also caps the output the
// bzip2 decoder stages for the host ($B2_DEC_WINDOW, default 4 GiB: most files are one window; down to 64 KiB as a
// test hook).  Implemented in api.cu.
size_t dec_window();

// ---- BWTC drivers (bwtc.cu), one for each direction: the host-buffer calls run them over a complete source and a
// result sink, the stream calls over read and write callbacks ----
size_t bwtc_bound(size_t n);
// BWTC.compressFile: file_size is the header's size field, or (u64)-1 for "size unknown" (lib/Util.js:118-124)
void bwtc_compress(Ctx& c, StreamIn& in, int level, u64 file_size, StreamOut& out);
// BWTC.decompressFile: every block goes to `out` as soon as its batch is decoded; on a data error the blocks in front of
// the failing check have gone out when the error is thrown
void bwtc_decompress(Ctx& c, StreamIn& in, StreamOut& out);

// ---- bzip2 decode drivers (decode.cu), one per kind of decode ----
// Each throws the reference's first error in stream order.  *out_n: the decoded size, or what the call says on an error.
// b2_bzip2_decompress_dev: d_in[0, n) into d_out, each block at its offset in the decoded stream.  A block that does not
// fit is only counted and the walk goes on past a data error, so a buffer too small throws with *out_n = the size needed.
// flavor: as bzip2_decompress_host's.
void bzip2_decompress_dev(Ctx& c, const u8* d_in, size_t n, int multistream, int flavor, u8* d_out, size_t out_cap, size_t* out_n);
// b2_bzip2_decompress_dev without an output buffer: the blocks are expanded only for their CRCs.
void bzip2_decompress_size(Ctx& c, const u8* d_in, size_t n, int multistream, int flavor, size_t* out_n);
// b2_bzip2_decompress_partial and b2_bzip2_decompress_stream: into `out`, which never receives a byte past the prefix the
// reference writes before an error (*out_n on an error).  flavor B2_BZ2_LIBBZ2 reads as libbz2 reads (b2_bzip2_decompress_flavor).
void bzip2_decompress_host(Ctx& c, StreamIn& in, int multistream, int flavor, StreamOut& out, size_t* out_n);
// What the replay of a table or a position list records in front of the first failure: per block its bit position and
// decoded length (the table rows), and per position the end of its bytes in the output (the list ends).
struct DecRows { std::vector<u64> pos, ends; std::vector<u32> len; };
// b2_bzip2_table_partial: the rows of the blocks in front of the first failure (stream CRCs are not checked).
void bzip2_table(Ctx& c, StreamIn& in, int multistream, DecRows& rows, size_t* out_n);
// b2_bzip2_decompress_blocks: the blocks at a non-empty list of bit positions, back to back in list order, from a complete
// input; rows.ends, and *out_n on an error, as bzip2_decompress_host's.
void bzip2_decompress_list(Ctx& c, StreamIn& in, const std::vector<u64>& positions, StreamOut& out, DecRows& rows, size_t* out_n);
// b2_bzip2_recover and b2_bzip2_recover_stream: one row per block magic of `in`, in position order, and into `out` the
// intact blocks' bytes or (repair) the repaired stream.  Damage is a result, not an error: only a CUDA failure or a
// callback abort throws.
void bzip2_recover(Ctx& c, StreamIn& in, bool repair, StreamOut& out, std::vector<b2_recovered_block>& rows);
// The sharded decodes (b2_dec_shard_open / _export / _finish over the whole input, b2_dec_share_open / _export / _finish
// over shares): one session of either kind at a time, ended by finish or by the next open, or released by b2_shutdown.
// The session reads in the flavor it was opened with.
void dec_shard_open(Ctx& c, const u8* d_in, size_t n, int rank, int world, int flavor, u64* info);
void dec_shard_export(u64* buf);
void dec_shard_finish(const u64* all, int multistream, u8* d_out, size_t out_cap, u64* res);
void dec_share_open(Ctx& c, const u8* d_buf, size_t hold, u64 g0, size_t share_len, size_t total, int flavor, u64* info);
void dec_share_export(u64* buf);
void dec_share_finish(const u64* all, size_t count, int multistream, u8* d_out, size_t out_cap, u64* res);
void dec_shard_release();
// BWT.unbwtransform of nb blocks at once (BWTC decode, b2_bwt_inverse): block b is the L column in slot b of d_L, h_n[b]
// bytes (1 <= n <= 2^20 - 2) with primary index h_pidx[b] (0 <= pidx <= n); the blocks go to d_out back to back.
void bwt_inverse_sentinel_batch(Ctx& c, const u8* d_L, const u32* h_n, const u32* h_pidx, u32 nb, u8* d_out);
