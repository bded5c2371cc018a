// decode.cu -- many-block parallel bzip2 decode on the GPU.
//
// Reference: lib/Bzip2.js:90-548 (Bunzip: _start_bunzip, _get_next_block, _read_bunzip, decode,
// decodeBlock, table).  The reference decodes strictly serially, one bit at a time.  Here:
//
//   k_scan_magic   : every bit offset is tested for the 48-bit block / end-of-stream magics
//                    (blocks start at arbitrary bit positions and a .bz2 has no index)
//   k_magic_at     : the same test at caller-given bit positions only (decompressBlock / decompressBlocks)
//   k_hdec         : one CTA (4 warps) per candidate block: header parse (symbol map, selectors, code
//                    length tables -- lib/Bzip2.js:137-275), canonical decode tables exactly as the
//                    reference builds them (limit/base/permute) plus a 9-bit LUT derived from them,
//                    then the Huffman symbol stream (lib/Bzip2.js:288-307): per 50-symbol group the
//                    (symbol, length) that would start at EVERY bit offset of a window, jump tables
//                    1/2/4 symbols ahead, and one thread following 13 jumps
//   k_unmtf_a/scan/map: RUNA/RUNB expansion and inverse move-to-front (lib/Bzip2.js:312-361), chunk
//                    parallel: one serial list pass per chunk that records start-list POSITIONS and
//                    the chunk's composite permutation, a per-block scan over the chunks, then a
//                    lane-parallel pass that maps positions to bytes and expands the runs
//   inverse BWT    : T-vector by one onesweep radix pass on the L column (lib/Bzip2.js:370-381),
//                    then the n-step pointer chase (lib/Bzip2.js:418-423) is broken into ~7000
//                    independent walks per block between sampled rows; every walk records the bytes
//                    it passes, a serial pass over the 7000 walk summaries orders them, and the block
//                    is assembled by copies (only what lies behind a walk's 512-byte record is
//                    walked again)
//   bwt_inverse_sentinel_batch: BWT.unbwtransform (lib/BWT.js:352-363) of a batch of blocks on the same walk kernels
//   k_derand       : libbz2 flavor only: the flipped bytes of randomised blocks, XORed in place before RLE1 decode
//   k_unrle_*      : RLE1 decode (lib/Bzip2.js:424-436): count bytes are identified from local
//                    synchronisation points (8 bytes per thread, decided in registers), output
//                    offsets from tile sums + one warp scan per block, tiles expanded in shared
//                    memory, CRC32 per block
//   host           : one driver per kind of decode (enc.h).  A chain decode is one rolling loop over windows of
//                    the compressed input (DecIn: a host source or a device buffer) and batches of blocks: it walks
//                    the block chain (a block must start exactly where the previous one ended) after every batch,
//                    folds/validates CRCs, delivers the settled blocks (to a device buffer, a host sink, or only
//                    for their CRCs) and raises the reference's errors in stream order.  A position list uploads
//                    the whole input once and walks its blocks in list order, without a chain.  The sharded decodes
//                    run the same batch, walk and device delivery over the whole file or a rank's share.  Block recovery walks every
//                    candidate by intactness instead of by the chain and splices the intact blocks' bits (k_splice).
#include <algorithm>
#include <memory>
#include <vector>
#include "enc.h"
#include "radix.cuh"
#include "radix_host.cuh"

#define WHOLEPI 0x314159265359ull
#define SQRTPI 0x177245385090ull
#define SEL_CAP 32768
#define DEC_OK 0
#define DEC_NOT_BZIP (-2)
#define DEC_EOF (-3)
#define DEC_DATA_ERROR (-5)
#define DEC_OBSOLETE (-7)

struct Cand {
  u64 pos;     // bit position of the magic
  u32 type;    // 1 = block, 2 = end of stream
  u32 next32;  // the 32 bits that follow the magic (block CRC / stream CRC)
};

struct CandRes {
  int status;      // 0 or a (negative) reference error code
  u32 detail;      // 1 = "initial position out of bounds"
  u32 m;           // decoded symbols incl. EOB
  u32 orig;        // origPointer
  u32 sym_total;   // distinct bytes
  u32 n;           // block length after un-MTF (filled later)
  u32 rawlen;      // bytes after RLE1 decode (filled later)
  u32 open;        // 1 = decoding it read up to the end of an input window that is not the end of the file: not final
  u32 rand;        // libbz2 flavor only: the randomised bit is set (the compressjs flavor fails the block instead)
  u32 run4;        // the pre-RLE1 bytes end on the fourth byte of a run, without its count byte (k_unrle_tileoff)
  u64 endbit;      // bit position just behind the EOB code
  u8 sym_to_byte[256];
};

// ---- magic test -----------------------------------------------------------------------------
// The words wi .. wi+3 of the stream (big endian) hold the 80 bits that a candidate starting in word wi can span: the
// 48-bit magic and the 32 bits behind it.  The device copy of the input (window) is zero padded: for wi < (n + 3) / 4
// the reads stay below n + 32.
struct MagicWords { u32 w0, w1, w2, w3; };
__device__ __forceinline__ MagicWords magic_words(const u8* __restrict__ in, u64 wi) {
  const u32* words = reinterpret_cast<const u32*>(in);
  return {__byte_perm(words[wi], 0, 0x0123), __byte_perm(words[wi + 1], 0, 0x0123), __byte_perm(words[wi + 2], 0, 0x0123),
          __byte_perm(words[wi + 3], 0, 0x0123)};
}
// Is there a magic at bit pos = 32 wi + b of the buffer, pos < lim?  If so, found(type, next32): type 1 = block, 2 = end
// of stream, next32 = the 32 bits behind it.  The first 32 bits of the magic are tested with one funnel shift and one
// compare; the rest, rarely reached, sits inside that branch (a callback rather than a return value keeps the scan loop
// free of a second branch per offset).
template <class F>
__device__ __forceinline__ void magic_test(const MagicWords& w, u32 b, u64 pos, u64 lim, F&& found) {
  const u32 M1 = (u32)(WHOLEPI >> 16), M2 = (u32)(SQRTPI >> 16);
  const u32 h = __funnelshift_l(w.w1, w.w0, b);          // stream bits [b, b + 32) of this word pair
  if (h == M1 || h == M2) {
    const u32 mid = __funnelshift_l(w.w2, w.w1, b);      // bits [b + 32, b + 64)
    const u64 v = ((u64)h << 16) | (mid >> 16);
    if ((v == WHOLEPI || v == SQRTPI) && pos < lim) {
      const u32 lo = __funnelshift_l(w.w3, w.w2, b);     // bits [b + 64, b + 96)
      found(v == WHOLEPI ? 1u : 2u, (mid << 16) | (lo >> 16));
    }
  }
}

// ---- magic scan ---------------------------------------------------------------------------
// One thread per aligned 32-bit word of the n-byte window = 32 bit offsets.  The window starts at bit base_bit of the
// file (a multiple of 32); magics at window offsets below lim are recorded, with their position in the file.
__global__ void k_scan_magic(const u8* __restrict__ in, u64 n, u64 base_bit, u64 lim, Cand* __restrict__ cands, u32* count, u32 cap) {
  const u64 wi = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (wi >= (n + 3) / 4) return;
  const MagicWords w = magic_words(in, wi);
#pragma unroll 8
  for (u32 b = 0; b < 32; b++) {
    const u64 pos = wi * 32 + b;
    magic_test(w, b, pos, lim, [&](u32 type, u32 next32) {
      const u32 idx = atomicAdd(count, 1u);
      if (idx < cap) {
        Cand c;
        c.pos = base_bit + pos; c.type = type; c.next32 = next32;
        cands[idx] = c;
      }
    });
  }
}

// ---- magic at given positions -----------------------------------------------------------------
// One thread per requested bit position (a list decode: no scan of the whole stream).  type 0: no magic there.
__global__ void k_magic_at(const u8* __restrict__ in, u64 n, const u64* __restrict__ pos, u64 count, Cand* __restrict__ cands) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  Cand c;
  c.pos = pos[i]; c.type = 0; c.next32 = 0;
  if (c.pos < n * 8)  // no reads past the stream
    magic_test(magic_words(in, c.pos >> 5), (u32)(c.pos & 31), c.pos, n * 8, [&](u32 type, u32 next32) { c.type = type; c.next32 = next32; });
  cands[i] = c;
}

// ---- bit reader (one thread) ----------------------------------------------------------------
struct BitReader {
  const u32* words; u64 nwords; u64 widx; u64 buf; u32 avail;
  __device__ __forceinline__ u32 fetch() {
    u32 w = widx < nwords ? words[widx] : 0u;  // bits past EOF read as zeros (lib/BitStream.js:88-89)
    widx++;
    return __byte_perm(w, 0, 0x0123);
  }
  __device__ __forceinline__ void init(const u8* base, u64 nbytes, u64 bitpos) {
    words = reinterpret_cast<const u32*>(base);
    nwords = (nbytes + 3) / 4;  // the input buffer is zero padded to a multiple of 4 (+16)
    widx = bitpos >> 5;
    const u32 skip = (u32)(bitpos & 31);
    buf = (u64)fetch() << 32;
    buf <<= skip;
    avail = 32 - skip;
  }
  __device__ __forceinline__ void ensure() {
    if (avail <= 32) { buf |= (u64)fetch() << (32 - avail); avail += 32; }
  }
  __device__ __forceinline__ u32 peek(u32 k) { return k ? (u32)(buf >> (64 - k)) : 0u; }
  __device__ __forceinline__ void skip(u32 k) { buf <<= k; avail -= k; }
  __device__ __forceinline__ u32 get(u32 k) { ensure(); u32 v = peek(k); skip(k); return v; }
  __device__ __forceinline__ u64 tell() const { return widx * 32 - avail; }
};

// ---- header + Huffman decode: one CTA per candidate ------------------------------------------
// One CTA per block.  The per-group phases are spread over the CTA's warps, and a block's ~18 000 groups are strictly
// serial, so a launch lasts as long as one block takes: with all SM slots taken (10 x 128 threads on 132 SMs: 1320 blocks,
// a 1 GiB file) four warps per block give the best throughput; with fewer blocks the same thread budget goes to fewer, wider CTAs
// (256 or 512 threads: fewer window offsets per thread, a shorter group).
#define HD_THREADS 128
#define HD_LUT_BITS 9   // 6 tables x 512 entries: keeps a warp's state under 19 KB so that 12 blocks fit per SM
#define HD_WIN 512
#define HD_STAGE 64
struct HdecWarp {
  int limit[HUFF_MAXGROUPS][22];
  int base[HUFF_MAXGROUPS][22];
  u16 permute[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];
  u16 lut[HUFF_MAXGROUPS][1 << HD_LUT_BITS];
  u8 len[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];
  int minlen[HUFF_MAXGROUPS], maxlen[HUFF_MAXGROUPS];
  int status; u32 ngroups, nsel, symcount;
  // speculative window decode of the symbol stream
  u32 win[HD_STAGE + 20]; // staged stream words (big-endian), refilled every ~2048 bits
  u16 wsym[HD_WIN + 32]; // symbol that would start at every bit offset of the window; tail stays 0
  u8 wlen[HD_WIN + 32]; // its code length (0 = no valid code there); tail stays 0
  u16 spos[HUFF_GROUP + 6];
  u16 J1[HD_WIN + 32], J2[HD_WIN + 32], J4[HD_WIN + 32];  // chain jump tables: 1, 2 and 4 symbols ahead
  u16 q4[16];
  u32 c_cnt, c_pos, c_flag;
  u64 P0;
};

// code longer than the LUT covers: the reference's limit search (lib/Bzip2.js:296-306); returns sym | len << 9,
// 0 when no code of the table starts with these 20 bits
__device__ __noinline__ u32 hdec_slow(const HdecWarp& s, u32 g, u32 bits20, int minLen, int maxLen) {
  int i = minLen;
  int j = (int)(bits20 >> (20 - i));
  for (;;) {
    if (i > maxLen) return 0;                                            // :299
    if (j <= s.limit[g][i]) break;
    i++;
    if (i > 20) return 0;
    j = (int)(bits20 >> (20 - i));
  }
  const int jj = j - s.base[g][i];
  if (jj >= 0 && jj < HUFF_MAXSYM) return (u32)s.permute[g][jj] | ((u32)i << 9);  // :306
  return 0;
}

// 128 threads: 10 CTAs per SM (45 registers, 19 KB of shared memory each), so that the ~1200 blocks of a 1 GiB file are
// resident at once on the 132 SMs of an H100.  At 9 per SM (1188 slots) the last blocks ran as a second wave: 66 ms
// instead of 44 ms per GiB (H100 SXM, 400 W power limit).
// The input is a window of nbytes bytes that starts at bit base_bit of the file (a multiple of 32) and is zero padded
// behind; candidate positions and endbit are bits of the file.  A result that depends on no bit at or past the window's
// end is what the whole file gives; any other is marked open unless the window ends where the file does (`last`).
// LB (the libbz2 flavor) decodes a randomised block (its bytes are derandomised after the inverse BWT: k_derand) and
// rejects a selector MTF code of groupCount ones, as libbz2 does; without it this is the reference's decoder, which
// leaves `rand` unset.  A template argument, so that the compressjs flavor's kernel is compiled as before.
template <int HD_T, bool LB>
__global__ void __launch_bounds__(HD_T, HD_T == 128 ? 10 : 1152 / HD_T)
k_hdec(const u8* __restrict__ in, u64 nbytes, u64 base_bit, u32 last, const Cand* __restrict__ cands, u32 count, u32 dbuf_size,
       u8* __restrict__ sel_buf, u16* __restrict__ sym_out, CandRes* __restrict__ res) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  HdecWarp& s = *reinterpret_cast<HdecWarp*>(smem_raw);
  const u32 lane = threadIdx.x;  // 0..HD_T-1: one CTA per candidate block
  const u32 ci = blockIdx.x;
  if (ci >= count) return;
  const Cand cd = cands[ci];
  CandRes* r = res + ci;
  u8* sel = sel_buf + (size_t)ci * SEL_CAP;
  u16* so = sym_out + ((size_t)ci << SEG_SHIFT);
  BitReader br;
  u32 symTotal = 0;
  if (lane == 0) {
    s.status = 0;
    r->detail = 0; r->m = 0; r->n = 0; r->rawlen = 0; r->endbit = 0;
    br.init(in, nbytes, cd.pos - base_bit + 48 + 32);
    do {
      if (LB) r->rand = br.get(1);
      else if (br.get(1)) { s.status = DEC_OBSOLETE; break; }           // lib/Bzip2.js:143
      const u32 orig = br.get(24);
      r->orig = orig;
      if (orig > dbuf_size) { s.status = DEC_DATA_ERROR; r->detail = 1; break; }  // :146
      const u32 t16 = br.get(16);
      for (int i = 0; i < 16; i++) {
        if (t16 & (1u << (15 - i))) {
          const u32 k = br.get(16);
          for (int j = 0; j < 16; j++)
            if (k & (1u << (15 - j))) r->sym_to_byte[symTotal++] = (u8)(i * 16 + j);
        }
      }
      const u32 gc = br.get(3);
      if (gc < 2 || gc > 6) { s.status = DEC_DATA_ERROR; break; }    // :167
      const u32 ns = br.get(15);
      if (ns == 0) { s.status = DEC_DATA_ERROR; break; }             // :174
      u8 mtf[HUFF_MAXGROUPS + 2];  // the reference's list is a zero-filled 256-entry buffer: slot gc reads as 0
      for (u32 i = 0; i < HUFF_MAXGROUPS + 2; i++) mtf[i] = (u8)(i < gc ? i : 0);
      bool bad = false;
      const u32 jmax = LB ? gc - 1 : gc;  // the most ones a selector's MTF code may have
      for (u32 i = 0; i < ns && !bad; i++) {
        u32 j = 0;
        while (br.get(1)) { if (j >= jmax) { bad = true; break; } j++; }   // :184-185
        if (bad) break;
        const u8 v = mtf[j];
        for (u32 k = j; k > 0; k--) mtf[k] = mtf[k - 1];
        mtf[0] = v;
        sel[i] = v;
      }
      if (bad) { s.status = DEC_DATA_ERROR; break; }
      const u32 symCount = symTotal + 2;
      for (u32 g = 0; g < gc && !bad; g++) {
        int t = (int)br.get(5);
        for (u32 i = 0; i < symCount; i++) {
          for (;;) {
            if (t < 1 || t > 20) { bad = true; break; }               // :203
            if (!br.get(1)) break;
            if (!br.get(1)) t++; else t--;
          }
          if (bad) break;
          s.len[g][i] = (u8)t;
        }
      }
      if (bad) { s.status = DEC_DATA_ERROR; break; }
      s.ngroups = gc; s.nsel = ns; s.symcount = symCount;
    } while (0);
    r->sym_total = symTotal;
  }
  __syncthreads();
  if (s.status != 0) {
    // a header error is decided by the bits read so far
    if (lane == 0) { r->status = s.status; r->open = !last && br.tell() > nbytes * 8; }
    return;
  }
  const u32 gc = s.ngroups, symCount = s.symcount;
  // ---- limit / base / permute exactly as lib/Bzip2.js:216-274, one lane per table ----
  if (lane < gc) {
    const u32 g = lane;
    int minLen = s.len[g][0], maxLen = s.len[g][0];
    for (u32 i = 1; i < symCount; i++) {
      const int l = s.len[g][i];
      if (l > maxLen) maxLen = l; else if (l < minLen) minLen = l;
    }
    s.minlen[g] = minLen; s.maxlen[g] = maxLen;
    int temp[22];
    for (int i = 0; i < 22; i++) { temp[i] = 0; s.limit[g][i] = 0; s.base[g][i] = 0; }
    for (u32 i = 0; i < HUFF_MAXSYM; i++) s.permute[g][i] = 0;
    int pp = 0;
    for (int i = minLen; i <= maxLen; i++)
      for (u32 t = 0; t < symCount; t++)
        if (s.len[g][t] == i) s.permute[g][pp++] = (u16)t;
    for (u32 i = 0; i < symCount; i++) temp[s.len[g][i]]++;
    pp = 0;
    int t = 0;
    for (int i = minLen; i < maxLen; i++) {
      pp += temp[i];
      s.limit[g][i] = pp - 1;
      pp <<= 1;
      t += temp[i];
      s.base[g][i + 1] = pp - t;
    }
    s.limit[g][maxLen] = pp + temp[maxLen] - 1;
    s.base[g][minLen] = 0;
  }
  __syncthreads();
  // ---- LUT (HD_LUT_BITS bits) derived from the reference's decode loop (lib/Bzip2.js:296-307) ----
  for (u32 e = lane; e < gc << HD_LUT_BITS; e += HD_T) {
    const u32 g = e >> HD_LUT_BITS, p = e & ((1u << HD_LUT_BITS) - 1);
    const int minLen = s.minlen[g], maxLen = s.maxlen[g];
    u16 ent = 0;  // 0 = needs more than HD_LUT_BITS bits (or fails): take the slow path
    int i = minLen;
    if (i <= HD_LUT_BITS) {
      int j = (int)(p >> (HD_LUT_BITS - i));
      for (;;) {
        if (i > maxLen) break;
        if (j <= s.limit[g][i]) {
          const int jj = j - s.base[g][i];
          if (jj >= 0 && jj < HUFF_MAXSYM) ent = (u16)((i << 9) | s.permute[g][jj]);
          break;
        }
        i++;
        if (i > HD_LUT_BITS) break;
        j = (j << 1) | (int)((p >> (HD_LUT_BITS - i)) & 1);
      }
    }
    s.lut[g][p] = ent;
  }
  __syncthreads();
  // ---- symbol stream (lib/Bzip2.js:288-307).  Per 50-symbol group the table is fixed, so all 32
  // lanes decode the (symbol, length) that WOULD start at every bit offset of a 512-bit window, and
  // lane 0 only follows the chain pos += len[pos] through shared memory; the symbols on the chain are
  // then written out by the whole warp. ----
  {
    const u32 ns = s.nsel, eob = s.symcount - 1;  // symTotal + 1
    if (lane == 0) s.P0 = br.tell();
    __syncthreads();
    u64 P = s.P0;
    const u32* words = reinterpret_cast<const u32*>(in);
    const u64 nwords = (nbytes + 3) / 4;
    u32 m = 0, selector = 0;
    int status = 0;
    bool done = false;
    if (lane < 32) { s.wlen[HD_WIN + lane] = 0; s.wsym[HD_WIN + lane] = 0; }
    u64 stage_w0 = ~0ull;  // index of the stream word held in win[0]
    u32 wlim = HD_WIN;     // bit offsets decoded per window: adapts to the size of the previous group
    __syncthreads();
    while (!done) {
      if (selector >= ns) { status = DEC_DATA_ERROR; break; }          // :291
      const u32 g = sel[selector++];
      const u16* lut = s.lut[g];
      const int minLen = s.minlen[g], maxLen = s.maxlen[g];
      u32 remaining = HUFF_GROUP;
      while (remaining && !done) {
        // (re)stage HD_STAGE + 18 words when the 544-bit window would leave the staged range
        const u64 w0 = P >> 5;
        if (stage_w0 == ~0ull || w0 < stage_w0 || w0 + 18 > stage_w0 + HD_STAGE + 18) {
          __syncthreads();
          for (u32 i = lane; i < HD_STAGE + 18; i += HD_T) {
            const u64 wi = w0 + i;
            const u32 wv = wi < nwords ? words[wi] : 0u;
            s.win[i] = __byte_perm(wv, 0, 0x0123);
          }
          stage_w0 = w0;
          __syncthreads();
        }
        const u32 shiftbase = (u32)(P & 31);
        u32 j1r[HD_WIN / HD_T], j2r[HD_WIN / HD_T];  // this thread's jump targets, kept in registers between the passes
        {
          // thread t decodes offsets t, t+128, ...: same bit shift every time
          const u32 sh = (shiftbase + lane) & 31;
          const u32* wp = s.win + (u32)(w0 - stage_w0) + ((shiftbase + lane) >> 5);
#pragma unroll
          for (u32 k = 0; k < HD_WIN / HD_T; k++) {
            const u32 o = lane + HD_T * k;
            j1r[k] = o;
            if (o < wlim) {
              const u32 hiw = wp[(HD_T / 32) * k], low = wp[(HD_T / 32) * k + 1];
              const u32 bits20 = __funnelshift_l(low, hiw, sh) >> 12;
              u32 ent = lut[bits20 >> (20 - HD_LUT_BITS)];
              if (!ent) ent = hdec_slow(s, g, bits20, minLen, maxLen);
              const u32 len = ent >> 9;
              s.wsym[o] = (u16)(ent & 511u);
              s.wlen[o] = (u8)len;
              // J1[o] = o + len[o] (an offset without a code maps to itself, one beyond the window parks there)
              j1r[k] = min(o + len, wlim + 31u);
              s.J1[o] = (u16)j1r[k];
            }
          }
        }
        if (lane < 32) {
          // everything behind the decoded window parks the chain
          const u32 o = wlim + lane;
          s.wlen[o] = 0; s.wsym[o] = 0;
          s.J1[o] = (u16)o; s.J2[o] = (u16)o; s.J4[o] = (u16)o;
        }
        __syncthreads();
#pragma unroll
        for (u32 k = 0; k < HD_WIN / HD_T; k++)
          if (lane + HD_T * k < wlim) j2r[k] = s.J1[j1r[k]];
#pragma unroll
        for (u32 k = 0; k < HD_WIN / HD_T; k++)
          if (lane + HD_T * k < wlim) s.J2[lane + HD_T * k] = (u16)j2r[k];
        __syncthreads();
#pragma unroll
        for (u32 k = 0; k < HD_WIN / HD_T; k++)
          if (lane + HD_T * k < wlim) j1r[k] = s.J2[j2r[k]];
#pragma unroll
        for (u32 k = 0; k < HD_WIN / HD_T; k++)
          if (lane + HD_T * k < wlim) s.J4[lane + HD_T * k] = (u16)j1r[k];
        __syncthreads();
        if (lane == 0) {
          // the only serial part: 13 dependent shared-memory loads cover 52 symbols
          u32 pos = 0;
#pragma unroll
          for (u32 i = 0; i < 13; i++) { s.q4[i] = (u16)pos; pos = s.J4[pos]; }
        }
        __syncthreads();
        if (lane < 13) {
          const u32 p0 = s.q4[lane], p1 = s.J1[p0], p2 = s.J1[p1], p3 = s.J1[p2];
          s.spos[4 * lane] = (u16)p0; s.spos[4 * lane + 1] = (u16)p1; s.spos[4 * lane + 2] = (u16)p2; s.spos[4 * lane + 3] = (u16)p3;
        }
        __syncthreads();
        if (lane < 32) {
          // first warp: where does the group stop inside this window?
          const u32 lim = remaining;  // <= 50
          u32 first_stop = 0xffffffffu, first_eob = 0xffffffffu;
          for (u32 i = lane; i < lim; i += 32) {
            const u32 p = s.spos[i];
            if (s.wlen[p] == 0 && first_stop == 0xffffffffu) first_stop = i;  // no code here, or past the window
            const u32 sy = s.wsym[p];
            if (sy >= eob && sy > 1 && first_eob == 0xffffffffu) first_eob = i;
          }
          first_stop = __reduce_min_sync(FULL_MASK, first_stop);
          first_eob = __reduce_min_sync(FULL_MASK, first_eob);
          u32 cntw = lim, flag = 0;
          if (first_eob < first_stop && first_eob < lim) { cntw = first_eob + 1; flag = 1; }
          else if (first_stop < lim) { cntw = first_stop; flag = (s.spos[first_stop] < wlim) ? 2u : 0u; }  // :299/:306 vs. window exhausted
          if (lane == 0) { s.c_cnt = cntw; s.c_pos = s.spos[cntw]; s.c_flag = flag; }
        }
        __syncthreads();
        const u32 cnt = s.c_cnt, flag = s.c_flag;
        if (m + cnt >= SEG_SIZE) { status = DEC_DATA_ERROR; done = true; break; }
        if (lane < cnt) so[m + lane] = s.wsym[s.spos[lane]];  // cnt <= 50
        m += cnt;
        remaining -= cnt;
        P += s.c_pos;
        {
          // next window: enough for a whole group at the current bits/symbol plus slack
          const u32 est = cnt ? (s.c_pos * HUFF_GROUP) / cnt + 64u : HD_WIN;
          wlim = min((u32)HD_WIN, max(96u, (est + 31u) & ~31u));
        }
        if (flag == 2) { status = DEC_DATA_ERROR; done = true; }
        else if (flag == 1) done = true;
        __syncthreads();
      }
    }
    if (lane == 0) {
      r->status = status;
      r->m = m;
      r->endbit = base_bit + P;
      // a block that ends well is decided by the bits in front of its end; a failure by at most a window of codes
      // behind P (the speculative decode reads HD_WIN + 20 bits ahead)
      const u64 hi = status == 0 ? P : P + HD_WIN + 32;
      r->open = !last && hi > nbytes * 8;
    }
  }
}

// ---- inverse MTF + run expansion --------------------------------------------------------------
#define UM_CHUNK 4096
#define UM_WARPS 8
struct ChunkSum {
  u64 leadval;   // sum (d_j+1) << j over the leading run digits
  u32 nlead;     // number of leading run digits
  u32 rest;      // bytes produced by everything behind the leading digits
  u32 trail;     // run digits at the end of the chunk
  u32 allrun;    // chunk consists of run digits only
  u32 nsyms;
  u32 bad;
};

// One THREAD per 4 Ki-symbol chunk: the serial list pass of the reference (lib/Bzip2.js:355-360) on a private list that
// starts as the identity, so what comes out are POSITIONS IN THE CHUNK'S START LIST (k_unmtf_map turns them into bytes
// once k_unmtf_scan has composed the chunks' final lists).  The list lives in shared memory as 64-bit words, word k of
// thread t at [k][t]: no bank conflicts, whatever word a lane touches.  Moving list[idx] to the front shifts idx/8
// words by one byte: a short loop whose length follows the rank (small on anything compressible), against the 48
// warp instructions per symbol of a warp-wide register list.
#define UA_THREADS 128
__global__ void __launch_bounds__(UA_THREADS)
k_unmtf_a(const u16* __restrict__ sym, const CandRes* __restrict__ res, u32 ncand, u32 cps, ChunkSum* __restrict__ sums, u8* __restrict__ perms,
          u8* __restrict__ symb) {
  __shared__ u64 W[32][UA_THREADS];
  const u32 t = threadIdx.x;
  const u32 gchunk = blockIdx.x * UA_THREADS + t;
  const u32 ci = gchunk / cps, ch = gchunk % cps;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 m = r->m;
  const u32 start = ch * UM_CHUNK;
  if (start >= m) return;
  const u32 count = min((u32)UM_CHUNK, m - start);
  const u16* s = sym + ((size_t)ci << SEG_SHIFT) + start;
  const u32 symTotal = r->sym_total;
#pragma unroll 8
  for (u32 k = 0; k < 32; k++) W[k][t] = 0x0706050403020100ull + k * 0x0808080808080808ull;  // identity list
  u64 leadval = 0; u32 nlead = 0, rest = 0, krun = 0, bad = 0;
  bool seen_lit = false;
  u8* sb = symb + ((size_t)ci << SEG_SHIFT) + start;
  u32 front = 0;
  for (u32 base = 0; base < count; base += 8) {
    // eight symbols per step: one 16-byte load, one 8-byte store (the slot is 1 MiB: reading past `count` stays inside it)
    const uint4 q = *reinterpret_cast<const uint4*>(s + base);
    const u32 qw[4] = {q.x, q.y, q.z, q.w};
    u32 keep_lo = 0, keep_hi = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const u32 sy = (qw[j >> 1] >> (16 * (j & 1))) & 0xffffu;
      if (base + j < count) {
        if (sy <= 1) {
          if (!seen_lit) {
            if (nlead < 21) leadval += (u64)(sy + 1) << nlead; else bad = 1;   // >= 2^21 bytes: over any dbufSize
            nlead++;
          } else {
            if (krun < 21) rest = min(rest + ((sy + 1) << krun), 0x3fffffffu); else bad = 1;  // saturate: no wrap-around
            krun++;
          }
        } else {
          seen_lit = true; krun = 0;
          if (sy <= symTotal) {
            const u32 idx = sy - 1, wq = idx >> 3, bp = idx & 7u;
            const u64 x = W[wq][t];
            const u32 b = (u32)(x >> (8 * bp)) & 0xffu;
            u64 carry = b;
            for (u32 k = 0; k < wq; k++) {
              const u64 y = W[k][t];
              W[k][t] = (y << 8) | carry;
              carry = y >> 56;
            }
            const u64 msk = bp == 7 ? ~0ull : ((1ull << (8 * (bp + 1))) - 1ull);
            W[wq][t] = (((x << 8) | carry) & msk) | (x & ~msk);
            front = b;
            rest++;
          }
        }
      }
      if (j < 4) keep_lo |= front << (8 * j); else keep_hi |= front << (8 * (j - 4));
    }
    *reinterpret_cast<uint2*>(sb + base) = make_uint2(keep_lo, keep_hi);
  }
  {
    ChunkSum cs;
    cs.leadval = leadval; cs.nlead = nlead; cs.rest = rest; cs.trail = seen_lit ? krun : nlead; cs.allrun = seen_lit ? 0u : 1u;
    cs.nsyms = count; cs.bad = bad;
    sums[gchunk] = cs;
  }
  u64* p = reinterpret_cast<u64*>(perms + (size_t)gchunk * 256);
#pragma unroll 8
  for (u32 k = 0; k < 32; k++) p[k] = W[k][t];
}

struct ChunkStart {
  u32 k;    // run digits immediately before the chunk
  u32 off;  // output offset of the chunk
};

__global__ void __launch_bounds__(32)
k_unmtf_scan(CandRes* __restrict__ res, u32 ncand, u32 cps, u32 dbuf_size, const ChunkSum* __restrict__ sums, const u8* __restrict__ perms,
             u8* __restrict__ lists, ChunkStart* __restrict__ starts) {
  __shared__ u8 L[256], P[256];
  const u32 ci = blockIdx.x, lane = threadIdx.x;
  CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 m = r->m;
  const u32 nch = (m + UM_CHUNK - 1) / UM_CHUNK;
  for (u32 i = lane; i < 256; i += 32) L[i] = (u8)i;
  __syncwarp();
  u64 off = 0; u32 k = 0; int status = 0;
  for (u32 ch = 0; ch < nch; ch++) {
    const size_t gc = (size_t)ci * cps + ch;
    const ChunkSum cs = sums[gc];
    for (u32 i = lane; i < 256; i += 32) { lists[gc * 256 + i] = L[i]; P[i] = perms[gc * 256 + i]; }
    if (lane == 0) { ChunkStart st; st.k = k; st.off = (u32)off; starts[gc] = st; }
    if (cs.bad || (cs.nlead && k + cs.nlead > 32)) { status = DEC_DATA_ERROR; break; }
    off += (cs.leadval << k) + cs.rest;
    if (off > dbuf_size) { status = DEC_DATA_ERROR; break; }        // lib/Bzip2.js:338,354
    k = cs.allrun ? k + cs.nsyms : cs.trail;
    __syncwarp();
    u8 nl[8];
    for (int j = 0; j < 8; j++) nl[j] = L[P[lane * 8 + j]];
    __syncwarp();
    for (int j = 0; j < 8; j++) L[lane * 8 + j] = nl[j];
    __syncwarp();
  }
  if (lane == 0) {
    if (!status && r->orig >= (u32)off) status = DEC_DATA_ERROR;      // lib/Bzip2.js:368
    r->status = status;
    r->n = (u32)off;
  }
}

// Second pass, fully lane parallel: byte = sym_to_byte[start list[symb]], run digit i of a run weighs
// (digit+1) << i (lib/Bzip2.js:312-361); output offsets by a warp scan of the weights.
__global__ void __launch_bounds__(UM_WARPS * 32)
k_unmtf_map(const u16* __restrict__ sym, const u8* __restrict__ symb, const CandRes* __restrict__ res, u32 ncand, u32 cps,
            const u8* __restrict__ lists, const ChunkStart* __restrict__ starts, u8* __restrict__ tt) {
  __shared__ u8 Ts[UM_WARPS][256];
  const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const u32 gchunk = blockIdx.x * UM_WARPS + w;
  const u32 ci = gchunk / cps, ch = gchunk % cps;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 m = r->m;
  const u32 start = ch * UM_CHUNK;
  if (start >= m) return;
  const u32 count = min((u32)UM_CHUNK, m - start);
  const u16* s = sym + ((size_t)ci << SEG_SHIFT) + start;
  const u8* sb = symb + ((size_t)ci << SEG_SHIFT) + start;
  const u32 symTotal = r->sym_total;
  u8* T = Ts[w];
  {
    const u8* lp = lists + (size_t)gchunk * 256;
    const u8* s2b = r->sym_to_byte;
    for (u32 i = lane; i < 256; i += 32) T[i] = s2b[lp[i]];
  }
  __syncwarp();
  const ChunkStart st = starts[gchunk];
  u32 k = st.k, o = st.off;
  u8* out = tt + ((size_t)ci << SEG_SHIFT);
  for (u32 base = 0; base < count; base += 32) {
    const bool valid = base + lane < count;
    const u32 sy = valid ? s[base + lane] : 0xffffu;
    const u32 b = T[valid ? sb[base + lane] : 0];
    const bool isrun = sy <= 1;
    const u32 runmask = __ballot_sync(FULL_MASK, isrun);
    const u32 nonrun_below = ~runmask & lanemask_lt();
    const u32 kk = nonrun_below ? lane - (31 - __clz(nonrun_below)) - 1 : lane + k;
    const u32 wgt = isrun ? (sy + 1) << kk : (sy <= symTotal ? 1u : 0u);
    const u32 inc = warp_incl_add(wgt);
    const u32 tot = __shfl_sync(FULL_MASK, inc, 31);
    const u32 oo = o + inc - wgt;
    if (wgt == 1) out[oo] = (u8)b;
    // runs longer than one byte: short ones by their own lane, long ones by the whole warp
    const bool shortrun = wgt > 1 && wgt <= 16;
    if (shortrun) for (u32 x = 0; x < wgt; x++) out[oo + x] = (u8)b;
    u32 big = __ballot_sync(FULL_MASK, wgt > 16);
    while (big) {
      const u32 l = __ffs(big) - 1;
      big &= big - 1;
      const u32 bo = __shfl_sync(FULL_MASK, oo, l), bw = __shfl_sync(FULL_MASK, wgt, l), bb = __shfl_sync(FULL_MASK, b, l);
      for (u32 x = lane; x < bw; x += 32) out[bo + x] = (u8)bb;
    }
    o += tot;
    const u32 nonrun = ~runmask;
    k = nonrun ? (u32)__clz(nonrun) : k + 32;  // run digits at the end of this batch
  }
}

// ---- inverse BWT ------------------------------------------------------------------------------
#define IB_SHIFT 7
#define IB_STEP (1u << IB_SHIFT)
#define IB_SEGS (SEG_SIZE / IB_STEP + 1)  // sampled rows per block + the start row
#define IB_VCAP 16384

#define IB_CAP 512u   // bytes a walk records on its way (four sampling steps); 1.8 % of the bytes lie behind that and are re-walked

struct Seg { u32 len, next; };
struct Visit { u32 row, off, len; };

// The bytes a walk passes are kept in a slot of IB_CAP bytes per sampled row (slotA: the 8192 multiples of 2^IB_SHIFT of
// every block, 4 MiB per block; slotB: the start row's slot at the head of the block's 4 MiB), so that once the order of
// the walks is known the block is assembled by copying instead of walking it a second time.
__device__ __forceinline__ u8* ib_slot(u8* slotA, u8* slotB, u32 ci, u32 sid) {
  return sid < IB_SEGS - 1 ? slotA + ((size_t)ci << (SEG_SHIFT + 2)) + (size_t)sid * IB_CAP : slotB + ((size_t)ci << (SEG_SHIFT + 2));
}

// walk from every sampled row (multiples of 2^IB_SHIFT and the start row) to the next sampled row
__global__ void k_ibwt_walk1(const u32* __restrict__ P, const CandRes* __restrict__ res, u32 ncand, Seg* __restrict__ segs, u32* __restrict__ capr,
                             u8* __restrict__ slotA, u8* __restrict__ slotB) {
  const u32 gid = blockIdx.x * blockDim.x + threadIdx.x;
  const u32 ci = gid / IB_SEGS, sid = gid % IB_SEGS;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 n = r->n;
  const u32* p = P + ((size_t)ci << SEG_SHIFT);
  const u32 r0 = p[r->orig] >> 8;  // first row whose byte is output (lib/Bzip2.js:386-391)
  u32 a;
  if (sid == IB_SEGS - 1) { if ((r0 & (IB_STEP - 1)) == 0) return; a = r0; }
  else { a = sid << IB_SHIFT; if (a >= n) return; }
  uint4* slot = reinterpret_cast<uint4*>(ib_slot(slotA, slotB, ci, sid));
  u32 row = a, steps = 0, rowcap = 0;
  // 32 steps at a time: the bytes of one chunk go out as ONE 32-byte sector (a sector written four bytes at a time is
  // evicted half full while 300 000 walks stream through the L2)
  for (bool more = true; more;) {
    u32 w[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (u32 k = 0; k < 32; k++) {
      const u32 e = p[row];
      w[k >> 2] |= (e & 0xffu) << (8u * (k & 3u));
      row = e >> 8;
      steps++;
      if (steps == IB_CAP) rowcap = row;
      if (!((row & (IB_STEP - 1)) != 0 && row != r0 && steps < n)) { more = false; break; }
    }
    const u32 chunk = (steps - 1) >> 5;
    if (chunk < IB_CAP / 32) {
      slot[2 * chunk] = make_uint4(w[0], w[1], w[2], w[3]);
      slot[2 * chunk + 1] = make_uint4(w[4], w[5], w[6], w[7]);
    }
  }
  Seg sg;
  sg.len = steps;
  sg.next = ((row & (IB_STEP - 1)) == 0) ? (row >> IB_SHIFT) : (IB_SEGS - 1);
  segs[(size_t)ci * IB_SEGS + sid] = sg;
  capr[(size_t)ci * IB_SEGS + sid] = rowcap;
}

// order the segments along the chain that starts at the start row.  One CTA per block: the segment
// table (64 KB) is staged in shared memory so that the serial walk costs a shared-memory load per step.
// tails: the visits that are longer than their slot (indices into the block's visit list).
__global__ void __launch_bounds__(128)
k_ibwt_chain(const u32* __restrict__ P, const CandRes* __restrict__ res, u32 ncand, const Seg* __restrict__ segs,
             Visit* __restrict__ visits, u32* __restrict__ nvisits, u32* __restrict__ tails, u32* __restrict__ ntails) {
  extern __shared__ __align__(8) unsigned char chain_smem[];
  Seg* ss = reinterpret_cast<Seg*>(chain_smem);
  const u32 ci = blockIdx.x;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0) { if (threadIdx.x == 0) { nvisits[ci] = 0; ntails[ci] = 0; } return; }
  const u32 n = r->n;
  const u32 nseg = min((u32)IB_SEGS, (n >> IB_SHIFT) + 2);
  for (u32 i = threadIdx.x; i < nseg; i += blockDim.x) ss[i] = segs[(size_t)ci * IB_SEGS + i];
  if (threadIdx.x == 0) ss[IB_SEGS - 1] = segs[(size_t)ci * IB_SEGS + IB_SEGS - 1];
  __syncthreads();
  if (threadIdx.x != 0) return;
  const u32* p = P + ((size_t)ci << SEG_SHIFT);
  const u32 r0 = p[r->orig] >> 8;
  u32 cur = ((r0 & (IB_STEP - 1)) == 0) ? (r0 >> IB_SHIFT) : (IB_SEGS - 1);
  u32 off = 0, nv = 0, nt = 0;
  Visit* v = visits + (size_t)ci * IB_VCAP;
  u32* tl = tails + (size_t)ci * IB_VCAP;
  while (off < n) {
    const Seg sg = ss[cur];
    const u32 len = min(sg.len, n - off);
    if (nv >= IB_VCAP) { nv = 0xffffffffu; nt = 0; break; }  // degenerate (periodic) block: fall back to one serial walk
    Visit vv;
    vv.row = (cur == IB_SEGS - 1) ? r0 : (cur << IB_SHIFT);
    vv.off = off; vv.len = len;
    if (len > IB_CAP) tl[nt++] = nv;
    v[nv++] = vv;
    off += len;
    cur = sg.next;
  }
  nvisits[ci] = nv;
  ntails[ci] = nt;
}

// Every visit's recorded bytes are copied to their place in the block: one warp per visit, aligned 32-bit words in the
// middle (realigned from the slot with a funnel shift), single bytes at the two ends (the neighbouring visits own the
// rest of those words).  IB_PLACE_CTAS CTAs share the visits of a block.
#define IB_PLACE_CTAS 4
#define IB_PLACE_THREADS 256
__global__ void __launch_bounds__(IB_PLACE_THREADS)
k_ibwt_place(const u32* __restrict__ P, const CandRes* __restrict__ res, u32 ncand, const Visit* __restrict__ visits,
             const u32* __restrict__ nvisits, const u8* __restrict__ slotA, const u8* __restrict__ slotB, u8* __restrict__ out) {
  const u32 ci = blockIdx.x / IB_PLACE_CTAS;
  if (ci >= ncand) return;
  if (res[ci].status != 0) return;
  const u32 nv = nvisits[ci];
  if (nv == 0xffffffffu) return;
  const u32 lane = threadIdx.x & 31u;
  const u32 wstride = IB_PLACE_CTAS * (IB_PLACE_THREADS / 32);
  const u32* p = P + ((size_t)ci << SEG_SHIFT);
  const u32 r0 = p[res[ci].orig] >> 8;
  const bool r0_own = (r0 & (IB_STEP - 1)) != 0;
  u8* ob = out + ((size_t)ci << SEG_SHIFT);
  for (u32 vi = (blockIdx.x % IB_PLACE_CTAS) * (IB_PLACE_THREADS / 32) + (threadIdx.x >> 5); vi < nv; vi += wstride) {
    const Visit v = visits[(size_t)ci * IB_VCAP + vi];
    const u32 sid = (r0_own && v.row == r0) ? (IB_SEGS - 1) : (v.row >> IB_SHIFT);
    const u8* srcb = ib_slot(const_cast<u8*>(slotA), const_cast<u8*>(slotB), ci, sid);
    const u32* src = reinterpret_cast<const u32*>(srcb);
    u8* o = ob + v.off;
    const u32 len = min(v.len, IB_CAP);
    const u32 head = min(len, (4u - ((u32)(size_t)o & 3u)) & 3u);   // bytes in front of the first aligned word
    const u32 nwords = (len - head) >> 2;
    if (lane < head) o[lane] = srcb[lane];
    u32* ow = reinterpret_cast<u32*>(o + head);
    const u32 sh = 8u * head;                                        // word w of the destination = source bytes head + 4w ..
    for (u32 w = lane; w < nwords; w += 32) {
      const u32 lo = src[w], hi = head ? src[w + 1] : 0u;           // src[w + 1] stays inside the slot: head + 4w + 3 < len <= IB_CAP
      ow[w] = __funnelshift_r(lo, hi, sh);
    }
    const u32 done = head + 4u * nwords;
    if (lane < len - done) o[done + lane] = srcb[done + lane];
  }
}

// what lies behind the recorded part of a long walk is walked again; so is a whole degenerate block
__global__ void k_ibwt_tail(const u32* __restrict__ P, const CandRes* __restrict__ res, u32 ncand, const Visit* __restrict__ visits,
                            const u32* __restrict__ nvisits, const u32* __restrict__ tails, const u32* __restrict__ ntails,
                            const u32* __restrict__ capr, u8* __restrict__ out) {
  const u32 gid = blockIdx.x * blockDim.x + threadIdx.x;
  const u32 ci = gid / IB_VCAP, ti = gid % IB_VCAP;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 nv = nvisits[ci];
  const u32* p = P + ((size_t)ci << SEG_SHIFT);
  u8* o = out + ((size_t)ci << SEG_SHIFT);
  u32 row, off, len;
  if (nv == 0xffffffffu) {
    if (ti != 0) return;
    row = p[r->orig] >> 8; off = 0; len = r->n;
  } else {
    if (ti >= ntails[ci]) return;
    const Visit v = visits[(size_t)ci * IB_VCAP + tails[(size_t)ci * IB_VCAP + ti]];
    const u32 r0 = p[r->orig] >> 8;
    const u32 sid = (v.row == r0 && (r0 & (IB_STEP - 1)) != 0) ? (IB_SEGS - 1) : (v.row >> IB_SHIFT);
    row = capr[(size_t)ci * IB_SEGS + sid]; off = v.off + IB_CAP; len = v.len - IB_CAP;
  }
  for (u32 t = 0; t < len; t++) {
    const u32 e = p[row];
    o[off + t] = (u8)e;
    row = e >> 8;
  }
}

static void dec_attr_once();

// The four walk launches of the inverse BWT over cnt blocks, from their vectors P (P[row] = successor << 8 | byte, slot
// layout): the sampled-row walks, recording into slotA / slotB (4 MiB per block each), their chain, the placement of what
// they recorded and the walks behind the records.  Each block goes back to front into its slot at out.
static void ibwt_walks(Ctx& c, const u32* P, const CandRes* res, u32 cnt, Seg* segs, u32* capr, Visit* visits, u32* nvis, u32* tails,
                       u32* ntails, u8* slotA, u8* slotB, u8* out) {
  k_ibwt_walk1<<<(cnt * IB_SEGS + 127) / 128, 128, 0, c.stream>>>(P, res, cnt, segs, capr, slotA, slotB);
  KLAUNCH(c); KCHECK();
  k_ibwt_chain<<<cnt, 128, sizeof(Seg) * IB_SEGS, c.stream>>>(P, res, cnt, segs, visits, nvis, tails, ntails);
  KLAUNCH(c); KCHECK();
  k_ibwt_place<<<cnt * IB_PLACE_CTAS, IB_PLACE_THREADS, 0, c.stream>>>(P, res, cnt, visits, nvis, slotA, slotB, out);
  KLAUNCH(c); KCHECK();
  k_ibwt_tail<<<(cnt * IB_VCAP + 127) / 128, 128, 0, c.stream>>>(P, res, cnt, visits, nvis, tails, ntails, capr, out);
  KLAUNCH(c); KCHECK();
}

// ---- BWT.unbwtransform (lib/BWT.js:352-363): inverse of the sentinel BWT ------------------------------
// Reference walk: t = 0; for i = n-1..0: U[i] = T[t]; t = LF[t] + C[T[t]]; t += (t < pidx).  LF[t] + C[T[t]] is
// the rank x of position t in the stable order by byte, i.e. the inverse of the sorted-position vector that one
// radix pass produces.  P[t] = next(t) << 8 | T[t] feeds the same sampled-row walks as the bzip2 decoder; the
// spare slot 2^20-1 holds the pseudo start entry (orig) whose successor is row 0.  The walk reaches row n only when
// pidx == n (the reference then reads T[n], undefined, as 0): P[n] = 0 reproduces that.  Block = blockIdx.y.
__global__ void k_unbwt_pack(const u8* __restrict__ L, const u32* __restrict__ sorted_pos, const u32* __restrict__ d_n,
                             const u32* __restrict__ d_pidx, u32* __restrict__ P) {
  const u32 x = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  const u32 n = d_n[b], pidx = d_pidx[b];
  const size_t base = (size_t)b << SEG_SHIFT;
  if (x == 0) { P[base + SEG_SIZE - 1] = 0; P[base + n] = 0; }
  if (x >= n) return;
  const u32 t = sorted_pos[base + x] & SEG_MASK;
  P[base + t] = ((x + (x < pidx ? 1u : 0u)) << 8) | L[base + t];
}
__global__ void k_unbwt_setup(CandRes* res, const u32* __restrict__ d_n, u32 nb) {
  const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  CandRes* r = res + b;
  const u32 n = d_n[b];
  r->status = 0; r->detail = 0; r->m = 0; r->orig = SEG_SIZE - 1; r->sym_total = 0; r->n = n; r->rawlen = n; r->open = 0; r->rand = 0; r->run4 = 0; r->endbit = 0;
}
// the walks write each block back to front into its slot; the blocks go out front to back and back to back
__global__ void k_reverse_blocks(const u8* __restrict__ in, const u32* __restrict__ d_n, const u64* __restrict__ d_off, u8* __restrict__ out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  const u32 n = d_n[b];
  if (i < n) out[d_off[b] + n - 1 - i] = in[((size_t)b << SEG_SHIFT) + i];
}
static void dec_attr_once() {
  static bool attr = false;
  if (attr) return;
  for (auto k : {k_hdec<128, false>, k_hdec<256, false>, k_hdec<512, false>, k_hdec<128, true>, k_hdec<256, true>, k_hdec<512, true>})
    CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HdecWarp)));
  CUDA_CHECK(cudaFuncSetAttribute(k_ibwt_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(Seg) * IB_SEGS)));
  attr = true;
}
// Scratch: about 14 MiB per block.
void bwt_inverse_sentinel_batch(Ctx& c, const u8* d_L, const u32* h_n, const u32* h_pidx, u32 nb, u8* d_out) {
  if (!nb) return;
  dec_attr_once();
  u32 nmax = 0; u64 ntot = 0;
  std::vector<u64> hoff(nb);
  for (u32 b = 0; b < nb; b++) { hoff[b] = ntot; ntot += h_n[b]; nmax = std::max(nmax, h_n[b]); }
  const size_t slots = (size_t)nb << SEG_SHIFT;
  DBuf<u32> valA(c, slots), valB(c, slots), slotA(c, slots), dn(c, nb), dpidx(c, nb), nvis(c, nb), ntails(c, nb);
  DBuf<u8> kout(c, slots), tmp(c, slots);
  DBuf<u64> doff(c, nb);
  DBuf<CandRes> res(c, nb);
  DBuf<Seg> segs(c, (size_t)nb * IB_SEGS);
  DBuf<Visit> visits(c, (size_t)nb * IB_VCAP);
  DBuf<u32> capr(c, (size_t)nb * IB_SEGS), tails(c, (size_t)nb * IB_VCAP);
  c.to_device(dn, h_n, 4 * nb);
  c.to_device(dpidx, h_pidx, 4 * nb);
  c.to_device(doff, hoff.data(), 8 * nb);
  // one stable counting-sort pass per block over the L column's bytes: vin = the positions in sorted order
  u8* kin = const_cast<u8*>(d_L);   // read only: a single pass writes kout
  u8* ko = kout.p;
  u32 *vin = valA.p, *vout = valB.p;
  radix_sort<u8>(c, kin, vin, ko, vout, dn.p, nb, SEG_SHIFT, nmax, 0, 1, true, ntot);
  u32* P = vout;    // the iota pass never read its value buffer
  const dim3 grid((nmax + 255) / 256, nb);
  k_unbwt_pack<<<grid, 256, 0, c.stream>>>(d_L, vin, dn, dpidx, P);
  KLAUNCH(c); KCHECK();
  k_unbwt_setup<<<(nb + 127) / 128, 128, 0, c.stream>>>(res, dn, nb);
  KLAUNCH(c); KCHECK();
  // the walks record into slotA (4 MiB per block); the start row's slot goes to the head of the block's 4 MiB of the
  // sorted positions, which k_unbwt_pack has consumed
  ibwt_walks(c, P, res, nb, segs, capr, visits, nvis, tails, ntails, reinterpret_cast<u8*>(slotA.p), reinterpret_cast<u8*>(vin), tmp);
  k_reverse_blocks<<<grid, 256, 0, c.stream>>>(tmp, dn, doff, d_out);
  KLAUNCH(c); KCHECK();
}

// ---- RLE1 decode ------------------------------------------------------------------------------
#define UR_THREADS 256
#define UR_ITEMS 8
#define UR_TILE (UR_THREADS * UR_ITEMS)
#define UE_STAGE 6144u   // bytes of expanded output a tile stages in shared memory

__device__ __forceinline__ bool unrle_sync(const u8* b, u32 i) {
  if (i == 0) return true;
  if (b[i] == b[i - 1]) return false;
  if (i >= 4 && b[i - 1] == b[i - 2] && b[i - 2] == b[i - 3] && b[i - 3] == b[i - 4]) return false;
  return true;
}
// the reference's loop (lib/Bzip2.js:424-436) from a synchronisation point i to the next one: cls[j] = 1 for repeat counts.
__device__ __noinline__ void unrle_walk(const u8* __restrict__ b, u8* __restrict__ c, u32 i, u32 n) {
  u32 j = i, run = 0;
  int prev = -1;
  for (;;) {
    const int v = b[j];
    c[j] = 0;
    run = (v == prev) ? run + 1 : 1;
    prev = v;
    j++;
    if (j >= n) break;
    if (run == 4) {
      c[j] = 1;
      j++;
      run = 0; prev = -1;
      if (j >= n) break;
    }
    if (unrle_sync(b, j)) break;
  }
}
// cls[i] = 1 when byte i is a repeat count.  A byte that differs from its predecessor and does not follow four equal
// bytes is certainly a literal that starts a new run (a synchronisation point); the bytes between two such points are
// classified by the serial loop.  One thread per 8 bytes: the 13 bytes that decide its synchronisation points sit in
// registers, a literal followed by another synchronisation point is final at once (all 8 of them: one 8-byte store),
// and only real run starts walk.
__global__ void __launch_bounds__(256) k_unrle_classify(const u8* __restrict__ rle, const CandRes* __restrict__ res, u32 ncand, u8* __restrict__ cls) {
  const u32 g = blockIdx.x * blockDim.x + threadIdx.x;
  const u32 ci = g >> (SEG_SHIFT - 3), i0 = (g & (SEG_MASK >> 3)) << 3;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0 || i0 >= r->n) return;
  const u32 n = r->n;
  const u8* b = rle + ((size_t)ci << SEG_SHIFT);
  u8* c = cls + ((size_t)ci << SEG_SHIFT);
  const u64 prev = i0 ? *reinterpret_cast<const u64*>(b + i0 - 8) : 0ull;
  const u64 cur = *reinterpret_cast<const u64*>(b + i0);
  const u64 next = (i0 + 8 < SEG_SIZE) ? *reinterpret_cast<const u64*>(b + i0 + 8) : 0ull;
  // E bit (j + 3): byte i0 + j equals its predecessor, j = -3 .. 8 (bytes past n only make a position look like a run: it walks)
  u32 E = 0;
#pragma unroll
  for (int j = -3; j <= 8; j++) {
    const u32 x = j < 0 ? (u32)(prev >> (8 * (j + 8))) : (j < 8 ? (u32)(cur >> (8 * j)) : (u32)(next >> (8 * (j - 8))));
    const u32 y = (j - 1) < 0 ? (u32)(prev >> (8 * (j - 1 + 8))) : ((j - 1) < 8 ? (u32)(cur >> (8 * (j - 1))) : (u32)(next >> (8 * (j - 1 - 8))));
    if (((x ^ y) & 0xffu) == 0 && (int)i0 + j >= 1) E |= 1u << (j + 3);
  }
  // S bit k: position i0 + k is a synchronisation point, k = 0 .. 8
  u32 S = 0;
#pragma unroll
  for (int k = 0; k <= 8; k++) {
    const bool e0 = (E >> (k + 3)) & 1u, run4 = ((E >> k) & 7u) == 7u && i0 + k >= 4;  // E(i-3), E(i-2), E(i-1)
    if (!e0 && !run4) S |= 1u << k;
  }
  if ((S & 0xffu) == 0xffu && i0 + 8 <= n) {
    // eight literals, each followed by a synchronisation point or the end... unless the ninth position continues a run of
    // the eighth: then position 7 starts a walk
    if ((S >> 8) & 1u || i0 + 8 >= n) { *reinterpret_cast<u64*>(c + i0) = 0ull; return; }
    *reinterpret_cast<u32*>(c + i0) = 0u;
    c[i0 + 4] = 0; c[i0 + 5] = 0; c[i0 + 6] = 0;
    unrle_walk(b, c, i0 + 7, n);
    return;
  }
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const u32 i = i0 + k;
    if (i < n && ((S >> k) & 1u)) {
      if (((S >> (k + 1)) & 1u) || i + 1 >= n) c[i] = 0;
      else unrle_walk(b, c, i, n);
    }
  }
}

// ---- derandomise (libbz2 flavor) ----------------------------------------------------------------
// libbz2's BZ2_rNums: the gaps between the flipped bytes of a randomised block (bzip2 0.9.0 and older wrote them).
static const int RNUMS[512] = {
    619, 720, 127, 481, 931, 816, 813, 233, 566, 247, 985, 724, 205, 454, 863, 491, 741, 242, 949, 214, 733, 859, 335, 708,
    621, 574, 73,  654, 730, 472, 419, 436, 278, 496, 867, 210, 399, 680, 480, 51,  878, 465, 811, 169, 869, 675, 611, 697,
    867, 561, 862, 687, 507, 283, 482, 129, 807, 591, 733, 623, 150, 238, 59,  379, 684, 877, 625, 169, 643, 105, 170, 607,
    520, 932, 727, 476, 693, 425, 174, 647, 73,  122, 335, 530, 442, 853, 695, 249, 445, 515, 909, 545, 703, 919, 874, 474,
    882, 500, 594, 612, 641, 801, 220, 162, 819, 984, 589, 513, 495, 799, 161, 604, 958, 533, 221, 400, 386, 867, 600, 782,
    382, 596, 414, 171, 516, 375, 682, 485, 911, 276, 98,  553, 163, 354, 666, 933, 424, 341, 533, 870, 227, 730, 475, 186,
    263, 647, 537, 686, 600, 224, 469, 68,  770, 919, 190, 373, 294, 822, 808, 206, 184, 943, 795, 384, 383, 461, 404, 758,
    839, 887, 715, 67,  618, 276, 204, 918, 873, 777, 604, 560, 951, 160, 578, 722, 79,  804, 96,  409, 713, 940, 652, 934,
    970, 447, 318, 353, 859, 672, 112, 785, 645, 863, 803, 350, 139, 93,  354, 99,  820, 908, 609, 772, 154, 274, 580, 184,
    79,  626, 630, 742, 653, 282, 762, 623, 680, 81,  927, 626, 789, 125, 411, 521, 938, 300, 821, 78,  343, 175, 128, 250,
    170, 774, 972, 275, 999, 639, 495, 78,  352, 126, 857, 956, 358, 619, 580, 124, 737, 594, 701, 612, 669, 112, 134, 694,
    363, 992, 809, 743, 168, 974, 944, 375, 748, 52,  600, 747, 642, 182, 862, 81,  344, 805, 988, 739, 511, 655, 814, 334,
    249, 515, 897, 955, 664, 981, 649, 113, 974, 459, 893, 228, 433, 837, 553, 268, 926, 240, 102, 654, 459, 51,  686, 754,
    806, 760, 493, 403, 415, 394, 687, 700, 946, 670, 656, 610, 738, 392, 760, 799, 887, 653, 978, 321, 576, 617, 626, 502,
    894, 679, 243, 440, 680, 879, 194, 572, 640, 724, 926, 56,  204, 700, 707, 151, 457, 449, 797, 195, 791, 558, 945, 679,
    297, 59,  87,  824, 713, 663, 412, 693, 342, 606, 134, 108, 571, 364, 631, 212, 174, 643, 304, 329, 343, 97,  430, 751,
    497, 314, 983, 374, 822, 928, 140, 206, 73,  263, 980, 736, 876, 478, 430, 305, 170, 514, 364, 692, 829, 82,  855, 953,
    676, 246, 369, 970, 294, 750, 807, 827, 150, 790, 288, 923, 804, 378, 215, 828, 592, 281, 565, 555, 710, 82,  896, 831,
    547, 261, 524, 462, 293, 465, 502, 56,  661, 821, 976, 991, 658, 869, 905, 758, 745, 193, 768, 550, 608, 933, 378, 286,
    215, 979, 792, 961, 61,  688, 793, 644, 986, 403, 106, 366, 905, 644, 372, 567, 466, 434, 645, 210, 389, 550, 919, 135,
    780, 773, 635, 389, 707, 100, 626, 958, 165, 504, 920, 176, 193, 713, 857, 265, 203, 50,  668, 108, 645, 990, 626, 197,
    510, 357, 358, 850, 858, 364, 936, 638};
#define DR_FLIPS 1655  // flipped bytes below 900 000 (the largest block)
__constant__ u32 c_flips[DR_FLIPS];

// The positions libbz2 XORs with 1 in a randomised block's pre-RLE1 bytes: togo counts down from rNums[t], t cycling
// through the table, and the byte where togo reaches 1 is flipped.  __constant__ memory belongs to a device's context,
// so the table is uploaded once per device (b2_init may bind another device after b2_shutdown; the library never
// resets a device, so a device's copy stays valid).
static void derand_table_once(int device) {
  static std::vector<bool> done;
  if (device < (int)done.size() && done[device]) return;
  std::vector<u32> f;
  int togo = 0, t = 0;
  for (u32 i = 0; i < 900000u; i++) {
    if (togo == 0) { togo = RNUMS[t]; t = (t + 1) & 511; }
    if (--togo == 1) f.push_back(i);
  }
  if (f.size() != DR_FLIPS) throw B2Error{B2_ERR_CUDA, "derandomise table has the wrong length"};
  CUDA_CHECK(cudaMemcpyToSymbol(c_flips, f.data(), sizeof(u32) * DR_FLIPS));
  if (device >= (int)done.size()) done.resize(device + 1, false);
  done[device] = true;
}

// One thread per (block, flip): the flipped bytes of every randomised block are XORed in place in its slot, before the
// count bytes are classified, so that everything behind (classes, lengths, expansion, CRC) sees derandomised bytes.
__global__ void k_derand(u8* __restrict__ rle, const CandRes* __restrict__ res, u32 ncand) {
  const u32 g = blockIdx.x * blockDim.x + threadIdx.x;
  const u32 ci = g / DR_FLIPS, f = g % DR_FLIPS;
  if (ci >= ncand) return;
  const CandRes* r = res + ci;
  if (r->status != 0 || !r->rand) return;
  const u32 p = c_flips[f];
  if (p < r->n) rle[((size_t)ci << SEG_SHIFT) + p] ^= 1u;
}

// expanded size of every tile (no chain between tiles: the per-block scan below is a separate, tiny kernel)
__global__ void __launch_bounds__(UR_THREADS)
k_unrle_tilesum(const u8* __restrict__ rle, const u8* __restrict__ cls, const CandRes* __restrict__ res, u32 tps, u32* __restrict__ tilesum) {
  __shared__ u32 ws[UR_THREADS / 32];
  const u32 tid = threadIdx.x;
  const u32 ci = blockIdx.x / tps, lt = blockIdx.x % tps;
  const CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 n = r->n;
  const u32 start = lt * UR_TILE;
  if (start >= n) return;
  const u8* b = rle + ((size_t)ci << SEG_SHIFT);
  const u8* c = cls + ((size_t)ci << SEG_SHIFT);
  u32 sum = 0;
  const u32 p0 = start + tid * UR_ITEMS;
  static_assert(UR_ITEMS == 8, "one 8-byte load per array");
  if (p0 < n) {
    const u64 bv = *reinterpret_cast<const u64*>(b + p0), cv = *reinterpret_cast<const u64*>(c + p0);
#pragma unroll
    for (int j = 0; j < UR_ITEMS; j++)
      if (p0 + j < n) sum += ((u32)(cv >> (8 * j)) & 0xffu) ? ((u32)(bv >> (8 * j)) & 0xffu) : 1u;
  }
  sum = warp_reduce_add(sum);
  if ((tid & 31u) == 0) ws[tid >> 5] = sum;
  __syncthreads();
  if (tid < 32) {
    u32 v = tid < UR_THREADS / 32 ? ws[tid] : 0u;
    v = warp_reduce_add(v);
    if (tid == 0) tilesum[(size_t)ci * tps + lt] = v;
  }
}
// one warp per block: output offset of every tile, decoded size of the block, and run4: the last four bytes are equal
// and none is a count byte.  The serial loop's run then counts four at the end (the byte in front of them is another
// value or a count byte: five equal literals cannot occur), and libbz2 wants the count byte behind them.
__global__ void __launch_bounds__(32)
k_unrle_tileoff(const u8* __restrict__ rle, const u8* __restrict__ cls, CandRes* __restrict__ res, u32 tps, const u32* __restrict__ tilesum,
                u32* __restrict__ tileoff) {
  const u32 ci = blockIdx.x, lane = threadIdx.x;
  CandRes* r = res + ci;
  if (r->status != 0) return;
  const u32 n = r->n;
  const u32 nt = (n + UR_TILE - 1) / UR_TILE;
  u32 run = 0;
  for (u32 t0 = 0; t0 < nt; t0 += 32) {
    const u32 t = t0 + lane;
    const u32 v = t < nt ? tilesum[(size_t)ci * tps + t] : 0u;
    const u32 inc = warp_incl_add(v);
    if (t < nt) tileoff[(size_t)ci * tps + t] = run + inc - v;
    run += __shfl_sync(FULL_MASK, inc, 31);
  }
  if (lane == 0) {
    r->rawlen = run;
    u32 run4 = 0;
    if (n >= 4) {
      const u8* b = rle + ((size_t)ci << SEG_SHIFT) + (n - 4);
      const u8* c = cls + ((size_t)ci << SEG_SHIFT) + (n - 4);
      run4 = b[0] == b[1] && b[1] == b[2] && b[2] == b[3] && !(c[0] | c[1] | c[2] | c[3]);
    }
    r->run4 = run4;
  }
}

__global__ void __launch_bounds__(UR_THREADS)
k_unrle_emit(const u8* __restrict__ rle, const u8* __restrict__ cls, const CandRes* __restrict__ res, u32 tps, const u32* __restrict__ tileoff,
             const u64* __restrict__ outbase, u8* __restrict__ out) {
  __shared__ u32 ws[UR_THREADS / 32 + 1];
  __shared__ __align__(16) u8 stg[UE_STAGE + 32];
  const u32 tid = threadIdx.x;
  const u32 ci = blockIdx.x / tps, lt = blockIdx.x % tps;
  const u64 ob = outbase[ci];
  if (ob == ~0ull) return;  // candidate is not part of the stream
  const CandRes* r = res + ci;
  const u32 n = r->n;
  const u32 start = lt * UR_TILE;
  if (start >= n) return;
  const u8* b = rle + ((size_t)ci << SEG_SHIFT);
  const u8* c = cls + ((size_t)ci << SEG_SHIFT);
  u32 len[UR_ITEMS];
  u32 sum = 0;
  const u32 p0 = start + tid * UR_ITEMS;
  u64 bv = 0, cv = 0;
  if (p0 < n) { bv = *reinterpret_cast<const u64*>(b + p0); cv = *reinterpret_cast<const u64*>(c + p0); }
#pragma unroll
  for (int j = 0; j < UR_ITEMS; j++) {
    const u32 p = p0 + j;
    len[j] = (p < n) ? (((u32)(cv >> (8 * j)) & 0xffu) ? ((u32)(bv >> (8 * j)) & 0xffu) : 1u) : 0u;
    sum += len[j];
  }
  u32 total;
  const u32 ex = block_excl_add<UR_THREADS, u32>(sum, ws, &total);
  u8* otile = out + ob + tileoff[(size_t)ci * tps + lt];
  // A tile that expands to at most UE_STAGE bytes (every tile of run-free data, most others) is put together in shared
  // memory, at the alignment (mod 16) it has in the output, and leaves in 16-byte stores; longer ones go out directly.
  const bool staged = total <= UE_STAGE;
  const u32 mis = (u32)(size_t)otile & 15u;
  u8* o = staged ? stg + mis + ex : otile + ex;
#pragma unroll
  for (int j = 0; j < UR_ITEMS; j++) {
    const u32 p = p0 + j;
    if (p < n) {
      if ((u32)(cv >> (8 * j)) & 0xffu) {
        const u8 v = b[p - 1];
        for (u32 x = 0; x < len[j]; x++) o[x] = v;
      } else {
        o[0] = (u8)(bv >> (8 * j));
      }
      o += len[j];
    }
  }
  if (!staged) return;
  __syncthreads();
  {
    const u32 last = mis + total;
    u8* og = otile - mis;  // 16-byte aligned
    for (u32 c16 = tid * 16u; c16 < last; c16 += UR_THREADS * 16u) {
      if (c16 >= mis && c16 + 16u <= last) {
        *reinterpret_cast<uint4*>(og + c16) = *reinterpret_cast<const uint4*>(stg + c16);
      } else {
        const u32 e = min(c16 + 16u, last);
        for (u32 x = max(c16, mis); x < e; x++) og[x] = stg[x];
      }
    }
  }
}

// ---- host ---------------------------------------------------------------------------------------
static std::string hexs(u32 v) {
  char b[16];
  snprintf(b, sizeof b, "%x", v);
  return b;
}

// kind: 0 block, 1 eos, 2 error, 3 an end-of-stream magic in a position list (no bytes, no stream CRC);
// off: offset in the decoded stream where the event happens (a block's start).  A block event carries its bit position,
// its stored CRC (a), its decoded length and the slot of its results (in the batch; in the file for the sharded decode).
struct Event { int kind; size_t slot; u32 a, b; int code; std::string msg; u64 off; u64 pos; u32 len; };

static const u32 UR_TPS = SEG_SIZE / UR_TILE;
#define DEC_KEEP_CLS 16384u
// blocks per decode batch ($B2_DEC_BATCH: test hook, small batches exercise the batch seams on small inputs)
static u32 dec_batch_blocks(const Ctx& c) {
  if (const char* e = getenv("B2_DEC_BATCH")) { const int v = atoi(e); if (v >= 1) return (u32)v; }
  return std::max(c.bwt_batch, 2048u);
}
static u32 dec_keep_cls_limit() {
  if (const char* e = getenv("B2_DEC_KEEP_CLS")) { const int v = atoi(e); if (v >= 0) return (u32)v; }  // test hook
  return DEC_KEEP_CLS;
}

// Scratch of one decode batch, allocated for the largest batch of a call and reused by every batch: about 20 MiB per block
// (the radix sort's keys and values, 16 MiB, are most of it).
struct DecScratch {
  u32 cap = 0;
  DBuf<u16> sym;
  DBuf<u8> selbuf, tt, symb, perms, lists;
  DBuf<ChunkSum> sums;
  DBuf<ChunkStart> starts;
  DBuf<u32> keyA, keyB, valA, valB, dn, nvis, tilesum, capr, tails, ntails;
  DBuf<Seg> segs;
  DBuf<Visit> visits;
  std::vector<u32> hn;
  void alloc(Ctx& c, u32 nbm) {
    if (nbm <= cap) return;
    cap = nbm;
    const size_t cps = SEG_SIZE / UM_CHUNK, slots = (size_t)nbm << SEG_SHIFT;
    sym.alloc(c, slots);
    selbuf.alloc(c, (size_t)nbm * SEL_CAP); tt.alloc(c, slots); symb.alloc(c, slots);
    sums.alloc(c, nbm * cps); perms.alloc(c, nbm * cps * 256); lists.alloc(c, nbm * cps * 256); starts.alloc(c, nbm * cps);
    keyA.alloc(c, slots); keyB.alloc(c, slots); valA.alloc(c, slots); valB.alloc(c, slots);
    dn.alloc(c, nbm); nvis.alloc(c, nbm); tilesum.alloc(c, (size_t)nbm * UR_TPS);
    segs.alloc(c, (size_t)nbm * IB_SEGS); visits.alloc(c, (size_t)nbm * IB_VCAP);
    capr.alloc(c, (size_t)nbm * IB_SEGS); tails.alloc(c, (size_t)nbm * IB_VCAP); ntails.alloc(c, nbm);
    hn.resize(nbm);
  }
};

// One decode batch: the cnt block candidates dcand[0, cnt) of the input window `in` (wbytes bytes from bit base_bit of the
// file; `last`: the window ends with the file) through the Huffman stage, un-MTF, the inverse BWT (into the slots at rle)
// and the RLE1 length scan (count-byte classes into the slots at cls, tile offsets into tileoff).  Results in rb on the
// device and in hres on the host.
static void dec_batch(Ctx& c, DecScratch& B, const u8* in, u64 wbytes, u64 base_bit, bool last, const Cand* dcand, u32 cnt, int flavor,
                      CandRes* rb, CandRes* hres, u8* rle, u8* cls, u32* tileoff) {
  // The kernels decode every candidate under the largest block size: the members of a multistream file may have
  // different levels (lib/Bzip2.js:105-124 re-reads the level per member), and which member a candidate belongs to is
  // only known when the host walks the chain, where the member's own limit is applied (block_event).
  const u32 dbuf_size = 900000u;
  const u32 cps = SEG_SIZE / UM_CHUNK, ur_tps = UR_TPS;
  B.alloc(c, cnt);
  dec_attr_once();
  {
    // the per-block Huffman stage is one CTA per block and latency bound: it gets the whole batch at once
    StageScope ss(c, ST_HDEC);
    static int sms = 0;
    if (!sms) CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device));
    const bool lb = flavor == B2_BZ2_LIBBZ2;
    const u32 t = cnt <= 2u * (u32)sms ? 512 : cnt <= 4u * (u32)sms ? 256 : HD_THREADS;
    auto k = t == 512 ? (lb ? k_hdec<512, true> : k_hdec<512, false>)
           : t == 256 ? (lb ? k_hdec<256, true> : k_hdec<256, false>) : (lb ? k_hdec<HD_THREADS, true> : k_hdec<HD_THREADS, false>);
    k<<<cnt, t, sizeof(HdecWarp), c.stream>>>(in, wbytes, base_bit, last, dcand, cnt, dbuf_size, B.selbuf, B.sym, rb);
    KLAUNCH(c); KCHECK();
  }
  {
    StageScope ss(c, ST_UNMTF);
    const u32 chunks = cnt * cps;
    k_unmtf_a<<<(chunks + UA_THREADS - 1) / UA_THREADS, UA_THREADS, 0, c.stream>>>(B.sym, rb, cnt, cps, B.sums, B.perms, B.symb);
    KLAUNCH(c); KCHECK();
    k_unmtf_scan<<<cnt, 32, 0, c.stream>>>(rb, cnt, cps, dbuf_size, B.sums, B.perms, B.lists, B.starts);
    KLAUNCH(c); KCHECK();
    k_unmtf_map<<<(chunks + UM_WARPS - 1) / UM_WARPS, UM_WARPS * 32, 0, c.stream>>>(B.sym, B.symb, rb, cnt, cps, B.lists, B.starts, B.tt);
    KLAUNCH(c); KCHECK();
  }
  CUDA_CHECK(cudaMemcpyAsync(hres, rb, sizeof(CandRes) * cnt, cudaMemcpyDeviceToHost, c.stream));
  CUDA_CHECK(cudaStreamSynchronize(c.stream));
  u32 nmax = 0; u64 ntot = 0;
  for (u32 i = 0; i < cnt; i++) { B.hn[i] = hres[i].status == 0 ? hres[i].n : 0; nmax = std::max(nmax, B.hn[i]); ntot += B.hn[i]; }
  if (nmax) {
    StageScope ss(c, ST_IBWT);
    CUDA_CHECK(cudaMemcpyAsync(B.dn, B.hn.data(), cnt * 4, cudaMemcpyHostToDevice, c.stream));
    // T-vector: one stable counting-sort pass over the L column itself (byte keys, the values are the row numbers);
    // the pass writes P[row] = successor << 8 | L[row] directly (radix.cuh: pack epilogue)
    u8* kin = B.tt.p; u8* kout = nullptr;
    u32 *vin = B.valA, *vout = B.valB;
    u32* Pp = B.keyB;
    radix_sort<u8>(c, kin, vin, kout, vout, B.dn, cnt, SEG_SHIFT, nmax, 0, 1, true, ntot, nullptr, B.tt.p, Pp);
    // all blocks of the batch walk together: the launch lasts as long as its longest segment walk, so fewer,
    // bigger launches win over keeping the packed T-vectors L2 resident (measured: 75 ms -> 36 ms per GiB).
    // The walks record into the free key / value buffers of the sort (4 MiB per block each).
    ibwt_walks(c, Pp, rb, cnt, B.segs, B.capr, B.visits, B.nvis, B.tails, B.ntails, reinterpret_cast<u8*>(B.keyA.p),
               reinterpret_cast<u8*>(B.valA.p), rle);
  }
  if (nmax) {
    StageScope ss(c, ST_UNRLE);
    const u32 nslots = cnt << SEG_SHIFT;
    if (flavor == B2_BZ2_LIBBZ2 && std::any_of(hres, hres + cnt, [](const CandRes& r) { return r.status == 0 && r.rand; })) {
      derand_table_once(c.device);
      k_derand<<<(cnt * DR_FLIPS + 255) / 256, 256, 0, c.stream>>>(rle, rb, cnt);
      KLAUNCH(c); KCHECK();
    }
    k_unrle_classify<<<(nslots / 8 + 255) / 256, 256, 0, c.stream>>>(rle, rb, cnt, cls);
    KLAUNCH(c); KCHECK();
    k_unrle_tilesum<<<cnt * ur_tps, UR_THREADS, 0, c.stream>>>(rle, cls, rb, ur_tps, B.tilesum);
    KLAUNCH(c); KCHECK();
    k_unrle_tileoff<<<cnt, 32, 0, c.stream>>>(rle, cls, rb, ur_tps, B.tilesum, tileoff);
    KLAUNCH(c); KCHECK();
    CUDA_CHECK(cudaMemcpyAsync(hres, rb, sizeof(CandRes) * cnt, cudaMemcpyDeviceToHost, c.stream));
  }
  CUDA_CHECK(cudaStreamSynchronize(c.stream));
  c.stats.blocks += cnt;
}

// ---- the compressed input ----
// A host stream (StreamIn, whose length is known once it has ended) or a device buffer holding bytes [off, off + n) of
// an input of `total` bytes (a share of a sharded stream; the whole input when off = 0 and total = n).  The drivers
// read the input through these calls only, at stream offsets.
struct DecIn {
  StreamIn* s = nullptr;
  const u8* d = nullptr;
  size_t n = 0;
  u64 off = 0;
  size_t total = 0;
  explicit DecIn(StreamIn& in) : s(&in) {}
  DecIn(const u8* d_in, size_t n_) : d(d_in), n(n_), total(n_) {}
  DecIn(const u8* d_in, size_t n_, u64 off_, size_t total_) : d(d_in), n(n_), off(off_), total(total_) {}
  size_t length() const { return s ? (s->eof ? s->base + s->have : SIZE_MAX) : total; }  // a stream's once it has ended
  u64 end() const { return s ? s->base + s->have : off + n; }  // the end of the bytes there are so far
  // Up to k bytes at bytepos (a member header, or a magic the input may cut off) into h; returns how many there are.  They
  // may lie past the window: a stream reads one byte more, which tells whether the input ends behind them.
  size_t head(Ctx& c, u64 bytepos, u8* h, size_t k = 4) {
    if (s) s->fill(bytepos + k + 1);
    const size_t avail = (size_t)std::min<u64>(k, end() - bytepos);
    if (s) {
      memcpy(h, s->at(bytepos), avail);
    } else {
      CUDA_CHECK(cudaMemcpyAsync(h, d + (bytepos - off), avail, cudaMemcpyDeviceToHost, c.stream));
      CUDA_CHECK(cudaStreamSynchronize(c.stream));
    }
    return avail;
  }
  // As much of [a, a + len) as the input has into the device buffer win, zero padded (aligned word reads past the end
  // must be safe); returns its length.  A stream keeps its bytes from a on and reads one byte past a + len, so its end is
  // known exactly when a complete input would show it (until then no window is the last one).  A device buffer that
  // starts behind a (a share, whose window starts at a word boundary) reads zeros in front of off.
  u64 window(Ctx& c, DBuf<u8>& win, u64 a, u64 want) {
    if (s) {
      s->drop(a);
      s->fill(a + want + 1);
    }
    const u64 len = std::min<u64>(want, end() - a);
    if (len + 32 > win.n) win.alloc(c, len + 32);
    CUDA_CHECK(cudaMemsetAsync(win.p + (len & ~(u64)3), 0, 32 + (len & 3), c.stream));
    if (s) {
      StageScope st(c, ST_H2D);
      if (len) CUDA_CHECK(cudaMemcpyAsync(win, s->at(a), len, cudaMemcpyHostToDevice, c.stream));
    } else if (len) {
      const u64 lead = std::min<u64>(off > a ? off - a : 0, len);
      if (lead) CUDA_CHECK(cudaMemsetAsync(win, 0, lead, c.stream));
      if (len > lead) CUDA_CHECK(cudaMemcpyAsync(win.p + lead, d + (a + lead - off), len - lead, cudaMemcpyDeviceToDevice, c.stream));
    }
    return len;
  }
};

// ---- the block chain (lib/Bzip2.js:454-481 / 508-548) ----
struct Chain {
  int multistream = 0;
  int flavor = B2_BZ2_COMPRESSJS;  // B2_BZ2_LIBBZ2: the rules of include/b2bz.h's b2_bzip2_decompress_flavor
  u32 cur_dbuf = 0;         // dbufSize of the member the walk is in (lib/Bzip2.js:121)
  u64 pos = 32;             // bit position of the next magic
  u32 stream_crc = 0;
  u64 total_out = 0;        // decoded bytes of the blocks walked
  size_t li = 0;            // position list: the next entry
  bool done = false;        // end of the stream reached, or an error recorded
  std::vector<Event> events;
};

// a block on the chain; false when it ends the walk (its error is recorded)
static bool block_event(Chain& ch, const Cand& cd, const CandRes& r, size_t slot) {
  // the member's own limits, in the reference's order: randomised bit (:143), origPointer (:146), then the body
  if (r.status != DEC_OBSOLETE && r.orig > ch.cur_dbuf) {
    ch.events.push_back({2, slot, 0, 0, DEC_DATA_ERROR, "Data error: initial position out of bounds", ch.total_out, 0, 0});
    return false;
  }
  if (r.status != 0) {
    std::string msg = r.status == DEC_OBSOLETE ? "Obsolete (pre 0.9.5) bzip format not supported." : "Data error";
    if (r.detail == 1) msg += ": initial position out of bounds";
    ch.events.push_back({2, slot, 0, 0, r.status, msg, ch.total_out, 0, 0});
    return false;
  }
  if (r.n > ch.cur_dbuf) {  // dbufCount would have run over dbufSize (lib/Bzip2.js:338,354)
    ch.events.push_back({2, slot, 0, 0, DEC_DATA_ERROR, "Data error", ch.total_out, 0, 0});
    return false;
  }
  if (ch.flavor == B2_BZ2_LIBBZ2 && r.run4) {  // libbz2 wants the count byte of the last run of four
    ch.events.push_back({2, slot, 0, 0, DEC_DATA_ERROR, "Data error", ch.total_out, 0, 0});
    return false;
  }
  ch.events.push_back({0, slot, cd.next32, 0, 0, "", ch.total_out, cd.pos, r.rawlen});
  ch.total_out += r.rawlen;
  return true;
}

// The first failure in stream order: event index, code, message, and the bytes the reference has written when it throws
// (a block's own bytes go out before its CRC check).
struct DecErr { long ev = -1; int code = 0; std::string msg; u64 prefix = 0; };

// ---- one decode ----
// Its input, the device window [a, a + wl) of it (last: the window ends the input), the magics found there, the decode
// batch, the chain, and what its replay found.
struct Decode {
  Ctx& c;
  DecIn in;
  const size_t W = dec_window();
  const u32 DB;
  DBuf<u8> win, stage;
  u64 a = 0, wl = 0;
  bool last = false;
  std::vector<Cand> cands;  // the window's magics: sorted by position, or a position list's in list order
  std::vector<size_t> blk;  // the block candidates among them (indices into cands, in order)
  DecScratch B;
  DBuf<Cand> dcand;
  // the decoded blocks waiting for their expansion, one slot each: the L column, the count-byte classes, the tile
  // offsets and the device results.  A sharded share of more than DEC_KEEP_CLS blocks keeps no classes: cls holds one
  // batch's, found again on expansion.
  DBuf<u8> rle, cls;
  DBuf<u32> tileoff;
  DBuf<CandRes> dres;
  bool keep_cls = true;
  std::vector<CandRes> hres;
  size_t kb = 0;  // the batch: block candidates [kb, kb + cnt), in slots [0, cnt)
  u32 cnt = 0;
  std::vector<u64> ob;   // per slot of a delivery: its output offset (~0: not expanded)
  std::vector<u32> got;  // and the CRC of what it expanded to
  Chain ch;
  DecErr E;
  DecRows rows;
  // A share session's imported candidates (parallel to cands): the bytes behind an end-of-stream magic, which only its
  // owner's buffer holds (byte k at bits 8k, their count at bits 32 and up).  Empty: the walk reads the input.
  std::vector<u64> tails;
  // up to 4 bytes at bytepos, behind end-of-stream candidate ci, into h; returns how many there are
  size_t eos_head(size_t ci, u64 bytepos, u8* h) {
    if (tails.empty()) return in.head(c, bytepos, h);
    for (int k = 0; k < 4; k++) h[k] = (u8)(tails[ci] >> (8 * k));
    return (size_t)(tails[ci] >> 32);
  }
  // A libbz2 share session's copy of the stream's last bytes, from the rows (kind 3): by the walk the caller's buffer is
  // gone, and the rank whose block ends the chain may not hold the stream's end.  Unset: the walk reads the input.
  bool end_rows = false;
  std::vector<u8> end_bytes;
  // up to k bytes at bytepos, which lies in the input's last 10 bytes (a magic the input cuts off), into h; returns how
  // many there are
  size_t end_head(u64 bytepos, u8* h, size_t k) {
    if (!end_rows) return in.head(c, bytepos, h, k);
    const u64 len = in.length(), e0 = len - end_bytes.size();
    if (bytepos < e0) throw B2Error{B2_ERR_BAD_ARG, "the share rows lack the stream's last bytes"};
    const size_t avail = (size_t)std::min<u64>(k, len - bytepos);
    memcpy(h, end_bytes.data() + (bytepos - e0), avail);
    return avail;
  }
  // reads no header: every block is held to the largest dbufSize (the recovery decodes blocks wherever they are)
  struct NoHeader {};
  Decode(Ctx& c_, const DecIn& in_, NoHeader) : c(c_), in(in_), DB(dec_batch_blocks(c_)) { ch.cur_dbuf = 900000u; }
  // reads the first header (lib/Bzip2.js:105-124 _start_bunzip)
  Decode(Ctx& c_, const DecIn& in_) : c(c_), in(in_), DB(dec_batch_blocks(c_)) {
    u8 hdr[4] = {0, 0, 0, 0};
    first_header(hdr, in.head(c, 0, hdr));
  }
  // the stream's first `avail` (up to 4) bytes set the first member's dbufSize, or throw
  void first_header(const u8* hdr, size_t avail) {
    if (avail < 4 || hdr[0] != 'B' || hdr[1] != 'Z' || hdr[2] != 'h') throw B2Error{DEC_NOT_BZIP, "Not bzip data: bad magic"};
    const int level = hdr[3] - 0x30;
    if (level < 1 || level > 9) throw B2Error{DEC_NOT_BZIP, "Not bzip data: level out of range"};
    ch.cur_dbuf = 100000u * (u32)level;
  }
  void load(u64 a_, u64 len) {
    a = a_;
    wl = in.window(c, win, a, len);
    last = a + wl == in.length();
  }
  // Every magic of the window below window bit lim, sorted by position, and the block candidates among them.
  void scan(u64 lim) {
    StageScope ss(c, ST_SCAN);
    // Highly repetitive input compresses to a few dozen bytes per block (and multistream files may hold thousands of
    // tiny members), so the number of magics is not bounded by the usual ~100 KB per block: when the first guess is too
    // small the scan counts them all and runs once more with exactly that capacity.
    u32 cap = (u32)(wl / 8000 + 1024);
    DBuf<Cand> dc(c, cap);
    DBuf<u32> dcount(c, 1);
    u32 cnt = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
      CUDA_CHECK(cudaMemsetAsync(dcount, 0, 4, c.stream));
      k_scan_magic<<<(unsigned)(((wl + 3) / 4 + 255) / 256), 256, 0, c.stream>>>(win, wl, a * 8, lim, dc, dcount, cap);
      KLAUNCH(c); KCHECK();
      CUDA_CHECK(cudaMemcpyAsync(&cnt, dcount, 4, cudaMemcpyDeviceToHost, c.stream));
      CUDA_CHECK(cudaStreamSynchronize(c.stream));
      if (cnt <= cap) break;
      cap = cnt;
      dc.alloc(c, cap);
    }
    if (cnt > cap) throw B2Error{B2_ERR_CUDA, "magic scan did not settle"};
    cands.resize(cnt);
    if (cnt) CUDA_CHECK(cudaMemcpyAsync(cands.data(), dc, sizeof(Cand) * cnt, cudaMemcpyDeviceToHost, c.stream));
    CUDA_CHECK(cudaStreamSynchronize(c.stream));
    std::sort(cands.begin(), cands.end(), [](const Cand& x, const Cand& y) { return x.pos < y.pos; });
    blk.clear();
    for (size_t i = 0; i < cands.size(); i++) if (cands[i].type == 1) blk.push_back(i);
  }
  // the first block candidate at or behind bit position pos (an index into blk)
  size_t blk_from(u64 pos) const {
    return (size_t)(std::lower_bound(blk.begin(), blk.end(), pos, [&](size_t ci, u64 p) { return cands[ci].pos < p; }) - blk.begin());
  }
  // slots for nb blocks, the classes of ncls
  void alloc(size_t nb, size_t ncls) {
    rle.alloc(c, nb << SEG_SHIFT); cls.alloc(c, ncls << SEG_SHIFT); tileoff.alloc(c, nb * UR_TPS); dres.alloc(c, nb);
  }
  // slots for the largest batch of the window, kept for the largest of the call
  void reserve() {
    const size_t nbm = std::min<size_t>(DB, blk.size());
    if (nbm > dres.n) { alloc(nbm, nbm); dcand.alloc(c, nbm); }
  }
  // decode block candidates [j0, j0 + n) into slots [s0, s0 + n), their results into h
  void decode(size_t j0, u32 n, size_t s0, CandRes* h) {
    std::vector<Cand> bc(n);
    for (u32 i = 0; i < n; i++) bc[i] = cands[blk[j0 + i]];
    CUDA_CHECK(cudaMemcpyAsync(dcand, bc.data(), sizeof(Cand) * n, cudaMemcpyHostToDevice, c.stream));
    dec_batch(c, B, win, wl, a * 8, last, dcand, n, ch.flavor, dres.p + s0, h, rle.p + (s0 << SEG_SHIFT), cls.p + (keep_cls ? s0 << SEG_SHIFT : 0),
              tileoff.p + s0 * UR_TPS);
  }
  // Expand the slots of [s0, s1) whose ob is not ~0 (RLE1 decode) to dout + ob, and CRC each into got; hres, ob and got
  // are indexed by slot.  Without the classes, DB slots at a time are classified again first.
  void expand(size_t s0, size_t s1, const CandRes* h, const u64* ob, u8* dout, u32* got) {
    const size_t step = keep_cls ? s1 - s0 : DB;
    for (size_t k0 = s0; k0 < s1; k0 += step) {
      const u32 m = (u32)std::min<size_t>(step, s1 - k0);
      StageScope ss(c, ST_UNRLE);
      u8* kcls = cls.p + (keep_cls ? k0 << SEG_SHIFT : 0);
      DBuf<u64> dob(c, m);
      CUDA_CHECK(cudaMemcpyAsync(dob, ob + k0, 8 * (size_t)m, cudaMemcpyHostToDevice, c.stream));
      if (!keep_cls) {
        k_unrle_classify<<<(unsigned)((((size_t)m << SEG_SHIFT) / 8 + 255) / 256), 256, 0, c.stream>>>(rle.p + (k0 << SEG_SHIFT), dres.p + k0, m, kcls);
        KLAUNCH(c); KCHECK();
      }
      k_unrle_emit<<<(unsigned)((size_t)m * UR_TPS), UR_THREADS, 0, c.stream>>>(rle.p + (k0 << SEG_SHIFT), kcls, dres.p + k0, UR_TPS,
                                                                                   tileoff.p + k0 * UR_TPS, dob, dout);
      KLAUNCH(c); KCHECK();
      std::vector<BlkInfo> ranges(m);
      for (u32 i = 0; i < m; i++) {
        memset(&ranges[i], 0, sizeof(BlkInfo));
        if (ob[k0 + i] != ~0ull) { ranges[i].s = ob[k0 + i]; ranges[i].e = ob[k0 + i] + h[k0 + i].rawlen; }
      }
      DBuf<BlkInfo> dr(c, m);
      DBuf<u32> dcrc(c, m);
      CUDA_CHECK(cudaMemcpyAsync(dr, ranges.data(), sizeof(BlkInfo) * m, cudaMemcpyHostToDevice, c.stream));
      crc_ranges(c, dout, dr, ranges, dcrc);
      CUDA_CHECK(cudaMemcpyAsync(got + k0, dcrc, 4 * (size_t)m, cudaMemcpyDeviceToHost, c.stream));
      CUDA_CHECK(cudaStreamSynchronize(c.stream));
    }
  }
  // the batch from block candidate kb on
  void batch() {
    cnt = (u32)std::min<size_t>(DB, blk.size() - kb);
    if (!cnt) return;
    hres.resize(cnt);
    decode(kb, cnt, 0, hres.data());
  }
  // the call's end: *out_n = the decoded size, or on a failure `failed` and the failure is thrown
  void finish(size_t* out_n, u64 failed) const {
    *out_n = (size_t)(E.ev >= 0 ? failed : ch.total_out);
    if (E.ev >= 0) throw B2Error{E.code, E.msg};
  }
};

// libbz2 flavor: does the input end before the 80 bits (magic + CRC) at bit pos, with every whole byte from pos on agreeing
// with the start of a block or end-of-stream magic?  libbz2 reads a magic a byte at a time, so a part byte never differs.
// Only an input whose length is known can be cut off there; a stream that has not ended yet has at least 80 more bits
// once a window is found to hold pos + 80.
static bool cut_magic(Decode& R, u64 pos) {
  const u64 len = R.in.length();
  if (len == SIZE_MAX || pos + 80 <= len * 8) return false;
  const u64 bits = len * 8 > pos ? len * 8 - pos : 0;
  const u32 groups = (u32)std::min<u64>(bits / 8, 6);  // whole bytes of the magic (the CRC behind it always agrees)
  if (!groups) return true;
  u8 h[7] = {0};
  const size_t got = R.end_head(pos >> 3, h, 7);
  const u32 sh = (u32)(pos & 7);
  bool blk = true, eos = true;
  for (u32 k = 0; k < groups; k++) {
    const u32 hi = k < got ? h[k] : 0, lo = k + 1 < got ? h[k + 1] : 0;
    const u8 v = (u8)(((hi << 8 | lo) << sh) >> 8);
    blk = blk && v == (u8)(WHOLEPI >> (40 - 8 * k));
    eos = eos && v == (u8)(SQRTPI >> (40 - 8 * k));
  }
  return blk || eos;
}

// Walk R's chain from ch.pos over the sorted magics as far as the batch has final results (block candidate j of the batch
// is in slot j - kb).  Returns true when the walk stopped for input behind the device window: a magic the window's end
// (bit end_bit) may cut off, or a block whose decode reached that end.
static bool chain_walk(Decode& R, u64 end_bit) {
  Chain& ch = R.ch;
  const bool lb = ch.flavor == B2_BZ2_LIBBZ2;
  while (!ch.done) {
    if (lb && cut_magic(R, ch.pos)) {
      ch.events.push_back({2, 0, 0, 0, DEC_EOF, "Unexpected input EOF", ch.total_out, 0, 0}); ch.done = true; break;
    }
    if ((ch.pos + 7) / 8 >= R.in.length()) { ch.done = true; break; }  // 'eof' in inputStream && inputStream.eof() (lib/Bzip2.js:462)
    const auto it = std::lower_bound(R.cands.begin(), R.cands.end(), ch.pos, [](const Cand& x, u64 p) { return x.pos < p; });
    if (it == R.cands.end() || it->pos != ch.pos) {
      if (ch.pos + 80 > end_bit) return true;
      ch.events.push_back({2, 0, 0, 0, DEC_NOT_BZIP, "Not bzip data", ch.total_out, 0, 0}); ch.done = true; break;
    }
    if (it->type == 1) {
      const size_t j = R.blk_from(ch.pos);
      if (j >= R.kb + R.cnt) return false;  // in a later batch
      const CandRes& r = R.hres[j - R.kb];
      if (r.open) return true;
      ch.stream_crc = it->next32 ^ ((ch.stream_crc << 1) | (ch.stream_crc >> 31));  // lib/Bzip2.js:138-139
      if (!block_event(ch, *it, r, j - R.kb)) { ch.done = true; break; }
      ch.pos = r.endbit;
      continue;
    }
    ch.events.push_back({1, 0, ch.stream_crc, it->next32, 0, "", ch.total_out, 0, 0});
    ch.pos += 80;
    const u64 bytepos = (ch.pos + 7) / 8;
    if (!ch.multistream || bytepos >= R.in.length()) { ch.done = true; break; }
    // _start_bunzip on the byte stream (resyncs to the next byte)
    u8 h2[4] = {0, 0, 0, 0};
    const size_t avail = R.eos_head((size_t)(it - R.cands.begin()), bytepos, h2);
    if (lb) {
      // bzip2 -d: a tail that is not the start of "BZh1".."BZh9" is ignored; a cut-off header is a truncated file
      const char want[3] = {'B', 'Z', 'h'};
      bool match = true;
      for (size_t k = 0; k < avail; k++) match = match && (k < 3 ? h2[k] == (u8)want[k] : h2[k] >= '1' && h2[k] <= '9');
      if (!match) { ch.done = true; break; }
      if (avail < 4) { ch.events.push_back({2, 0, 0, 0, DEC_EOF, "Unexpected input EOF", ch.total_out, 0, 0}); ch.done = true; break; }
    }
    if (avail != 4 || h2[0] != 'B' || h2[1] != 'Z' || h2[2] != 'h') {
      ch.events.push_back({2, 0, 0, 0, DEC_NOT_BZIP, "Not bzip data: bad magic", ch.total_out, 0, 0}); ch.done = true; break;
    }
    const int lv = h2[3] - 0x30;
    if (lv < 1 || lv > 9) { ch.events.push_back({2, 0, 0, 0, DEC_NOT_BZIP, "Not bzip data: level out of range", ch.total_out, 0, 0}); ch.done = true; break; }
    ch.cur_dbuf = (u32)lv * 100000u;
    ch.stream_crc = 0;
    ch.pos = (bytepos + 4) * 8;
  }
  return false;
}

// The same for a position list (lib/Bzip2.js:482-503 once per position), in list order: cands[i] is the magic at the
// i-th position (type 0: none).
static void list_walk(Decode& R) {
  Chain& ch = R.ch;
  while (!ch.done) {
    if (ch.li >= R.cands.size()) { ch.done = true; break; }
    const Cand& cd = R.cands[ch.li];
    if (cd.type == 0) { ch.events.push_back({2, 0, 0, 0, DEC_NOT_BZIP, "Not bzip data", ch.total_out, 0, 0}); ch.done = true; break; }
    if (cd.type == 2) { ch.events.push_back({3, 0, 0, 0, 0, "", ch.total_out, 0, 0}); ch.li++; continue; }
    const size_t j = (size_t)(std::lower_bound(R.blk.begin(), R.blk.end(), ch.li) - R.blk.begin());
    if (j >= R.kb + R.cnt) return;  // in a later batch
    if (!block_event(ch, cd, R.hres[j - R.kb], j - R.kb)) { ch.done = true; break; }
    ch.li++;
  }
}

// Replay events [e0, e1) up to the first failure, which goes to R.E: block CRCs against R.got for the slots s whose offset
// R.ob[s - lo] is set (any other block passes: it was not expanded here, and in a sharded decode its owner checks it),
// stream CRCs unless for a table (Bzip2.table does not check them).  The rows and ends of everything in front of the
// failure go to R.rows.
static void replay(Decode& R, size_t e0, size_t e1, size_t lo, bool table) {
  DecErr& E = R.E;
  for (size_t ei = e0; ei < e1 && E.ev < 0; ei++) {
    const Event& ev = R.ch.events[ei];
    if (ev.kind == 0) {
      const size_t s = ev.slot - lo;
      if (ev.slot >= lo && s < R.ob.size() && R.ob[s] != ~0ull && R.got[s] != ev.a) {
        E.ev = (long)ei; E.code = DEC_DATA_ERROR; E.msg = "Data error: Bad block CRC (got " + hexs(R.got[s]) + " expected " + hexs(ev.a) + ")";
        E.prefix = ev.off + ev.len;
      }
      if (E.ev < 0) { R.rows.pos.push_back(ev.pos); R.rows.len.push_back(ev.len); }
    } else if (ev.kind == 1) {
      if (!table && ev.a != ev.b) {
        E.ev = (long)ei; E.code = DEC_DATA_ERROR; E.msg = "Data error: Bad stream CRC (got " + hexs(ev.a) + " expected " + hexs(ev.b) + ")";
        E.prefix = ev.off;
      }
    } else if (ev.kind == 2) {
      E.ev = (long)ei; E.code = ev.code; E.msg = ev.msg; E.prefix = ev.off;
    }
    if (E.ev < 0) R.rows.ends.push_back(ev.kind == 0 ? ev.off + ev.len : ev.off);
  }
}

// ---- deliveries: expand, CRC-check and replay the block events of [e0, e1), which a walk settled ----
// Device delivery: each block event whose slot s lies in [lo, lo + cnt) goes to dout + off - base from slot s - lo, if it
// fits below cap (one that does not is only counted: the caller reports the size needed).
static void deliver_dev(Decode& R, size_t e0, size_t e1, size_t lo, size_t cnt, u64 base, u8* dout, u64 cap) {
  R.ob.assign(cnt ? cnt : 1, ~0ull);
  R.got.assign(cnt ? cnt : 1, 0);
  for (size_t ei = e0; ei < e1; ei++) {
    const Event& ev = R.ch.events[ei];
    if (ev.kind == 0 && ev.slot >= lo && ev.slot < lo + cnt && ev.off - base + ev.len <= cap) R.ob[ev.slot - lo] = ev.off - base;
  }
  R.expand(0, cnt, R.hres.data() + lo, R.ob.data(), dout, R.got.data());
  replay(R, e0, e1, lo, false);
}

// The staged deliveries: the blocks go through a device staging buffer in groups of consecutive blocks of at most
// max(W, one block) bytes.  group(bytes, off, g_end, last_group) sees each group there (off: its offset in the decoded
// stream, g_end: the end of its events) and ends the delivery by returning false.
template <class Group>
static void stage_groups(Decode& R, size_t e0, size_t e1, Group group) {
  std::vector<size_t> settled;
  for (size_t ei = e0; ei < e1; ei++) if (R.ch.events[ei].kind == 0) settled.push_back(ei);
  R.ob.assign(R.cnt ? R.cnt : 1, ~0ull);
  R.got.assign(R.cnt ? R.cnt : 1, 0);
  for (size_t g0 = 0; g0 < settled.size();) {
    const Event& f = R.ch.events[settled[g0]];
    u64 bytes = f.len;
    size_t g1 = g0 + 1;
    while (g1 < settled.size() && bytes + R.ch.events[settled[g1]].len <= R.W) bytes += R.ch.events[settled[g1++]].len;
    const size_t s0 = f.slot, s1 = R.ch.events[settled[g1 - 1]].slot + 1;
    for (size_t g = g0; g < g1; g++) { const Event& ev = R.ch.events[settled[g]]; R.ob[ev.slot] = ev.off - f.off; }
    if (bytes > R.stage.n) R.stage.alloc(R.c, bytes);
    R.expand(s0, s1, R.hres.data(), R.ob.data(), R.stage, R.got.data());
    if (!group(bytes, f.off, settled[g1 - 1] + 1, g1 == settled.size())) return;
    g0 = g1;
  }
}

// Host delivery: each group's events are replayed before it leaves and the group is cut at the prefix the replay allows,
// so nothing past the prefix of b2_bzip2_decompress_partial ever reaches `out`.
static void deliver_host(Decode& R, size_t e0, size_t e1, StreamOut& out) {
  size_t er = e0;  // events replayed so far
  stage_groups(R, e0, e1, [&](u64 bytes, u64 off, size_t g_end, bool last_group) {
    replay(R, er, g_end, 0, false);
    er = g_end;
    const u64 keep = R.E.ev < 0 ? bytes : (R.E.prefix > off ? std::min<u64>(bytes, R.E.prefix - off) : 0);
    if (keep) {
      // no group follows the last one of a finished chain or a failure: a call of one batch makes one result buffer of
      // exactly its size and one copy
      out.reserve((size_t)keep, (R.ch.done && last_group) || R.E.ev >= 0, R.W);
      u8* dst = out.next();
      {
        StageScope s(R.c, ST_D2H);
        CUDA_CHECK(cudaMemcpyAsync(dst, R.stage, keep, cudaMemcpyDeviceToHost, R.c.stream));
      }
      out.put(dst, (size_t)keep);
    }
    return R.E.ev < 0;
  });
  replay(R, er, e1, 0, false);
}

// CRC-only delivery (a table, or a device decode without an output buffer): the blocks are expanded for their CRCs only.
static void deliver_crc(Decode& R, size_t e0, size_t e1, bool table) {
  stage_groups(R, e0, e1, [](u64, u64, size_t, bool) { return true; });
  replay(R, e0, e1, 0, table);
}

// ---- single-GPU drivers ----
// A chain decode: one rolling loop over input windows and decode batches.  Only the window [a, a + W) of the input is on
// the device (W = dec_window(); a is the chain's position, rounded down to 256 bytes).  The window's magics are decoded in
// position order, a batch at a time; after each batch the host walks the chain as far as final results allow, and
// deliver(e0, e1) delivers the blocks that walk settled.  The first chain position without a final result starts the
// next window; a window that would start where this one did is twice as long, so a block longer than W still decodes.
// The first failure in stream order ends the walk, unless past_error (the device delivery walks on for the needed size).
template <class Deliver>
static void chain_decode(Decode& R, int multistream, bool past_error, Deliver deliver) {
  Chain& ch = R.ch;
  ch.multistream = multistream;
  u64 prev_a = ~0ull;
  size_t wcur = R.W;
  while (!ch.done && (R.E.ev < 0 || past_error)) {
    const u64 a = (ch.pos >> 3) & ~(u64)255;
    wcur = a == prev_a ? wcur * 2 : R.W;
    prev_a = a;
    R.load(a, wcur);
    // a magic whose 80 bits (magic + CRC) run past the window's end belongs to the next window
    const u64 bits = R.wl * 8;
    R.scan(R.last ? bits : (bits >= 80 ? bits - 79 : 0));
    R.reserve();
    R.kb = R.blk_from(ch.pos);
    for (;;) {
      R.batch();
      const size_t e0 = ch.events.size();
      const bool need_window = chain_walk(R, R.last ? ~0ull : (R.a + R.wl) * 8);
      deliver(e0, ch.events.size());
      if (ch.done || (R.E.ev >= 0 && !past_error) || need_window) break;
      const size_t nk = R.blk_from(ch.pos);
      if (nk <= R.kb) throw B2Error{B2_ERR_CUDA, "bzip2 decode: the chain walk made no progress"};
      R.kb = nk;
    }
  }
  CUDA_CHECK(cudaStreamSynchronize(R.c.stream));
}

void bzip2_decompress_dev(Ctx& c, const u8* d_in, size_t n, int multistream, int flavor, u8* d_out, size_t out_cap, size_t* out_n) {
  *out_n = 0;
  Decode R(c, DecIn(d_in, n));
  R.ch.flavor = flavor;
  chain_decode(R, multistream, true, [&](size_t e0, size_t e1) {
    // a walk that settled no block expands nothing
    const auto& ev = R.ch.events;
    const bool any = std::any_of(ev.begin() + (long)e0, ev.begin() + (long)e1, [](const Event& x) { return x.kind == 0; });
    deliver_dev(R, e0, e1, 0, any ? R.cnt : 0, 0, d_out, out_cap);
  });
  if (R.ch.total_out > out_cap) {
    *out_n = (size_t)R.ch.total_out;
    throw B2Error{B2_ERR_BAD_ARG, "output buffer too small"};
  }
  R.finish(out_n, 0);
}

void bzip2_decompress_size(Ctx& c, const u8* d_in, size_t n, int multistream, int flavor, size_t* out_n) {
  *out_n = 0;
  Decode R(c, DecIn(d_in, n));
  R.ch.flavor = flavor;
  chain_decode(R, multistream, false, [&](size_t e0, size_t e1) { deliver_crc(R, e0, e1, false); });
  R.finish(out_n, 0);
}

void bzip2_decompress_host(Ctx& c, StreamIn& in, int multistream, int flavor, StreamOut& out, size_t* out_n) {
  *out_n = 0;
  Decode R(c, DecIn(in));
  R.ch.flavor = flavor;
  chain_decode(R, multistream, false, [&](size_t e0, size_t e1) { deliver_host(R, e0, e1, out); });
  R.finish(out_n, R.E.prefix);
}

void bzip2_table(Ctx& c, StreamIn& in, int multistream, DecRows& rows, size_t* out_n) {
  *out_n = 0;
  Decode R(c, DecIn(in));
  chain_decode(R, multistream, false, [&](size_t e0, size_t e1) { deliver_crc(R, e0, e1, true); });
  rows = std::move(R.rows);
  R.finish(out_n, 0);
}

// A position list: the whole input on the device, only the given positions tested for a magic, the blocks decoded a
// batch at a time in list order.  The first position without a magic raises "Not bzip data", so nothing behind it is
// decoded.
void bzip2_decompress_list(Ctx& c, StreamIn& in, const std::vector<u64>& positions, StreamOut& out, DecRows& rows, size_t* out_n) {
  *out_n = 0;
  Decode R(c, DecIn(in));
  const size_t n = R.in.length();  // the input is complete
  R.load(0, n);
  {
    StageScope ss(c, ST_SCAN);
    const size_t np = positions.size();
    DBuf<u64> dpos(c, np);
    DBuf<Cand> dc(c, np);
    R.cands.resize(np);
    CUDA_CHECK(cudaMemcpyAsync(dpos, positions.data(), 8 * np, cudaMemcpyHostToDevice, c.stream));
    k_magic_at<<<(unsigned)((np + 255) / 256), 256, 0, c.stream>>>(R.win, n, dpos, np, dc);
    KLAUNCH(c); KCHECK();
    CUDA_CHECK(cudaMemcpyAsync(R.cands.data(), dc, sizeof(Cand) * np, cudaMemcpyDeviceToHost, c.stream));
    CUDA_CHECK(cudaStreamSynchronize(c.stream));
  }
  for (size_t i = 0; i < R.cands.size(); i++) {
    if (R.cands[i].type == 0) { R.cands.resize(i + 1); break; }
    if (R.cands[i].type == 1) R.blk.push_back(i);
  }
  R.reserve();
  for (;;) {
    R.batch();
    const size_t e0 = R.ch.events.size();
    list_walk(R);
    deliver_host(R, e0, R.ch.events.size(), out);
    if (R.ch.done || R.E.ev >= 0) break;
    if (!R.cnt) throw B2Error{B2_ERR_CUDA, "bzip2 decode: the chain walk made no progress"};
    R.kb += R.cnt;
  }
  CUDA_CHECK(cudaStreamSynchronize(c.stream));
  rows = std::move(R.rows);
  R.finish(out_n, R.E.prefix);
}

// ---- block recovery ----------------------------------------------------------------------------
// Bit splice: range k copies bits [src, src + nbits) of the source to bits [dst, dst + nbits) of the destination (MSB
// first, any phase to any phase).  One CTA per range; each thread builds whole 32-bit destination words from two source
// words.  A word the range covers entirely is stored; the first and last words of a range may be shared with its
// neighbours and are ORed in, so the destination is zeroed first.  The source is read up to 8 bytes past its last range
// (the decode window is zero padded), the destination written up to the word that holds its last bit.
struct SpliceRange { u64 src, dst, nbits; };
__global__ void __launch_bounds__(256) k_splice(const u8* __restrict__ src, const SpliceRange* __restrict__ ranges, u8* __restrict__ dst) {
  const SpliceRange s = ranges[blockIdx.x];
  if (!s.nbits) return;
  const u32* sw = reinterpret_cast<const u32*>(src);
  u32* dw = reinterpret_cast<u32*>(dst);
  const u64 w0 = s.dst >> 5, w1 = (s.dst + s.nbits - 1) >> 5, e = s.dst + s.nbits;
  const long long off = (long long)s.src - (long long)s.dst;
  for (u64 w = w0 + threadIdx.x; w <= w1; w += blockDim.x) {
    const long long sb = (long long)(w * 32) + off;  // source bit of the word's first bit: >= -31
    const long long q = sb >> 5;
    const u32 hi = q >= 0 ? __byte_perm(sw[q], 0, 0x0123) : 0u, lo = __byte_perm(sw[q + 1], 0, 0x0123);
    const u32 v = __funnelshift_l(lo, hi, (u32)(sb & 31));
    const u64 b0 = w * 32;
    const u32 from = s.dst > b0 ? (u32)(s.dst - b0) : 0u, to = e < b0 + 32 ? (u32)(e - b0) : 32u;
    if (from == 0 && to == 32) {
      dw[w] = __byte_perm(v, 0, 0x0123);
    } else {
      const u32 m = (0xffffffffu >> from) & (to == 32 ? 0xffffffffu : ~(0xffffffffu >> to));
      atomicOr(dw + w, __byte_perm(v & m, 0, 0x0123));
    }
  }
}

// The walk's state and the output of a recovery.
struct Recover {
  Decode& R;
  bool repair;
  StreamOut& out;
  std::vector<b2_recovered_block>& rows;
  u64 end = 0;         // the bit behind the last intact block's end-of-block code
  u64 total = 0;       // recovered bytes so far
  u32 scrc = 0;        // combined CRC of the intact blocks (lib/Bzip2.js:138-139)
  u8 carry = 0;        // the repaired stream's last partial byte (carry_bits bits, MSB first)
  u32 carry_bits = 0;
  DBuf<u8> sbuf;       // one delivery group of the repaired stream
};

// n bytes at p (host) to the sink
static void rec_put_host(Recover& V, const u8* p, size_t n) {
  V.out.reserve(n, false, V.R.W);
  u8* d = V.out.next();
  memcpy(d, p, n);
  V.out.put(d, n);
}
// n bytes at d (device) to the sink
static void rec_put_dev(Recover& V, const u8* d, size_t n) {
  V.out.reserve(n, false, V.R.W);
  u8* h = V.out.next();
  {
    StageScope s(V.R.c, ST_D2H);
    CUDA_CHECK(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, V.R.c.stream));
  }
  V.out.put(h, n);
}

// The repaired stream's bits of one delivery group: the ranges (window bits) go back to back behind the carried partial
// byte, in one launch; the whole bytes go to the sink and the partial last byte is carried to the next group.
static void rec_splice(Recover& V, std::vector<SpliceRange>& sp) {
  if (sp.empty()) return;
  Ctx& c = V.R.c;
  u64 bits = V.carry_bits;
  for (auto& x : sp) { x.dst = bits; bits += x.nbits; }
  const size_t cap = ((bits + 31) / 32) * 4;
  if (cap > V.sbuf.n) V.sbuf.alloc(c, cap);
  CUDA_CHECK(cudaMemsetAsync(V.sbuf, 0, cap, c.stream));
  if (V.carry_bits) CUDA_CHECK(cudaMemcpyAsync(V.sbuf, &V.carry, 1, cudaMemcpyHostToDevice, c.stream));
  DBuf<SpliceRange> dsp(c, sp.size());
  CUDA_CHECK(cudaMemcpyAsync(dsp, sp.data(), sizeof(SpliceRange) * sp.size(), cudaMemcpyHostToDevice, c.stream));
  k_splice<<<(unsigned)sp.size(), 256, 0, c.stream>>>(V.R.win, dsp, V.sbuf);
  KLAUNCH(c); KCHECK();
  const size_t whole = (size_t)(bits / 8);
  V.carry_bits = (u32)(bits & 7);
  if (whole) rec_put_dev(V, V.sbuf, whole);
  V.carry = 0;
  if (V.carry_bits) CUDA_CHECK(cudaMemcpyAsync(&V.carry, V.sbuf.p + whole, 1, cudaMemcpyDeviceToHost, c.stream));
  CUDA_CHECK(cudaStreamSynchronize(c.stream));
}

// Settle the batch's candidates in position order, one staging group at a time: every candidate that decoded is
// expanded for its CRC, then the walk gives each its row, and the group's intact blocks go out (bytes: runs of
// consecutive blocks from staging; repair: their bit ranges spliced from the window).  Returns false when a candidate
// that starts at or behind the walk's end has no final result (its decode reached the end of a window that does not end
// the input): *next is then its position, and nothing from it on is settled.
static bool recover_batch(Recover& V, u64* next) {
  Decode& R = V.R;
  const u32 cnt = R.cnt;
  auto decoded = [&](u32 s) { return R.hres[s].status == 0 && !R.hres[s].open; };
  R.ob.assign(cnt, ~0ull);
  R.got.assign(cnt, 0);
  for (u32 g0 = 0; g0 < cnt;) {
    u64 bytes = 0;
    u32 g1 = g0;
    for (; g1 < cnt; g1++) {
      if (!decoded(g1)) continue;
      if (bytes && bytes + R.hres[g1].rawlen > R.W) break;
      R.ob[g1] = bytes;
      bytes += R.hres[g1].rawlen;
    }
    if (bytes) {
      if (bytes > R.stage.n) R.stage.alloc(R.c, bytes);
      R.expand(g0, g1, R.hres.data(), R.ob.data(), R.stage, R.got.data());
    }
    std::vector<SpliceRange> sp;
    u64 run0 = ~0ull, run1 = 0;  // staging bytes of the current run of intact blocks
    auto deliver = [&]() {
      if (run0 != ~0ull) rec_put_dev(V, R.stage.p + run0, run1 - run0);
      run0 = ~0ull;
      rec_splice(V, sp);
    };
    for (u32 s = g0; s < g1; s++) {
      const Cand& cd = R.cands[R.blk[R.kb + s]];
      const CandRes& r = R.hres[s];
      b2_recovered_block row = {cd.pos, 0, V.total, 0, cd.next32, 0, B2_REC_INSIDE};
      if (cd.pos >= V.end) {
        if (r.open) { deliver(); *next = cd.pos; return false; }
        if (r.status != 0) {
          row.status = r.status == DEC_OBSOLETE ? B2_REC_OBSOLETE : B2_REC_DATA_ERROR;
        } else {
          row.endbit = r.endbit; row.size = r.rawlen; row.got = R.got[s];
          row.status = row.got == cd.next32 ? B2_REC_INTACT : B2_REC_BAD_CRC;
        }
      }
      if (row.status == B2_REC_INTACT) {
        V.end = r.endbit;
        V.total += r.rawlen;
        V.scrc = cd.next32 ^ ((V.scrc << 1) | (V.scrc >> 31));
        if (V.repair) {
          sp.push_back({cd.pos - R.a * 8, 0, r.endbit - cd.pos});
        } else if (run0 != ~0ull && R.ob[s] == run1) {
          run1 += r.rawlen;
        } else {
          if (run0 != ~0ull) rec_put_dev(V, R.stage.p + run0, run1 - run0);
          run0 = R.ob[s]; run1 = run0 + r.rawlen;
        }
      }
      V.rows.push_back(row);
    }
    deliver();
    g0 = g1;
  }
  return true;
}

// Block recovery: every block magic of the input is a candidate, decoded as Bzip2.decompressBlock decodes a block of a
// BZh9 file, and walked in position order: a candidate that starts inside the last intact block is INSIDE, any other
// is INTACT when it decodes and its CRC matches (the walk's end moves behind it), else it gets the status its decode
// failed with.  The loop has the chain decode's shape: windows [a, a + W) of the input (no magic whose 80 bits cross a
// window's end is taken from it), batches of B candidates, and the next window starts at the first candidate without a
// final result, twice as long when it would start where this one did.  No header is read: any input is walked to its
// end.  The output is the intact blocks' bytes, or (repair) one BZh9 stream of their bits followed by the end-of-stream
// magic and the combined CRC.
void bzip2_recover(Ctx& c, StreamIn& in, bool repair, StreamOut& out, std::vector<b2_recovered_block>& rows) {
  Decode R(c, DecIn(in), Decode::NoHeader{});
  Recover V{R, repair, out, rows};
  if (repair) rec_put_host(V, reinterpret_cast<const u8*>("BZh9"), 4);
  u64 next = 0, prev_a = ~0ull;  // next: the first candidate position without a row
  size_t wcur = R.W;
  for (;;) {
    const u64 a = (next >> 3) & ~(u64)255;
    wcur = a == prev_a ? wcur * 2 : R.W;
    prev_a = a;
    R.load(a, wcur);
    const u64 bits = R.wl * 8, lim = R.last ? bits : (bits >= 80 ? bits - 79 : 0);
    if (R.wl) {
      R.scan(lim);
    } else {
      R.cands.clear(); R.blk.clear();
    }
    R.reserve();
    bool settled = true;
    for (R.kb = R.blk_from(next); R.kb < R.blk.size(); R.kb += R.cnt) {
      R.batch();
      if (!(settled = recover_batch(V, &next))) break;
    }
    if (settled) {
      if (R.last) break;
      next = std::max(next, R.a * 8 + lim);
    }
  }
  if (repair) {
    // the end-of-stream magic, the combined CRC and zero bits to the next byte, behind the carried bits
    u8 t[12] = {0};
    const u64 tail[2] = {SQRTPI, V.scrc};
    const u32 tlen[2] = {48, 32};
    u32 nb = V.carry_bits;
    t[0] = V.carry;
    for (int k = 0; k < 2; k++)
      for (int i = (int)tlen[k] - 1; i >= 0; i--, nb++)
        if ((tail[k] >> i) & 1) t[nb >> 3] |= (u8)(0x80u >> (nb & 7));
    rec_put_host(V, t, (nb + 7) / 8);
  }
  CUDA_CHECK(cudaStreamSynchronize(c.stream));
}

// ---- sharded decode (SURVEY.md section 8e): open on every rank, exchange results, finish ------------
// Two kinds of session, one slot, which differ only in their input, the candidates a rank owns and the rows it imports:
//  - the whole input (b2_dec_shard_*): every rank holds the stream, scans all of it (one window: the whole input, zero
//    padded) and decodes the share [lo, hi) of its block candidates; the rows are the block results, in candidate order.
//  - shares (b2_dec_share_*): a rank holds bytes [g0, g0 + hold) of the stream and owns the magics at bit positions
//    [8 g0, 8 (g0 + share_len)); it scans and decodes those only (one window over its buffer), and its rows carry the
//    candidates themselves, the bytes behind its end-of-stream magics and the stream's first bytes (include/b2bz.h); in
//    the libbz2 flavor, a rank whose buffer ends the stream also exports the stream's last bytes, which R4 reads.
// finish walks the chain over ALL candidates' results (imported from the other ranks), expands + CRC-checks the blocks
// of the own share and raises the reference's errors in stream order.  A rank keeps its share's results until the
// all-gather, so its device memory grows with its share of the file.
struct DecSession {
  Decode R;  // hres: one entry per block candidate (the own share's after open, all after the import)
  size_t lo = 0, hi = 0;
  // shares: the owned bit range, and the stream's first bytes from the rows (read by the rank that owns bit 0)
  bool share = false;
  u64 own0 = 0, own1 = 0;
  u8 hdr[4] = {0, 0, 0, 0};
  size_t hdr_n = 0;
  // libbz2 shares: the stream's last bytes, exported by a rank whose buffer ends the stream (ends: it does)
  bool ends = false;
  u8 last[10] = {0};
  size_t last_n = 0;

  bool libbz2() const { return R.ch.flavor == B2_BZ2_LIBBZ2; }
  // the detail word of a block's row: bit 1 carries run4 (R3) in the libbz2 flavor, so that every rank's walk sees it
  u64 detail(const CandRes& r) const { return r.detail | (libbz2() && r.run4 ? 2u : 0u); }
  static void set_detail(CandRes& r, u64 w) { r.detail = (u32)(w & ~2ull); r.run4 = (u32)(w >> 1 & 1); }

  DecSession(Ctx& c, const u8* d_in, size_t n, int rank, int world, int flavor) : R(c, DecIn(d_in, n)) {
    R.ch.flavor = flavor;
    R.load(0, n);
    R.in = DecIn(R.win.p, n);  // later headers are read from the session's copy: the caller's buffer may be gone by then
    R.scan(n * 8);
    const size_t nb_all = R.blk.size();
    R.hres.assign(nb_all, CandRes());
    for (auto& r : R.hres) { memset(&r, 0, sizeof r); r.status = DEC_DATA_ERROR; }
    lo = (size_t)rank * nb_all / (size_t)world;
    hi = (size_t)(rank + 1) * nb_all / (size_t)world;
    decode_own(n);
  }

  DecSession(Ctx& c, const u8* d_buf, size_t hold, u64 g0, size_t share_len, size_t total, int flavor)
      : R(c, DecIn(d_buf, hold, g0, total), Decode::NoHeader{}), share(true), own0(8 * g0), own1(8 * (g0 + share_len)) {
    R.ch.flavor = flavor;
    if (g0 == 0 && share_len) hdr_n = R.in.head(c, 0, hdr);
    ends = libbz2() && g0 + hold == total;
    last_n = ends ? std::min<size_t>(hold, sizeof last) : 0;
    if (last_n) R.in.head(c, total - last_n, last, last_n);
    if (share_len) {
      // One window over the buffer from the word that holds byte g0: k_scan_magic and k_hdec take a window that starts
      // at a multiple of 32 bits, and the bytes in front of g0 read as zeros.  The scan stops at the owned range's end
      // (the halo holds the 80 bits of a magic that starts in front of it); a magic in front of g0 is the rank before's.
      const u64 a = g0 & ~(u64)3;
      R.load(a, g0 + hold - a);
      R.scan(own1 - a * 8);
      R.cands.erase(R.cands.begin(), std::lower_bound(R.cands.begin(), R.cands.end(), own0, [](const Cand& x, u64 p) { return x.pos < p; }));
      // the bytes a multistream walk reads behind each end-of-stream magic (the next member's header)
      R.tails.assign(R.cands.size(), 0);
      R.blk.clear();
      for (size_t i = 0; i < R.cands.size(); i++) {
        if (R.cands[i].type == 1) { R.blk.push_back(i); continue; }
        const u64 bytepos = (R.cands[i].pos + 80 + 7) / 8;
        if (bytepos >= total) continue;
        u8 h[4] = {0, 0, 0, 0};
        const u64 k = R.in.head(c, bytepos, h);
        R.tails[i] = k << 32 | (u64)h[0] | (u64)h[1] << 8 | (u64)h[2] << 16 | (u64)h[3] << 24;
      }
    }
    hi = R.blk.size();
    R.hres.assign(hi, CandRes());
    decode_own(hold);
    R.win = DBuf<u8>();  // finish reads nothing of the input
  }

  // Decodes the own block candidates [lo, hi) into slots [0, hi - lo); in_bytes: the input the session holds.
  void decode_own(size_t in_bytes) {
    Ctx& c = R.c;
    const size_t nb = hi - lo;
    {
      // every block of the own share keeps 2 MiB (L column + count-byte classes; 1 MiB beyond DEC_KEEP_CLS blocks) until
      // the stream is assembled, and a batch of up to 2048 blocks needs ~20 MiB of scratch per block: say so instead of
      // failing inside an allocation
      const size_t need = nb * ((size_t)(nb <= dec_keep_cls_limit() ? 2 : 1) << 20) + std::min<size_t>(nb, R.DB) * ((size_t)20 << 20) + in_bytes;
      // memory the stream-ordered pool holds but does not use is available too: when that covers the call (every call
      // after the first of a kind) the driver is not asked at all -- cudaMemGetInfo takes milliseconds on a busy context
      uint64_t reserved = 0, used = 0;
      cudaMemPool_t pool;
      if (cudaDeviceGetDefaultMemPool(&pool, c.device) == cudaSuccess) {
        cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved);
        cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used);
      }
      cudaGetLastError();
      const size_t spare = (size_t)(reserved > used ? reserved - used : 0);
      size_t free_b = 0, total_b = 0;
      if (need > spare) {
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
          if (need > free_b + spare) {
            char msg[256];
            snprintf(msg, sizeof msg, "stream of %zu blocks needs about %zu MiB of device memory for one sharded call (%zu MiB free): decode it "
                                      "on more GPUs, or on one (decompressFile), whose device memory does not grow with the file", nb, need >> 20, free_b >> 20);
            throw B2Error{B2_ERR_CUDA, msg};
          }
        } else cudaGetLastError();
      }
    }
    // The count-byte classes of a block are needed twice (length scan here, expansion in finish).  Up to DEC_KEEP_CLS
    // blocks they stay on the device in between; a share of more blocks (tens of GB of level-1 data) keeps only the L
    // columns (1 MiB per block) and classifies a second time, batch by batch, when it expands them.
    R.keep_cls = nb <= dec_keep_cls_limit();
    R.alloc(nb ? nb : 1, R.keep_cls ? (nb ? nb : 1) : std::min<size_t>(nb, R.DB));
    R.dcand.alloc(c, std::max<size_t>(std::min<size_t>(nb, R.DB), 1));
    for (size_t k0 = 0; k0 < nb; k0 += R.DB) R.decode(lo + k0, (u32)std::min<size_t>(R.DB, nb - k0), k0, R.hres.data() + lo + k0);
    CUDA_CHECK(cudaStreamSynchronize(c.stream));
    R.B = DecScratch();  // the batch scratch is not kept until finish
  }

  // The rows of b2_dec_share_export, B2_SHARE_ROW words each: the stream's first bytes (on the rank that owns bit 0),
  // then every owned candidate in position order, then the stream's last bytes (libbz2, on a rank whose buffer ends it).
  size_t share_rows() const { return (size_t)(own0 == 0 && own1 > 0) + R.cands.size() + ends; }
  void share_export(u64* buf) const {
    u64* o = buf;
    if (own0 == 0 && own1 > 0) {
      memset(o, 0, 8 * B2_SHARE_ROW);
      o[10] = (u64)hdr_n << 32 | (u64)hdr[0] | (u64)hdr[1] << 8 | (u64)hdr[2] << 16 | (u64)hdr[3] << 24;
      o += B2_SHARE_ROW;
    }
    size_t j = 0;
    for (size_t i = 0; i < R.cands.size(); i++, o += B2_SHARE_ROW) {
      const Cand& cd = R.cands[i];
      memset(o, 0, 8 * B2_SHARE_ROW);
      o[0] = cd.pos; o[1] = cd.type; o[2] = cd.next32; o[10] = R.tails[i];
      if (cd.type != 1) continue;
      const CandRes& r = R.hres[j++];
      // an obsolete block's decode stops before its origPtr, which the walk does not read then
      o[3] = (u64)(long long)r.status; o[4] = detail(r); o[5] = r.endbit; o[6] = r.n; o[7] = r.rawlen;
      o[8] = r.status == DEC_OBSOLETE ? 0 : r.orig; o[9] = r.open;
    }
    if (ends) {
      memset(o, 0, 8 * B2_SHARE_ROW);
      o[0] = R.in.length() - last_n; o[1] = 3; o[2] = last_n;
      for (size_t k = 0; k < last_n; k++) o[3 + k / 8] |= (u64)last[k] << (8 * (k % 8));
    }
  }
  // Every rank's rows, in rank order, become the candidates and results the walk sees; the own ones keep the results
  // of this session's decode.
  void share_import(const u64* all, size_t count) {
    std::vector<Cand> cands;
    std::vector<u64> tails;
    std::vector<CandRes> hres;
    bool head = false;
    size_t own_c = 0, own_b = 0;
    const u64 total = R.in.length();
    for (size_t i = 0; i < count; i++) {
      const u64* o = all + i * B2_SHARE_ROW;
      if (o[1] == 3) {  // the stream's last bytes: the row with the most of them
        if (o[2] > 10 || o[0] + o[2] != total) throw B2Error{B2_ERR_BAD_ARG, "a share row of the stream's last bytes that does not end it"};
        if (o[2] > R.end_bytes.size()) {
          R.end_bytes.resize((size_t)o[2]);
          for (size_t k = 0; k < o[2]; k++) R.end_bytes[k] = (u8)(o[3 + k / 8] >> (8 * (k % 8)));
        }
        continue;
      }
      if (o[1] > 2 || (o[1] && !cands.empty() && o[0] <= cands.back().pos)) throw B2Error{B2_ERR_BAD_ARG, "share rows out of order or of an unknown kind"};
      if (o[1] == 0) {
        if (!head) for (int k = 0; k < 4; k++) hdr[k] = (u8)(o[10] >> (8 * k));
        if (!head) hdr_n = (size_t)std::min<u64>(o[10] >> 32, 4);
        head = true;
        continue;
      }
      const bool mine = o[0] >= own0 && o[0] < own1;
      own_c += mine;
      cands.push_back(Cand{o[0], (u32)o[1], (u32)o[2]});
      tails.push_back(o[10]);
      if (o[1] != 1) continue;
      if (mine) {
        if (own_b >= R.hres.size()) throw B2Error{B2_ERR_BAD_ARG, "the share rows do not hold this rank's candidates"};
        if (own_b == 0) lo = hres.size();
        hres.push_back(R.hres[own_b++]);
        continue;
      }
      CandRes r;
      memset(&r, 0, sizeof r);
      r.status = (int)(long long)o[3]; set_detail(r, o[4]); r.endbit = o[5]; r.n = (u32)o[6]; r.rawlen = (u32)o[7]; r.orig = (u32)o[8];
      r.open = (u32)o[9];
      hres.push_back(r);
    }
    if (own_c != R.cands.size() || own_b != R.hres.size()) throw B2Error{B2_ERR_BAD_ARG, "the share rows do not hold this rank's candidates"};
    if (!own_b) lo = 0;
    hi = lo + own_b;
    if (!head) hdr_n = 0;
    R.end_rows = libbz2();  // cut_magic reads the stream's end from the rows
    R.cands = std::move(cands);
    R.tails = std::move(tails);
    R.hres = std::move(hres);
    R.blk.clear();
    for (size_t i = 0; i < R.cands.size(); i++) if (R.cands[i].type == 1) R.blk.push_back(i);
  }

  // Walks the chain over every rank's results, expands the own blocks into d_out (or a buffer of its own), fills info
  // and returns true.  Throws the first failure in stream order; info[3] tells the ranks which failure is the earliest.
  // Returns false, having delivered nothing, when the walk reaches a block that decoded past the end of its owner's
  // buffer: only a share session has such blocks (a whole-input session's one window ends the input).
  bool finish(int multistream, u8* d_out, size_t out_cap, u64* info) {
    Chain& ch = R.ch;
    ch.multistream = multistream;
    R.kb = 0;  // the batch the walk sees: every block candidate
    R.cnt = (u32)R.hres.size();
    if (chain_walk(R, ~0ull)) return false;
    // own output window: [my_off, my_off + my_len) of the decoded stream, from the first to the last own block
    auto mine = [&](const Event& ev) { return ev.kind == 0 && ev.slot >= lo && ev.slot < hi; };
    const auto f = std::find_if(ch.events.begin(), ch.events.end(), mine);
    const auto l = std::find_if(ch.events.rbegin(), ch.events.rend(), mine);
    const u64 my_off = f == ch.events.end() ? 0 : f->off, my_len = f == ch.events.end() ? 0 : l->off + l->len - my_off;
    DBuf<u8> own;
    if (!d_out) {
      own.alloc(R.c, my_len ? my_len : 1);
      d_out = own.p;
      out_cap = my_len;
    } else if (my_len > out_cap) {
      throw B2Error{B2_ERR_BAD_ARG, "output buffer too small"};
    }
    deliver_dev(R, 0, ch.events.size(), lo, hi - lo, my_off, d_out, out_cap);
    info[0] = my_off; info[1] = my_len; info[2] = ch.total_out; info[3] = (u64)(long long)R.E.ev; info[4] = (u64)(long long)R.E.code;
    // the caller compares info[3] across ranks and keeps the earliest
    if (R.E.ev >= 0) throw B2Error{R.E.code, R.E.msg};
    return true;
  }
};

static std::unique_ptr<DecSession> g_shard;
void dec_shard_release() { g_shard.reset(); }
void dec_shard_open(Ctx& c, const u8* d_in, size_t n, int rank, int world, int flavor, u64* info) {
  g_shard.reset();
  g_shard = std::make_unique<DecSession>(c, d_in, n, rank, world, flavor);
  info[0] = g_shard->R.blk.size(); info[1] = g_shard->lo; info[2] = g_shard->hi;
}
static DecSession& session(bool share) {
  if (!g_shard || g_shard->share != share) throw B2Error{B2_ERR_BAD_ARG, share ? "no share decode in flight" : "no sharded decode in flight"};
  return *g_shard;
}
void dec_shard_export(u64* buf) {
  const DecSession& S = session(false);
  for (size_t i = S.lo; i < S.hi; i++) {
    const CandRes& r = S.R.hres[i];
    u64* o = buf + (i - S.lo) * 6;
    o[0] = (u64)(long long)r.status; o[1] = S.detail(r); o[2] = r.endbit; o[3] = r.n; o[4] = r.rawlen; o[5] = r.orig;
  }
}
void dec_shard_finish(const u64* all, int multistream, u8* d_out, size_t out_cap, u64* res) {
  session(false);
  const std::unique_ptr<DecSession> S = std::move(g_shard);  // the session ends with this call
  for (size_t i = 0; i < S->R.hres.size(); i++) {
    if (i >= S->lo && i < S->hi) continue;
    const u64* o = all + i * 6;
    CandRes& r = S->R.hres[i];
    r.status = (int)(long long)o[0]; DecSession::set_detail(r, o[1]); r.endbit = o[2]; r.n = (u32)o[3]; r.rawlen = (u32)o[4]; r.orig = (u32)o[5];
  }
  S->finish(multistream, d_out, out_cap, res);
}

void dec_share_open(Ctx& c, const u8* d_buf, size_t hold, u64 g0, size_t share_len, size_t total, int flavor, u64* info) {
  g_shard.reset();
  g_shard = std::make_unique<DecSession>(c, d_buf, hold, g0, share_len, total, flavor);
  info[0] = g_shard->share_rows(); info[1] = g_shard->R.cands.size(); info[2] = g_shard->R.blk.size();
}
void dec_share_export(u64* buf) { session(true).share_export(buf); }
void dec_share_finish(const u64* all, size_t count, int multistream, u8* d_out, size_t out_cap, u64* res) {
  session(true);
  const std::unique_ptr<DecSession> S = std::move(g_shard);  // the session ends with this call
  for (int k = 0; k < 6; k++) res[k] = 0;
  res[3] = ~0ull;
  S->share_import(all, count);
  try {
    S->R.first_header(S->hdr, S->hdr_n);  // lib/Bzip2.js:105-124 _start_bunzip: the stream's first failure
  } catch (const B2Error& e) {
    res[3] = 0; res[4] = (u64)(long long)e.code;
    throw;
  }
  res[5] = S->finish(multistream, d_out, out_cap, res) ? 0 : 1;
}
