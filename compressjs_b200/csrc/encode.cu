// encode.cu -- bit packing of the .bz2 stream and the compressFile driver.
//
// Reference: lib/Bzip2.js:879-929 (compressFile: "BZh"+level, per block magic/CRC/body,
// trailer magic + stream CRC, zero pad), :735-876 (compressBlock body layout, SURVEY.md
// Appendix B) and lib/BitStream.js:52-105 (MSB-first bit order).
//
// The reference pushes one bit at a time through a BitStream.  Here every block's total bit
// length is known after the Huffman stage, so an exclusive scan gives each block its final bit
// offset in the file and all blocks are packed in place concurrently:
//   k_offsets     : one warp: running bit cursor (scan) + stream CRC fold (rotl1 ^ crc, lib/Bzip2.js:917)
//   k_pack_header : per block: magic, CRC, pidx, symbol map, selectors (unary of the MTF'd table
//                   ids, offsets by prefix sum), code-length tables (delta coded)
//   k_pack_codes  : per 128 groups: every group's bit offset comes from the Huffman stage, so each
//                   thread encodes its 50 symbols straight into a shared-memory staging tile that is
//                   aligned to the global 32-bit word grid, then the tile is written out coalesced
//                   (only the two boundary words need atomics)
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <optional>
#include <vector>
#include "enc.h"

// ---- bit writers (stream is MSB first; words are stored big-endian) ----------------------
__device__ __forceinline__ u32 bswap32(u32 v) { return __byte_perm(v, 0, 0x0123); }

// OR `nbits` (<= 32) of `val` into a zero-initialised global stream at absolute bit `pos`
__device__ __forceinline__ void gput(u32* out, u64 pos, u32 nbits, u32 val) {
  if (nbits == 0) return;
  const u64 w = pos >> 5;
  const u32 o = (u32)(pos & 31);
  const u64 v = ((u64)val << (64 - nbits)) >> o;  // left aligned in 64 bits, then shifted to the offset
  const u32 hi = (u32)(v >> 32), lo = (u32)v;
  if (hi) atomicOr(&out[w], bswap32(hi));
  if (lo) atomicOr(&out[w + 1], bswap32(lo));
}

// Sequential writer for one thread that owns a contiguous bit range: words strictly inside the
// range are stored, the first and last (shared) words are OR-ed.
struct BitAcc {
  u32* out; u64 word; unsigned long long acc; u32 nb; bool first;
  __device__ __forceinline__ void init(u32* o, u64 pos) { out = o; word = pos >> 5; nb = (u32)(pos & 31); acc = 0; first = true; }
  __device__ __forceinline__ void put(u32 nbits, u32 val) {
    acc = (acc << nbits) | val;
    nb += nbits;
    if (nb >= 32) {
      const u32 wv = (u32)(acc >> (nb - 32));
      if (first) { atomicOr(&out[word], bswap32(wv)); first = false; }
      else out[word] = bswap32(wv);
      word++;
      nb -= 32;
      acc &= (1ull << nb) - 1;
    }
  }
  __device__ __forceinline__ void flush() {
    if (nb) {
      const u32 wv = (u32)(acc << (32 - nb));
      if (wv) atomicOr(&out[word], bswap32(wv));
    }
  }
};

// ---- offsets ---------------------------------------------------------------------------------
// state[0] = bit cursor, state[1] = stream crc.  One warp, 32 blocks per step: the bit offsets are a scan; the CRC fold
// s' = rotl1(s) ^ crc[k] is linear, so after all nblk blocks s = rotl_nblk(s0) ^ XOR_k rotl_(nblk-1-k)(crc[k]).
__global__ void __launch_bounds__(32) k_offsets(const HuffBlk* __restrict__ hb, const u32* __restrict__ crc, u32 nblk, u64* state,
                                                u64* __restrict__ bitoff, u64 cap_bits, u32* flag) {
  const u32 lane = threadIdx.x;
  u64 cur = state[0];
  const u32 s0 = (u32)state[1];
  u32 fold = 0;
  for (u32 k0 = 0; k0 < nblk; k0 += 32) {
    const u32 k = k0 + lane;
    const u64 b = k < nblk ? hb[k].body_bits : 0ull;
    if (k < nblk) fold ^= __funnelshift_l(crc[k], crc[k], (nblk - 1 - k) & 31u);
    const u64 inc = warp_incl_add(b);
    if (k < nblk) bitoff[k] = cur + inc - b;
    cur += __shfl_sync(FULL_MASK, inc, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) fold ^= __shfl_xor_sync(FULL_MASK, fold, o);
  if (lane == 0) {
    state[0] = cur;
    state[1] = __funnelshift_l(s0, s0, nblk & 31u) ^ fold;
    if (cur + 96 + 64 > cap_bits) *flag = 1;
  }
}

// ---- header --------------------------------------------------------------------------------
#define PH_THREADS 256
__global__ void __launch_bounds__(PH_THREADS)
k_pack_header(const u8* __restrict__ selmtf, const HuffBlk* __restrict__ hb_arr, const u32* __restrict__ used, const u32* __restrict__ pidx,
              const u32* __restrict__ crc, const u64* __restrict__ bitoff, const u32* __restrict__ flag, u32* __restrict__ out,
              u32* __restrict__ code_start, u32* __restrict__ codes) {
  __shared__ u32 ws[PH_THREADS / 32 + 1];
  __shared__ u32 tab_off[HUFF_MAXGROUPS + 1];
  if (*flag) return;
  const u32 blk = blockIdx.x, tid = threadIdx.x;
  const HuffBlk* hb = hb_arr + blk;
  const u32 ng = hb->ngroups, nsel = hb->nsel, A = hb->alpha + 2;
  if (ng == 0) return;
  const u64 P0 = bitoff[blk];
  // canonical codes (lib/Bzip2.js:581-600): ascending (length, symbol); the code of a symbol is the
  // number of code points of its length taken by everything that sorts before it
  for (u32 i = tid; i < ng * A; i += PH_THREADS) {
    const u32 t = i / A, sy = i % A;
    const u32 l = hb->len[t][sy];
    u32 codev = 0;
    for (u32 j = 0; j < A; j++) {
      const u32 lj = hb->len[t][j];
      if (lj < l || (lj == l && j < sy)) codev += 1u << (l - lj);
    }
    codes[((size_t)blk * HUFF_MAXGROUPS + t) * (HUFF_MAXSYM + 2) + sy] = (l << 24) | codev;
  }
  // fixed part
  u32 mapbits = 0;
  for (u32 r = 0; r < 16; r++) {
    const u32 w = used[blk * 8 + (r >> 1)];
    if ((w >> ((r & 1) * 16)) & 0xffffu) mapbits += 16;
  }
  const u64 Psel = P0 + 48 + 32 + 1 + 24 + 16 + mapbits + 3 + 15;
  if (tid == 0) {
    u64 p = P0;
    gput(out, p, 24, 0x314159u); p += 24;      // WHOLEPI lib/Bzip2.js:49
    gput(out, p, 24, 0x265359u); p += 24;
    gput(out, p, 32, crc[blk]); p += 32;
    gput(out, p, 1, 0); p += 1;                // not randomised
    gput(out, p, 24, pidx[blk]); p += 24;
    u32 compact = 0;
    for (u32 r = 0; r < 16; r++) {
      const u32 w = used[blk * 8 + (r >> 1)];
      if ((w >> ((r & 1) * 16)) & 0xffffu) compact |= 1u << (15 - r);
    }
    gput(out, p, 16, compact); p += 16;
    for (u32 r = 0; r < 16; r++) {
      const u32 w = (used[blk * 8 + (r >> 1)] >> ((r & 1) * 16)) & 0xffffu;
      if (w) {
        // bit j of the range (byte r*16+j) is written MSB first: reverse the 16 bits
        const u32 rev = __brev(w) >> 16;
        gput(out, p, 16, rev); p += 16;
      }
    }
    gput(out, p, 3, ng); p += 3;
    gput(out, p, 15, nsel); p += 15;
  }
  // selectors: j ones then a zero each
  const u8* sm = selmtf + (size_t)blk * SEL_STRIDE;
  const u32 per = (nsel + PH_THREADS - 1) / PH_THREADS;
  const u32 ga = min(nsel, tid * per), gb = min(nsel, ga + per);
  u32 mybits = 0;
  for (u32 g = ga; g < gb; g++) mybits += (u32)sm[g] + 1;
  u32 total;
  const u32 ex = block_excl_add<PH_THREADS, u32>(mybits, ws, &total);
  if (gb > ga) {
    BitAcc ba;
    ba.init(out, Psel + ex);
    for (u32 g = ga; g < gb; g++) {
      const u32 j = sm[g];
      ba.put(j + 1, ((1u << j) - 1) << 1);
    }
    ba.flush();
  }
  // tables
  const u64 Ptab = Psel + total;
  if (tid == 0) {
    u32 o = 0;
    for (u32 t = 0; t < ng; t++) {
      tab_off[t] = o;
      u32 bits = 5, cur = hb->len[t][0];
      for (u32 i = 0; i < A; i++) {
        const u32 l = hb->len[t][i];
        bits += 2 * (l > cur ? l - cur : cur - l) + 1;
        cur = l;
      }
      o += bits;
    }
    tab_off[ng] = o;
    code_start[blk] = (u32)(Ptab + o - P0);
  }
  __syncthreads();
  if (tid < ng) {
    BitAcc ba;
    ba.init(out, Ptab + tab_off[tid]);
    u32 cur = hb->len[tid][0];
    ba.put(5, cur);
    for (u32 i = 0; i < A; i++) {
      const u32 l = hb->len[tid][i];
      const u32 v = cur < l ? 2u : 3u;
      u32 d = cur < l ? l - cur : cur - l;
      while (d--) ba.put(2, v);
      ba.put(1, 0);
      cur = l;
    }
    ba.flush();
  }
}

// ---- codes ---------------------------------------------------------------------------------
// Accumulator of one thread's codes in the zeroed staging tile.  Every word goes in by a shared-memory atomicOr (the
// first and last words of a thread's range are shared with its neighbours), so a put has no branch: the warp's
// threads complete words at different symbols, and a divergent store path would run on nearly every symbol.  Bits
// above the 32 + nb that are still pending are never read, so the accumulator is not masked.
struct StageAcc {
  u32* stage; u32 word, nb; unsigned long long acc;
  __device__ __forceinline__ void init(u32* st, u32 pos) { stage = st; word = pos >> 5; nb = pos & 31; acc = 0; }
  __device__ __forceinline__ void put(u32 cv) {  // cv = len << 24 | code
    const u32 len = cv >> 24;
    acc = (acc << len) | (cv & 0xffffffu);
    nb += len;
    if (nb >= 32) {
      nb -= 32;
      atomicOr(&stage[word++], bswap32((u32)(acc >> nb)));
    }
  }
  __device__ __forceinline__ void flush() {
    if (nb) atomicOr(&stage[word], bswap32((u32)acc << (32 - nb)));
  }
};

// One thread per group, 128 groups per CTA.  The staging tile holds the worst case (every code 20 bits), so a CTA
// needs ~29 KB of shared memory and 7 fit on an SM.
#define PC_THREADS 128
#define PC_GROUPS PC_THREADS
#define PC_SYM_BYTES (PC_GROUPS * HUFF_GROUP)
#define PC_STAGE_WORDS ((31 + PC_GROUPS * HUFF_GROUP * 20 + 31) / 32)

struct PackSmem {
  u8 sym[PC_SYM_BYTES + 16];                  // the tile's symbols, low bytes (+ slack for a group's last word)
  u32 stage[PC_STAGE_WORDS];
  u32 code[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];  // len << 24 | code
};

__global__ void __launch_bounds__(PC_THREADS)
k_pack_codes(const u8* __restrict__ sym_lo, const unsigned long long* __restrict__ sym_hi, const u32* __restrict__ any_hi,
             const u8* __restrict__ sel, const HuffBlk* __restrict__ hb_arr, const u32* __restrict__ goff, const u64* __restrict__ bitoff,
             const u32* __restrict__ code_start, const u32* __restrict__ codes, const u32* __restrict__ flag, u32 tps, u32* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PackSmem& s = *reinterpret_cast<PackSmem*>(smem_raw);
  const u32 tid = threadIdx.x;
  const u32 blk = blockIdx.x / tps, lt = blockIdx.x % tps;
  const HuffBlk* hb = hb_arr + blk;
  const u32 nsel = hb->nsel, m = hb->m, ng = hb->ngroups, A = hb->alpha + 2;
  const u32 g0 = lt * PC_GROUPS;
  if (*flag || g0 >= nsel) return;
  const u32 g = g0 + tid, gend = min(nsel, g0 + PC_GROUPS);
  const u32* go = goff + (size_t)blk * SEL_STRIDE;
  const u32 o0 = go[g0], total = go[gend] - o0;
  const u32 my = g < nsel ? go[g] - o0 : 0u;
  const u32 tsel = g < nsel ? sel[(size_t)blk * SEL_STRIDE + g] : 0u;
  const unsigned long long hm = (g < nsel && any_hi[blk]) ? sym_hi[(size_t)blk * SEL_STRIDE + g] : 0ull;
  const u64 P = bitoff[blk] + code_start[blk] + o0;  // absolute bit of this tile's first code
  const u32 phase = (u32)(P & 31);
  const u32 nw = (phase + total + 31) >> 5;
  for (u32 i = tid; i < ng * A; i += PC_THREADS) {
    const u32 t = i / A, sy = i % A;
    s.code[t][sy] = codes[((size_t)blk * HUFF_MAXGROUPS + t) * (HUFF_MAXSYM + 2) + sy];
  }
  // the tile's symbols: 16-byte loads (the tile starts at byte 6400 lt of the slot); bytes past m are never coded
  const uint4* src = reinterpret_cast<const uint4*>(sym_lo + ((size_t)blk << SEG_SHIFT) + (size_t)g0 * HUFF_GROUP);
  for (u32 i = tid; i < PC_SYM_BYTES / 16; i += PC_THREADS) reinterpret_cast<uint4*>(s.sym)[i] = src[i];
  for (u32 i = tid; i < nw; i += PC_THREADS) s.stage[i] = 0;
  __syncthreads();
  if (g < nsel) {
    const u32* cw = s.code[tsel];
    StageAcc ba;
    ba.init(s.stage, phase + my);
    const u32 cnt = min(50u, m - 50u * g), base = tid * HUFF_GROUP;
    if (cnt == HUFF_GROUP && hm == 0) {  // all but a few groups: 13 aligned words, realigned by a funnel shift
      const u32* wp = reinterpret_cast<const u32*>(s.sym + (base & ~3u));
      const u32 sh = (base & 2u) * 8u;
      u32 nxt = wp[0];
#pragma unroll
      for (u32 k = 0; k < 13; k++) {
        const u32 cur = nxt;
        nxt = wp[k + 1];
        const u32 w = __funnelshift_r(cur, nxt, sh);
#pragma unroll
        for (u32 j = 0; j < (k < 12 ? 4u : 2u); j++) ba.put(cw[(w >> (8 * j)) & 0xffu]);
      }
    } else {
      for (u32 j = 0; j < cnt; j++) ba.put(cw[(u32)s.sym[base + j] | (u32)((hm >> j) & 1u) << 8]);
    }
    ba.flush();
  }
  __syncthreads();
  // stage words are already byte-swapped; copy out
  u32* dst = out + (P >> 5);
  for (u32 i = tid; i < nw; i += PC_THREADS) {
    const u32 v = s.stage[i];
    if (i == 0 || i == nw - 1) { if (v) atomicOr(&dst[i], v); }
    else dst[i] = v;
  }
}

void pack_batch(Ctx& c, const NarrowSyms& sym, const u8* d_sel, const u8* d_selmtf, const HuffBlk* d_hb, const u32* d_goff, const u32* d_used,
                const u32* d_pidx, const u32* d_crc, const u64* d_bitoff, const u32* d_flag, u32 nblk, u32 max_m, u32* d_out_words) {
  static bool attr = false;
  if (!attr) {
    CUDA_CHECK(cudaFuncSetAttribute(k_pack_codes, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PackSmem)));
    attr = true;
  }
  DBuf<u32> code_start(c, nblk), codes(c, (size_t)nblk * HUFF_MAXGROUPS * (HUFF_MAXSYM + 2));
  k_pack_header<<<nblk, PH_THREADS, 0, c.stream>>>(d_selmtf, d_hb, d_used, d_pidx, d_crc, d_bitoff, d_flag, d_out_words, code_start, codes);
  KLAUNCH(c); KCHECK();
  const u32 max_sel = (max_m + HUFF_GROUP - 1) / HUFF_GROUP;
  const u32 tps = (max_sel + PC_GROUPS - 1) / PC_GROUPS;
  k_pack_codes<<<nblk * tps, PC_THREADS, sizeof(PackSmem), c.stream>>>(sym.lo, sym.hi, sym.any_hi, d_sel, d_hb, d_goff, d_bitoff, code_start, codes,
                                                                      d_flag, tps, d_out_words);
  KLAUNCH(c); KCHECK();
}

// ---- file header / trailer ---------------------------------------------------------------
__global__ void k_file_header(u32* out, int level) {
  if (threadIdx.x || blockIdx.x) return;
  gput(out, 0, 8, 'B'); gput(out, 8, 8, 'Z'); gput(out, 16, 8, 'h'); gput(out, 24, 8, (u32)('0' + level));  // lib/Bzip2.js:903-906
}
__global__ void k_file_trailer(u32* out, const u64* state) {
  if (threadIdx.x || blockIdx.x) return;
  u64 p = state[0];
  gput(out, p, 24, 0x177245u); p += 24;  // SQRTPI lib/Bzip2.js:50
  gput(out, p, 24, 0x385090u); p += 24;
  gput(out, p, 32, (u32)state[1]);
}

__global__ void k_rebase(u32* out, u64 word_index, u64* state, u32 bits_in_word) {
  if (threadIdx.x || blockIdx.x) return;
  out[0] = word_index ? out[word_index] : out[0];
  state[0] = bits_in_word;
}

// One output stream being written: the running bit position lives on the device (state[0]); blocks of one or more
// RLE1 plans are appended batch by batch.  Shared by the device-resident entry points and the pipelined host path.
// whole_file: file header + blocks + trailer; otherwise the blocks alone, from bit `bit_phase` of d_out.
struct EncSession {
  Ctx& c;
  int level; u8* d_out; size_t cap_words; bool whole_file; int bit_phase;
  DBuf<u64> state; DBuf<u32> flag;
  std::vector<u32> all_crc;
  std::vector<b2_block_trace> tr;
  u32 cap_blocks = 0;
  DBuf<u8> T, U, dsel, dselmtf, sym_lo;
  DBuf<unsigned long long> sym_hi;
  DBuf<u32> dn, dcrc, dpidx, dm, dfreq, dused, dhist, sym_any_hi, dgoff;
  DBuf<HuffBlk> dhb;
  DBuf<u64> dbitoff;
  std::vector<u32> hn, hm, hp;
  std::vector<HuffBlk> hhb;
  std::vector<u64> hoff;
  std::function<void(u64)> on_batch;  // called after every batch with the bit position reached inside the window (host synchronised)
  u64 bit_base = 0;    // bits of the stream in front of d_out[0] (streaming: the output buffer is a window that is drained and rebased)
  u64 last_bit_end = 32;  // bit position (inside the window) behind the last block packed

  EncSession(Ctx& c_, int level_, u8* d_out_, size_t out_cap, bool whole_file_, int bit_phase_)
      : c(c_), level(level_), d_out(d_out_), cap_words(out_cap / 4), whole_file(whole_file_), bit_phase(bit_phase_) {
    if (((size_t)d_out) & 3) throw B2Error{B2_ERR_BAD_ARG, "output buffer must be 4-byte aligned"};
    if (cap_words < 8) throw B2Error{B2_ERR_BAD_ARG, "output buffer too small"};
    CUDA_CHECK(cudaMemsetAsync(d_out, 0, cap_words * 4, c.stream));
    state.alloc(c, 4);
    flag.alloc(c, 1);
    u64 h_state[4] = {whole_file ? 32ull : (u64)bit_phase, 0, 0, 0};
    c.to_device(state, h_state, sizeof h_state);
    CUDA_CHECK(cudaMemsetAsync(flag, 0, 4, c.stream));
    if (whole_file) {  // the header goes first: finished words are handed out while later batches are still encoding
      k_file_header<<<1, 32, 0, c.stream>>>(reinterpret_cast<u32*>(d_out), level);
      KLAUNCH(c); KCHECK();
    }
    c.sync();
  }
  void reserve(u32 nb) {
    if (nb <= cap_blocks) return;
    cap_blocks = nb;
    T.alloc(c, (size_t)nb << SEG_SHIFT); U.alloc(c, (size_t)nb << SEG_SHIFT); sym_lo.alloc(c, (size_t)nb << SEG_SHIFT);
    sym_hi.alloc(c, (size_t)nb * SEL_STRIDE); sym_any_hi.alloc(c, nb); dgoff.alloc(c, (size_t)nb * SEL_STRIDE);
    CUDA_CHECK(cudaMemsetAsync(sym_hi, 0, (size_t)nb * SEL_STRIDE * 8, c.stream));
    CUDA_CHECK(cudaMemsetAsync(sym_any_hi, 0, (size_t)nb * 4, c.stream));
    dn.alloc(c, nb); dcrc.alloc(c, nb); dpidx.alloc(c, nb); dm.alloc(c, nb);
    dfreq.alloc(c, (size_t)nb * HUFF_MAXSYM); dused.alloc(c, (size_t)nb * 8); dhist.alloc(c, (size_t)nb * 256);
    dsel.alloc(c, (size_t)nb * SEL_STRIDE); dselmtf.alloc(c, (size_t)nb * SEL_STRIDE);
    dhb.alloc(c, nb); dbitoff.alloc(c, nb);
    hn.resize(nb); hm.resize(nb); hp.resize(nb); hhb.resize(nb); hoff.resize(nb);
  }
  // append blocks [first, first+count) of `plan` (made over d_in[0,n)); raw_base = offset of d_in in the whole input
  void encode(const u8* d_in, size_t n, const Rle1Plan& plan, size_t first, size_t count, u64 raw_base) {
    if (!count) return;
    // balanced batches: ceil(count / batches) blocks each, so that no tiny tail batch starves the per-block kernels
    const u32 nbatches = (u32)((count + c.bwt_batch - 1) / c.bwt_batch);
    const u32 B = (u32)((count + nbatches - 1) / nbatches);
    reserve((u32)std::min<size_t>(B, count));
    // all stage temporaries of one batch come to ~40 bytes per slot; size the pool for the batch class once
    const u32 half = c.bwt_batch / 2, quarter = c.bwt_batch / 4;
    if (B > quarter) c.prewarm((size_t)(B > half ? std::max<u32>(B, c.bwt_batch) : half) * 40 << SEG_SHIFT);
    const NarrowSyms sym{sym_lo, sym_hi, sym_any_hi};
    const size_t done0 = all_crc.size();
    all_crc.resize(done0 + count);
    tr.resize(done0 + count);
    for (size_t k0 = 0; k0 < count; k0 += B) {
      const u32 nb = (u32)std::min<size_t>(B, count - k0);
      u32 nmax = 0;
      for (u32 b = 0; b < nb; b++) { hn[b] = plan.h_blocks[first + k0 + b].n; nmax = std::max(nmax, hn[b]); }
      {
        StageScope s(c, ST_RLE1);
        rle1_materialize(c, d_in, n, plan, first + k0, nb, T, dn, dcrc);
      }
      {
        StageScope s(c, ST_BWT);
        CUDA_CHECK(cudaMemsetAsync(dpidx, 0, nb * 4, c.stream));
        bwt_forward_batch(c, T, U, dn, hn.data(), nb, dpidx, false, nullptr, dhist);
      }
      {
        StageScope s(c, ST_MTF);
        mtf_rle2_batch(c, T, U, dn, hn.data(), nb, sym, dm, dfreq, dused, dhist);
      }
      {
        StageScope s(c, ST_HUFF);
        huffman_batch(c, sym, dm, dfreq, dused, nb, dsel, dselmtf, dhb, dgoff);
      }
      {
        StageScope s(c, ST_PACK);
        k_offsets<<<1, 32, 0, c.stream>>>(dhb, dcrc, nb, state, dbitoff, (u64)cap_words * 32, flag);
        KLAUNCH(c); KCHECK();
        pack_batch(c, sym, dsel, dselmtf, dhb, dgoff, dused, dpidx, dcrc, dbitoff, flag, nb, nmax + 1, reinterpret_cast<u32*>(d_out));
      }
      // per-block bookkeeping for the host (trace + CRCs)
      c.to_host(hm.data(), dm, nb * 4);
      c.to_host(hp.data(), dpidx, nb * 4);
      c.to_host(hhb.data(), dhb, nb * sizeof(HuffBlk));
      c.to_host(hoff.data(), dbitoff, nb * 8);
      c.to_host(all_crc.data() + done0 + k0, dcrc, nb * 4);
      c.sync();
      for (u32 b = 0; b < nb; b++) {
        b2_block_trace& t = tr[done0 + k0 + b];
        const BlkInfo& bi = plan.h_blocks[first + k0 + b];
        t.n = (int32_t)bi.n; t.pidx = (int32_t)hp[b]; t.m = (int32_t)hm[b]; t.alpha = (int32_t)hhb[b].alpha;
        t.ngroups = (int32_t)hhb[b].ngroups; t.nsel = (int32_t)hhb[b].nsel; t.crc = all_crc[done0 + k0 + b]; t.pad = 0;
        t.raw_start = raw_base + bi.s; t.raw_len = bi.e - bi.s; t.bit_start = bit_base + hoff[b]; t.bit_len = hhb[b].body_bits;
      }
      c.stats.blocks += nb;
      last_bit_end = hoff[nb - 1] + hhb[nb - 1].body_bits;
      if (on_batch) on_batch(last_bit_end);
    }
  }
  // Streaming: everything in front of the word that is still being filled has been handed out; that word moves to the
  // start of the window, the rest of the window is cleared and the device cursor restarts behind the carried bits.
  // `used_bytes` = how much of the window the batches since the last rebase may have touched.
  void rebase(size_t used_bytes) {
    const u64 wi = last_bit_end >> 5;
    k_rebase<<<1, 32, 0, c.stream>>>(reinterpret_cast<u32*>(d_out), wi, state, (u32)(last_bit_end & 31));
    KLAUNCH(c); KCHECK();
    const size_t clear = std::min(cap_words * 4, (used_bytes + 7) & ~(size_t)3);
    if (clear > 4) CUDA_CHECK(cudaMemsetAsync(d_out + 4, 0, clear - 4, c.stream));
    bit_base += wi * 32;
    last_bit_end &= 31;
    c.sync();
  }
  // file trailer (whole files), final size; returns the bit position reached
  u64 finish(size_t* out_n) {
    u32 h_flag = 0;
    u64 h_state[4];
    if (whole_file) {
      k_file_trailer<<<1, 32, 0, c.stream>>>(reinterpret_cast<u32*>(d_out), state);
      KLAUNCH(c); KCHECK();
    }
    c.to_host(h_state, state, sizeof h_state);
    c.to_host(&h_flag, flag, 4);
    c.sync();
    if (h_flag) throw B2Error{B2_ERR_BAD_ARG, "output buffer too small for the compressed stream"};
    // whole files: trailer 48 + 32 bits, zero padded (lib/BitStream.js:68-73)
    *out_n = whole_file ? (size_t)((bit_base + h_state[0] + 80 + 7) / 8) : (size_t)((bit_base + h_state[0] + 7) / 8);
    c.trace = tr;
    return bit_base + h_state[0];
  }
};

// ---- device-resident entry points ------------------------------------------------------------------------------
// The plan of b2_bzip2_plan(_flavor), _plan_spec or _plan_share(_flavor), kept for the next b2_bzip2_encode_range_dev
// (_flavor).  That call takes it if (buffer, length, level, flavor) match; the cache is empty afterwards either way.
// compress_dev drops it too.  The two flavors cut different blocks, so a plan never serves the other flavor.
struct PlanCache {
  std::optional<Rle1Plan> plan;
  const u8* ptr = nullptr; size_t n = 0; int level = 0, flavor = B2_BZ2_COMPRESSJS;
  std::optional<Rle1Plan> take(const u8* p, size_t n_, int level_, int flavor_) {
    std::optional<Rle1Plan> r;
    if (plan && p == ptr && n_ == n && level_ == level && flavor_ == flavor) r = std::move(plan);
    plan.reset();
    return r;
  }
  void put(Rle1Plan&& p, const u8* p_, size_t n_, int level_, int flavor_) {
    plan = std::move(p); ptr = p_; n = n_; level = level_; flavor = flavor_;
  }
};
static PlanCache g_plan;
void bzip2_release_plan() { g_plan.plan.reset(); rle1_release_share_probe(); }

void bzip2_compress_dev(Ctx& c, const u8* d_in, size_t n, int level, u8* d_out, size_t out_cap, size_t* out_n) {
  g_plan.plan.reset();
  rle1_release_share_probe();
  Rle1Plan plan;
  rle1_plan(c, d_in, n, level, plan);
  c.trace.clear();
  EncSession S(c, level, d_out, out_cap, true, 0);
  S.encode(d_in, n, plan, 0, plan.nblocks, 0);
  S.finish(out_n);
}

size_t bzip2_plan(Ctx& c, const u8* d_in, size_t n, int level) {
  g_plan.plan.reset();
  Rle1Plan plan;
  rle1_plan(c, d_in, n, level, plan);
  c.trace.clear();
  const size_t nb = plan.nblocks;
  g_plan.put(std::move(plan), d_in, n, level, c.bz_flavor);
  return nb;
}

// info = {raw start, raw end of the blocks cut, first, planned, cut, last}
static void range_info(const Rle1Plan& plan, size_t first, size_t count, u64 last, u64* info) {
  info[0] = plan.nblocks ? plan.h_blocks.front().s : 0;
  info[1] = plan.nblocks ? plan.h_blocks.back().e : 0;
  info[2] = first; info[3] = count; info[4] = plan.nblocks; info[5] = last;
}

// Speculative range plan (multi-GPU, whole input on every rank): the blocks of rank `rank` of `world` among the
// total guess, cut from the speculative boundary.  info[5] = the total guess.
void bzip2_plan_spec(Ctx& c, const u8* d_in, size_t n, int level, int rank, int world, u64* info) {
  g_plan.plan.reset();
  Rle1Plan plan;
  rle1_scan_tiles(c, d_in, n, plan);
  const size_t total = plan.total_guess(level);
  const size_t first = (size_t)rank * total / world, count = (size_t)(rank + 1) * total / world - first;
  rle1_cut_range(c, d_in, n, level, plan, first, count);
  c.trace.clear();
  range_info(plan, first, count, total, info);
  g_plan.put(std::move(plan), d_in, n, level, B2_BZ2_COMPRESSJS);
}

// Blocks [first, first+count) without file header and trailer, from bit `bit_phase` of d_out.
void bzip2_encode_range(Ctx& c, const u8* d_in, size_t n, int level, size_t first, size_t count, int bit_phase, u8* d_out, size_t out_cap,
                        u64* out_bits, u32* block_crcs) {
  std::optional<Rle1Plan> plan = g_plan.take(d_in, n, level, c.bz_flavor);
  if (!plan) rle1_plan(c, d_in, n, level, plan.emplace());
  c.trace.clear();
  const size_t nb_all = plan->first_index + plan->nblocks;  // exact plans: first_index == 0
  first = std::min(first, nb_all);
  count = std::min(count, nb_all - first);
  if (first < plan->first_index) throw B2Error{B2_ERR_BAD_ARG, "block range is not covered by the cached range plan"};
  EncSession S(c, level, d_out, out_cap, false, bit_phase);
  S.encode(d_in, n, *plan, first - plan->first_index, count, 0);  // h_blocks[k] is global block first_index + k
  size_t bytes = 0;
  const u64 bits = S.finish(&bytes);
  if (out_bits) *out_bits = bits - (u64)bit_phase;
  if (block_crcs) std::copy(S.all_crc.begin(), S.all_crc.end(), block_crcs);
}

// ---- multi-GPU: every rank holds a share of the input (plus some bytes of the next share) ---------------------
// summary of a share for the planner of the other ranks: out = {aggregate run state, length of the leading run,
// RLE1 bytes of the share when no run enters it, share length}
void bzip2_share_summary(Ctx& c, const u8* d_in, size_t n, u64* out) {
  out[0] = out[1] = out[2] = 0; out[3] = n;
  Rle1Plan plan;
  rle1_scan_tiles(c, d_in, n, plan, 0, 0, out);
  out[2] = plan.w_total;
}
// Cut blocks [first, first+count) of the whole input inside this rank's buffer (share + halo): st0 / W0 = run state
// and RLE1 output in front of the buffer (from the summaries of the ranks before).  The blocks are located by the
// speculated boundary W = first * blockSize, exact unless a run-phase slip happened earlier in the file: the caller
// checks that the pieces of all ranks chain up.  info = {raw start, raw end (buffer offsets), first, planned, cut,
// W at the end of the buffer}.  The plan is kept for the b2_bzip2_encode_range_dev call that follows.
void bzip2_plan_share(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t first, size_t count, u64* info) {
  g_plan.plan.reset();
  Rle1Plan plan;
  rle1_scan_tiles(c, d_buf, n, plan, st0, W0);
  rle1_cut_range(c, d_buf, n, level, plan, first, count);
  range_info(plan, first, count, plan.w_total, info);
  g_plan.put(std::move(plan), d_buf, n, level, B2_BZ2_COMPRESSJS);
}
// libbz2 flavor: table row d = the cut of the share when its first block has drift d (see k_cut_table).
void bzip2_share_cut_table(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t share_len, u64 dmax, u32* table) {
  rle1_share_cut_table(c, d_buf, n, level, st0, W0, share_len, dmax, table);
}
// The share plan of either flavor.  compressjs: bzip2_plan_share (drift unused).  libbz2: the blocks [first, first+count)
// from the entry W = first * blockSize + drift that the host chained from the tables.  info as bzip2_plan_share's.
void bzip2_plan_share_flavor(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t first, size_t count, u64 drift, u64* info) {
  if (c.bz_flavor != B2_BZ2_LIBBZ2) { bzip2_plan_share(c, d_buf, n, level, st0, W0, first, count, info); return; }
  g_plan.plan.reset();
  Rle1Plan plan;
  rle1_cut_share_libbz2(c, d_buf, n, level, st0, W0, first, drift, count, plan);
  range_info(plan, first, count, plan.w_total, info);
  g_plan.put(std::move(plan), d_buf, n, level, B2_BZ2_LIBBZ2);
}

// Bzip2.compressFile from a host source into a host sink: b2_bzip2_compress (the caller's buffer, complete from the
// start, into the result buffer) and b2_bzip2_compress_stream (read and write callbacks).  With a pinned input the
// upload is cut into chunks on a copy stream; block boundaries only depend on the bytes before them (lib/Bzip2.js:636-667
// consumes its input strictly forward), so every block but the last of a plan over the prefix that has arrived is final
// and is encoded while the rest is still in flight.  Finished words of the output go back on a second copy stream after
// every batch and are handed to `out` one batch behind, so a write callback never waits for the copy just queued.
// `in` keeps the bytes from the window's start on and is read until it holds more than a window or the input ends, so a
// window is the last one exactly when the input ends in it: however the input arrives, the windows, blocks and stream
// are the same.
void bzip2_compress_host(Ctx& c, StreamIn& in, int level, u8* d_in, size_t win, u8* d_out, size_t out_cap, StreamOut& out,
                         size_t* out_n, bool pinned_in) {
  // d_in holds `win` bytes, d_out `out_cap` bytes (>= b2_bzip2_bound(win)).  An input of at most win bytes is one window
  // (the usual case).  A longer one STREAMS through the device in windows -- every window is uploaded, planned and
  // encoded like a small file whose last block is kept back (it may go on in the next window), the next window starts at
  // the first raw byte that has not been consumed, and the output window is drained and rebased in between: device
  // memory is bounded by the window, not by the file (lib/Bzip2.js:879-929 reads its input strictly forward, too).
  size_t CH = (size_t)64 << 20;
  if (const char* e = getenv("B2_H2D_CHUNK")) {  // test hook: small chunks exercise the prefix planning on small inputs
    const long long v = atoll(e);
    if (v >= 4096) CH = (size_t)v;
  }
  const bool trace_host = getenv("B2_TRACE_HOST") != nullptr;  // debug: host-side timeline on stderr
  const auto t_start = std::chrono::steady_clock::now();
  auto mark = [&](const char* what, size_t v) {
    if (trace_host) fprintf(stderr, "[b2 host] %8.2f ms  %s %zu\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count(), what, v);
  };
  const size_t max_ch = (win + CH - 1) / CH + 1;
  std::vector<cudaEvent_t> ev(max_ch);
  struct Cleanup {
    std::vector<cudaEvent_t>& ev; Ctx& c;
    ~Cleanup() {
      cudaStreamSynchronize(c.h2d_stream); cudaStreamSynchronize(c.d2h_stream);
      for (auto e : ev) if (e) cudaEventDestroy(e);
    }
  } cleanup{ev, c};
  for (auto& e : ev) { e = nullptr; CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); }
  c.trace.clear();
  EncSession S(c, level, d_out, out_cap, true, 0);
  mark("session ready", 0);
  u8* h_out = nullptr;     // where the current output window's byte 0 goes on the host
  size_t h_room = 0;       // bytes from h_out on that `out` has room for
  size_t copied = 0;       // bytes of the current output window already on their way to the host
  size_t out_base = 0;     // offset in the output of the window's byte 0
  size_t sent = 0;         // bytes of the current output window handed to `out`
  bool d2h_started = false, h2d_started = false;
  // hand over what the copies queued so far bring to the host
  auto drain = [&]() {
    out.put(h_out + sent, copied - sent);
    sent = copied;
  };
  S.on_batch = [&](u64 bit_end) {
    const size_t ready = (size_t)(bit_end / 32) * 4;  // whole words below the one still being filled
    if (ready > copied) {
      drain();  // the previous batch's words: their copy has had a batch's time to land
      if (ready > h_room) throw B2Error{B2_ERR_BAD_ARG, "output buffer too small for the compressed stream"};
      if (!d2h_started) { c.copy_begin(c.d2h_stream, 1); d2h_started = true; }
      CUDA_CHECK(cudaMemcpyAsync(h_out + copied, d_out + copied, ready - copied, cudaMemcpyDeviceToHost, c.d2h_stream));
      copied = ready;
    }
  };
  size_t file_pos = 0;  // raw bytes consumed by finished blocks
  for (bool first_window = true;; first_window = false) {
    // the window and one byte more when there is one: a window that holds the rest of the input is the last one
    in.drop(file_pos);
    const size_t end = in.fill(file_pos + win + 1);
    const size_t wlen = std::min(win, end - file_pos);
    const bool last_window = in.eof && file_pos + wlen == end;
    const u8* src = in.at(file_pos);
    if (!first_window) {
      // the previous window's output is on its way: wait for it, then reuse both windows
      CUDA_CHECK(cudaStreamSynchronize(c.d2h_stream));
      drain();
      S.rebase(copied + 8);
      out_base += copied;
      copied = sent = 0;
    }
    h_out = out.next();
    h_room = out.cap - (size_t)(h_out - out.buf);
    const size_t nch = (pinned_in && wlen > CH) ? (wlen + CH - 1) / CH : (wlen ? 1 : 0);
    if (!h2d_started) { c.copy_begin(c.h2d_stream, 0); h2d_started = true; }
    for (size_t i = 0; i < nch; i++) {
      const size_t o = nch == 1 ? 0 : i * CH, len = nch == 1 ? wlen : std::min(CH, wlen - o);
      CUDA_CHECK(cudaMemcpyAsync(d_in + o, src + o, len, cudaMemcpyHostToDevice, c.h2d_stream));
      CUDA_CHECK(cudaEventRecord(ev[i], c.h2d_stream));
    }
    c.copy_end(c.h2d_stream, 0);
    mark("uploads queued, chunks", nch);
    size_t resume = 0, have = 0;  // raw bytes of the window planned so far / chunks known to have arrived
    bool progressed = false;
    while (resume < wlen) {
      // block on the next chunk we need, then take every further chunk that has landed meanwhile
      if (have < nch) { CUDA_CHECK(cudaEventSynchronize(ev[have])); have++; }
      while (have < nch && cudaEventQuery(ev[have]) == cudaSuccess) have++;
      const size_t avail = have == nch ? wlen : have * CH;
      const bool last = avail == wlen;
      mark("chunks arrived", have);
      Rle1Plan plan;
      rle1_plan(c, d_in + resume, avail - resume, level, plan);
      // only the very end of the FILE closes a short block; the last block of any other prefix may still grow (libbz2
      // flavor: its closing piece may go on).  Every other block ends before the prefix does, and the next prefix starts
      // on a block start, where both flavors start a fresh run state.
      const size_t nfinal = (last && last_window) ? plan.nblocks : (plan.nblocks ? plan.nblocks - 1 : 0);
      mark("planned, final blocks", nfinal);
      if (!nfinal) {
        if (last) break;  // the rest of this window is less than one block: it opens the next window
        continue;         // the prefix holds less than one full block: wait for more
      }
      S.encode(d_in + resume, avail - resume, plan, 0, nfinal, file_pos + resume);
      mark("encoded", nfinal);
      resume += plan.h_blocks[nfinal - 1].e;
      progressed = true;
      if (last && !last_window) break;
    }
    if (!last_window && !progressed) throw B2Error{B2_ERR_BAD_ARG, "streaming window too small: it does not hold one whole block (raise B2_STREAM_WINDOW)"};
    file_pos += resume;
    if (last_window) break;
    CUDA_CHECK(cudaStreamSynchronize(c.h2d_stream));  // the next window overwrites d_in
  }
  size_t total = 0;
  S.finish(&total);
  *out_n = total;
  const size_t tail = *out_n - out_base;  // bytes of the last window, trailer included
  if (tail > h_room) throw B2Error{B2_ERR_BAD_ARG, "output buffer too small for the compressed stream"};
  if (!d2h_started) c.copy_begin(c.d2h_stream, 1);
  CUDA_CHECK(cudaMemcpyAsync(h_out + copied, d_out + copied, tail - copied, cudaMemcpyDeviceToHost, c.d2h_stream));
  c.copy_end(c.d2h_stream, 1);
  mark("finished, bytes left to download", tail - copied);
  copied = tail;
  CUDA_CHECK(cudaStreamSynchronize(c.d2h_stream));
  drain();
  mark("download done", *out_n);
}

// ---- fragment shift for the multi-GPU gather -------------------------------------------------
// dst holds src's first nbits starting at bit `phase` (MSB first); bits outside the fragment are 0.
__global__ void k_bitshift(const u32* __restrict__ src, u64 nbits, u32 phase, u32* __restrict__ dst, u64 nwords_out) {
  const u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nwords_out) return;
  const u64 src_words = (nbits + 31) >> 5;
  const u32 cur = w < src_words ? bswap32(src[w]) : 0u;
  const u32 prv = (w > 0 && w - 1 < src_words) ? bswap32(src[w - 1]) : 0u;
  u32 v = phase ? ((prv << (32 - phase)) | (cur >> phase)) : cur;
  // clear everything behind bit (phase + nbits)
  const u64 endbit = (u64)phase + nbits;
  const u64 wstart = w << 5;
  if (endbit <= wstart) v = 0;
  else if (endbit < wstart + 32) v &= ~(0xffffffffu >> (u32)(endbit - wstart));
  dst[w] = bswap32(v);
}
void bitshift_device(Ctx& c, const void* src, u64 nbits, int phase, void* dst) {
  const u64 nwords = ((u64)phase + nbits + 31) >> 5;
  if (nwords == 0) return;
  k_bitshift<<<(unsigned)((nwords + 255) / 256), 256, 0, c.stream>>>((const u32*)src, nbits, (u32)phase, (u32*)dst, nwords);
  KLAUNCH(c); KCHECK();
  c.sync();
}
