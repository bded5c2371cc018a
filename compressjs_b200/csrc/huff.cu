// huff.cu -- per-block Huffman table search and code-length assignment on the GPU.
//
// Reference: lib/Bzip2.js:826-843 (table count rule, two seed tables), :671-684
// (assignSelectors), :685-733 (optimizeHuffmanGroups: split the most used table at the median
// group cost -- STABLE sort, see SURVEY.md section 7), :551-579 (StaticHuffman ctor) and
// lib/HuffmanAllocator.js (huffalloc.cuh).
//
// One CTA owns one bzip2 block for the whole search (the refinement rounds are sequential
// inside a block); hundreds of blocks are in flight, two CTAs per SM, so the serial phases of one
// block (table builds, scans) hide behind the symbol passes of others.  Inside the CTA:
//   * the search makes 9 passes over the block's symbols (4 rounds of assign + recount, one final
//     assign), and a batch's symbols are far larger than L2, so every pass streams from HBM.  The
//     zero-run coder writes the symbols in one byte each plus a 50-bit mask per group of the symbols
//     >= 256 (NarrowSyms, enc.h); the passes stream them (1 byte per symbol, + 8 bytes per group in
//     the rare blocks that have a symbol >= 256), staged through shared memory a tile of 256 groups
//     at a time.  Counting the symbols during the assign pass and re-reading only the groups the
//     split moved measured slower (scattered per-thread loads), so recount stays a pass
//   * a 50-symbol group is costed under all tables at once: the <=6 code lengths of a symbol are
//     packed 5 bits apart into one 32-bit word, stored 16 times ([sym][lane & 15]: at most a 2-way
//     bank conflict per lookup); even and odd fields go to two accumulators whose fields are 10 bits
//     apart (a group costs at most 50 x 20 < 1024 bits)
//   * the stable median split needs no sort: histogram of costs -> threshold cost, then an
//     ordered prefix count among the groups that sit exactly on the threshold
//   * tables are rebuilt with a rank-by-counting sort of (freq<<9|sym) and one thread per table
//     running the exact in-place allocator
//   * after the final assign pass the costs of the groups are still in shared memory: their scan gives
//     every group's bit offset inside the block's code section, so the packer needs no counting pass
#include "enc.h"
#include "huffalloc.cuh"

#define HF_THREADS 256
#define HF_TILE_GROUPS 256
#define HF_TILE_BYTES (HF_TILE_GROUPS * HUFF_GROUP)
#define HF_TILE_VEC (HF_TILE_BYTES / 16)               // 16-byte pieces of a tile
#define HF_TILE_REGS ((HF_TILE_VEC + HF_THREADS - 1) / HF_THREADS)
#define HF_COPIES 16                                   // copies of the lookup table (32 would not leave room for 2 CTAs per SM)
#define HF_EVEN 0x01F07C1Fu                            // the 5-bit fields of tables 0, 2, 4 (bits 0, 10, 20)

struct HuffSmem {
  u8 tile[HF_TILE_BYTES + 16];         // staged low bytes of 256 groups (+ slack for the 14th word of the last group)
  u16 cost[SEL_STRIDE];                // best cost per group
  u8 sel[SEL_STRIDE];                  // selector per group
  u32 tbl[HUFF_MAXSYM][HF_COPIES];     // packed code lengths (5 bits per table), one copy per lane & 15
  u32 freq[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];
  int work[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];   // allocator arrays (sorted frequencies -> lengths)
  u32 skey[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];   // sort keys (freq << 9 | sym)
  u16 order[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];  // sorted position -> symbol
  u8 len[HUFF_MAXGROUPS][HUFF_MAXSYM + 6];
  u32 chist[1024];
  u32 ws[HF_THREADS / 32 + 1];
  u32 gcount[HUFF_MAXGROUPS];
  u32 misc[8];
};

// s.len of `ntab` tables -> the packed lookup s.tbl (all threads)
template <class S>
__device__ void pack_lengths(S& s, u32 ntab, u32 A) {
  for (u32 i = threadIdx.x; i < A * HF_COPIES; i += HF_THREADS) {
    const u32 sym = i / HF_COPIES;
    u32 p = 0;
    for (u32 t = 0; t < ntab; t++) p |= (u32)s.len[t][sym] << (5 * t);
    s.tbl[sym][i % HF_COPIES] = p;
  }
  __syncthreads();
}

// build the code lengths of `ntab` tables from s.freq (all threads)
__device__ void build_tables(HuffSmem& s, u32 ntab, u32 A) {
  const u32 tid = threadIdx.x;
  for (u32 i = tid; i < ntab * A; i += HF_THREADS) {
    const u32 t = i / A, sym = i % A;
    s.skey[t][sym] = (s.freq[t][sym] << 9) | sym;  // lib/Bzip2.js:566-568
  }
  __syncthreads();
  // rank by counting (keys are unique)
  for (u32 i = tid; i < ntab * A; i += HF_THREADS) {
    const u32 t = i / A, sym = i % A;
    const u32 k = s.skey[t][sym];
    u32 r = 0;
    for (u32 j = 0; j < A; j++) r += (s.skey[t][j] < k) ? 1u : 0u;
    s.order[t][r] = (u16)sym;
    s.work[t][r] = (int)(k >> 9);
  }
  __syncthreads();
  if (tid < ntab) ha_allocate(s.work[tid], (int)A, 20);  // MAX_HUFCODE_BITS lib/Bzip2.js:40
  __syncthreads();
  for (u32 i = tid; i < ntab * A; i += HF_THREADS) {
    const u32 t = i / A, r = i % A;
    s.len[t][s.order[t][r]] = (u8)s.work[t][r];
  }
  __syncthreads();
  pack_lengths(s, ntab, A);
}

// Tiles of 256 groups are staged through shared memory; the next tile's loads (and each thread's own
// group mask) are issued into registers before the current tile is consumed, so the L2/HBM latency
// overlaps the math.  The symbols are read-only for the whole kernel.
struct TileRegs {
  uint4 r[HF_TILE_REGS];
  unsigned long long hm;  // bit j: symbol j of the thread's group is >= 256
};
__device__ __forceinline__ void tile_fetch(TileRegs& t, const u8* nar, const unsigned long long* hmask, u32 g0, u32 nsel, bool any_hi) {
  const uint4* src = reinterpret_cast<const uint4*>(nar + (size_t)g0 * HUFF_GROUP);
#pragma unroll
  for (int k = 0; k < HF_TILE_REGS; k++) {
    const u32 i = k * HF_THREADS + threadIdx.x;
    if (i < HF_TILE_VEC) t.r[k] = __ldg(src + i);
  }
  t.hm = any_hi && g0 + threadIdx.x < nsel ? __ldg(hmask + g0 + threadIdx.x) : 0ull;
}
__device__ __forceinline__ void tile_store(const TileRegs& t, u8* tile) {
#pragma unroll
  for (int k = 0; k < HF_TILE_REGS; k++) {
    const u32 i = k * HF_THREADS + threadIdx.x;
    if (i < HF_TILE_VEC) reinterpret_cast<uint4*>(tile)[i] = t.r[k];
  }
}

// Calls f(sym) for the cnt symbols of the thread's group in the tile (bytes 50*tid ..).  Full groups
// without a symbol >= 256 (all but a few) read 13 words; odd-numbered groups start 2 bytes into a
// word and are realigned by a funnel shift.
template <class F>
__device__ __forceinline__ void for_group(const u8* tile, u32 cnt, unsigned long long hm, F f) {
  const u32 base = threadIdx.x * HUFF_GROUP;
  if (cnt == HUFF_GROUP && hm == 0) {
    const u32* wp = reinterpret_cast<const u32*>(tile + (base & ~3u));
    const u32 sh = (base & 2u) * 8u;
    u32 nxt = wp[0];
#pragma unroll
    for (u32 k = 0; k < 13; k++) {
      const u32 cur = nxt;
      nxt = wp[k + 1];
      const u32 w = __funnelshift_r(cur, nxt, sh);
      f(w & 0xffu);
      f((w >> 8) & 0xffu);
      if (k < 12) {
        f((w >> 16) & 0xffu);
        f(w >> 24);
      }
    }
  } else {
    for (u32 j = 0; j < cnt; j++) f((u32)tile[base + j] | (u32)((hm >> j) & 1u) << 8);
  }
}

// lib/Bzip2.js:671-684: every group goes to the table that codes it in the fewest bits
// (ties -> lowest table index).  Fills s.sel / s.cost.
template <class S>
__device__ __forceinline__ void assign_selectors(S& s, const u8* nar, const unsigned long long* hmask, u32 m, u32 nsel, u32 ntab,
                                                 bool any_hi) {
  const u32 tid = threadIdx.x, lane = tid % HF_COPIES;
  TileRegs tr;
  tile_fetch(tr, nar, hmask, 0, nsel, any_hi);
  for (u32 g0 = 0; g0 < nsel; g0 += HF_TILE_GROUPS) {
    tile_store(tr, s.tile);
    const unsigned long long hm = tr.hm;
    __syncthreads();
    if (g0 + HF_TILE_GROUPS < nsel) tile_fetch(tr, nar, hmask, g0 + HF_TILE_GROUPS, nsel, any_hi);
    const u32 g = g0 + tid;
    if (g < nsel) {
      const u32 cnt = min(50u, m - 50u * g);
      u32 ae = 0, ao = 0;
      for_group(s.tile, cnt, hm, [&](u32 sy) {
        const u32 v = s.tbl[sy][lane];
        ae += v & HF_EVEN;
        ao += (v >> 5) & HF_EVEN;
      });
      const u32 c[HUFF_MAXGROUPS] = {ae & 1023u, ao & 1023u, (ae >> 10) & 1023u, (ao >> 10) & 1023u, ae >> 20, ao >> 20};
      u32 best = 0, bc = c[0];
#pragma unroll
      for (u32 t = 1; t < HUFF_MAXGROUPS; t++)
        if (t < ntab && c[t] < bc) { best = t; bc = c[t]; }
      s.sel[g] = (u8)best;
      s.cost[g] = (u16)bc;
    }
    __syncthreads();
  }
}

template <class S>
__device__ __forceinline__ void recount(S& s, const u8* nar, const unsigned long long* hmask, u32 m, u32 nsel, u32 ntab, bool any_hi) {
  const u32 tid = threadIdx.x;
  for (u32 i = tid; i < ntab * (HUFF_MAXSYM + 2); i += HF_THREADS) (&s.freq[0][0])[i] = 0;
  TileRegs tr;
  tile_fetch(tr, nar, hmask, 0, nsel, any_hi);
  __syncthreads();
  for (u32 g0 = 0; g0 < nsel; g0 += HF_TILE_GROUPS) {
    tile_store(tr, s.tile);
    const unsigned long long hm = tr.hm;
    __syncthreads();
    if (g0 + HF_TILE_GROUPS < nsel) tile_fetch(tr, nar, hmask, g0 + HF_TILE_GROUPS, nsel, any_hi);
    const u32 g = g0 + tid;
    if (g < nsel) {
      u32* f = s.freq[s.sel[g]];
      for_group(s.tile, min(50u, m - 50u * g), hm, [&](u32 sy) { atomicAdd(&f[sy], 1u); });
    }
    __syncthreads();
  }
}

// ---- move-to-front over <= 6 table ids, list packed as six nibbles -------------------------------
__device__ __forceinline__ u32 mtf6_find(u32 list, u32 v) {
  u32 j = 0;
#pragma unroll
  for (u32 k = 1; k < HUFF_MAXGROUPS; k++) j = (((list >> (4 * k)) & 15u) == v) ? k : j;
  return j;
}
__device__ __forceinline__ u32 mtf6_front(u32 list, u32 j) {  // move the entry at position j to the front
  const u32 v = (list >> (4 * j)) & 15u;
  const u32 low = list & ((1u << (4 * j)) - 1u);
  const u32 high = list & ~((1u << (4 * (j + 1))) - 1u);
  return high | (low << 4) | v;
}
// The selector MTF is value based ("find table id v"), so a run of selectors is summarised by its
// RECENCY list: the distinct ids it used, most recent first (count in bits 28..31, unused nibbles 0).
// list after the run from any start list Y = R ++ (Y minus R).
__device__ __forceinline__ u32 rec_apply(u32 R, u32 v) {
  u32 cnt = R >> 28, lst = R & 0x00ffffffu, j = cnt;
#pragma unroll
  for (u32 k = 0; k < HUFF_MAXGROUPS; k++) j = (k < cnt && ((lst >> (4 * k)) & 15u) == v) ? k : j;
  if (j == cnt) {
    lst = ((lst << 4) | v) & 0x00ffffffu;
    cnt++;
  } else {
    const u32 low = lst & ((1u << (4 * j)) - 1u);
    const u32 high = lst & ~((1u << (4 * (j + 1))) - 1u);
    lst = high | (low << 4) | v;
  }
  return (cnt << 28) | lst;
}
__device__ __forceinline__ bool rec_has(u32 R, u32 v) {
  const u32 cnt = R >> 28;
  bool f = false;
#pragma unroll
  for (u32 k = 0; k < HUFF_MAXGROUPS; k++) f = f || (k < cnt && ((R >> (4 * k)) & 15u) == v);
  return f;
}
__device__ __forceinline__ u32 rec_op(u32 A, u32 B) {  // A = earlier run, B = later run
  u32 cnt = B >> 28, lst = B & 0x00ffffffu;
  const u32 ca = A >> 28;
#pragma unroll
  for (u32 k = 0; k < HUFF_MAXGROUPS; k++) {
    const u32 v = (A >> (4 * k)) & 15u;
    if (k < ca && !rec_has(B, v)) { lst |= v << (4 * cnt); cnt++; }
  }
  return (cnt << 28) | lst;
}
__device__ __forceinline__ u32 rec_full(u32 R) {  // R ++ (identity minus R): the full 6-entry list
  u32 cnt = R >> 28, lst = R & 0x00ffffffu;
#pragma unroll
  for (u32 v = 0; v < HUFF_MAXGROUPS; v++)
    if (!rec_has(R, v)) { lst |= v << (4 * cnt); cnt++; }
  return lst;
}

// The block's results once its selectors and code lengths are final (s.sel, s.len of ng tables, s.cost = every group's
// code bits under its table): group bit offsets, selectors, their MTF, lengths and the block's bit count.
template <class S>
__device__ void write_block(S& s, u32 blk, u32 m, u32 alpha, u32 nsel, u32 ng, const u32* __restrict__ used, u8* __restrict__ sel_out,
                            u8* __restrict__ selmtf_out, HuffBlk* __restrict__ hb, u32* __restrict__ goff_out) {
  const u32 tid = threadIdx.x, A = alpha + 2;
  // ---- results + bit accounting ----
  // bit offset of every group inside the code section: every warp scans a contiguous eighth of the groups
  // (coalesced, lane-strided), after a block scan of the eighths' sums.  A block codes at most 900001 x 20 bits.
  unsigned long long bits;
  {
    const u32 w = tid >> 5, lane = tid & 31;
    const u32 per = (nsel + HF_THREADS / 32 - 1) / (HF_THREADS / 32);
    const u32 ga = min(nsel, w * per), gb = min(nsel, ga + per);
    u32 part = 0;
    for (u32 g = ga + lane; g < gb; g += 32) part += s.cost[g];
    part = warp_reduce_add(part);
    if (lane == 0) s.ws[w] = part;
    __syncthreads();
    u32 carry = 0, total = 0;
    for (u32 i = 0; i < HF_THREADS / 32; i++) {
      const u32 x = s.ws[i];
      carry += i < w ? x : 0u;
      total += x;
    }
    u32* go = goff_out + (size_t)blk * SEL_STRIDE;
    for (u32 g0 = ga; g0 < gb; g0 += 32) {
      const u32 g = g0 + lane;
      const u32 c = g < gb ? (u32)s.cost[g] : 0u;
      const u32 inc = warp_incl_add(c);
      if (g < gb) go[g] = carry + inc - c;
      carry += __shfl_sync(FULL_MASK, inc, 31);
    }
    if (tid == 0) go[nsel] = total;
    bits = total;
    __syncthreads();
  }
  u8* so = sel_out + (size_t)blk * SEL_STRIDE;
  for (u32 g = tid; g < nsel; g += HF_THREADS) so[g] = s.sel[g];
  for (u32 i = tid; i < ng * A; i += HF_THREADS) hb->len[i / A][i % A] = s.len[i / A][i % A];
  // selectors: MTF over the table ids, unary (lib/Bzip2.js:850-862).  Parallel over threads: every
  // thread composes the permutation of its run of selectors, an exclusive scan of the compositions
  // gives its start list, then it replays its run.
  u32 selbits = 0;
  {
    const u32 per = (nsel + HF_THREADS - 1) / HF_THREADS;
    const u32 ga = min(nsel, tid * per), gb = min(nsel, ga + per);
    u32 P = 0;  // empty recency list
    for (u32 g = ga; g < gb; g++) P = rec_apply(P, s.sel[g]);
    u32* sa = s.chist;          // reuse: 2 x 256 words
    u32* sb = s.chist + HF_THREADS;
    sa[tid] = P;
    __syncthreads();
    u32 *src = sa, *dst = sb;
    for (u32 o = 1; o < HF_THREADS; o <<= 1) {
      u32 x = src[tid];
      if (tid >= o) x = rec_op(src[tid - o], x);
      dst[tid] = x;
      __syncthreads();
      u32* tmp = src; src = dst; dst = tmp;
    }
    u32 L = rec_full(tid ? src[tid - 1] : 0u);
    u8* sm = selmtf_out + (size_t)blk * SEL_STRIDE;
    for (u32 g = ga; g < gb; g++) {
      const u32 j = mtf6_find(L, s.sel[g]);
      L = mtf6_front(L, j);
      sm[g] = (u8)j;
      selbits += j + 1;
    }
    __syncthreads();
  }
  {
    unsigned long long b2 = selbits;
    __shared__ unsigned long long red2[HF_THREADS / 32];
    for (int o = 16; o > 0; o >>= 1) b2 += __shfl_xor_sync(FULL_MASK, b2, o);
    if ((tid & 31) == 0) red2[tid >> 5] = b2;
    __syncthreads();
    b2 = 0;
    for (int i = 0; i < HF_THREADS / 32; i++) b2 += red2[i];
    bits += b2;
  }
  if (tid == 0) {
    // header: 48 magic + 32 crc + 1 + 24 pidx + 16 + 16 per used range + 3 + 15 (lib/Bzip2.js:740-758, 847-849)
    unsigned long long hbits = 48 + 32 + 1 + 24 + 16 + 3 + 15;
    for (u32 r = 0; r < 16; r++) {
      const u32 w = used[blk * 8 + (r >> 1)];
      if ((w >> ((r & 1) * 16)) & 0xffffu) hbits += 16;
    }
    // tables: 5 bits + per symbol 2*|delta| + 1 (lib/Bzip2.js:610-629)
    for (u32 t = 0; t < ng; t++) {
      hbits += 5;
      u32 cur = s.len[t][0];
      for (u32 i = 0; i < A; i++) {
        const u32 l = s.len[t][i];
        hbits += 2 * (l > cur ? l - cur : cur - l) + 1;
        cur = l;
      }
    }
    hb->ngroups = ng; hb->nsel = nsel; hb->alpha = alpha; hb->m = m;
    hb->body_bits = hbits + bits;
  }
}

__global__ void __launch_bounds__(HF_THREADS, 2)
k_huffman(const u8* __restrict__ sym_lo, const unsigned long long* __restrict__ sym_hi, const u32* __restrict__ any_hi_arr,
          const u32* __restrict__ m_arr, const u32* __restrict__ freq0, const u32* __restrict__ used, u8* __restrict__ sel_out,
          u8* __restrict__ selmtf_out, HuffBlk* __restrict__ hb_out, u32* __restrict__ goff_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  HuffSmem& s = *reinterpret_cast<HuffSmem*>(smem_raw);
  const u32 tid = threadIdx.x;
  const u32 blk = blockIdx.x;
  const u32 m = m_arr[blk];
  HuffBlk* hb = hb_out + blk;
  if (m == 0) {
    if (tid == 0) { hb->ngroups = 0; hb->nsel = 0; hb->alpha = 0; hb->m = 0; hb->body_bits = 0; }
    return;
  }
  u32 alpha = 0;
  for (int k = 0; k < 8; k++) alpha += __popc(used[blk * 8 + k]);
  const u32 A = alpha + 2;                    // RUNA, RUNB, alpha-1 MTF positions, EOB
  const u32 nsel = (m + HUFF_GROUP - 1) / HUFF_GROUP;
  const u8* nar = sym_lo + ((size_t)blk << SEG_SHIFT);
  const unsigned long long* hmask = sym_hi + (size_t)blk * SEL_STRIDE;
  const bool any_hi = any_hi_arr[blk] != 0;
  u32 target;                                 // lib/Bzip2.js:826-830
  if (m >= 2400) target = 6; else if (m >= 1200) target = 5; else if (m >= 600) target = 4; else if (m >= 200) target = 3; else target = 2;
  // seed tables: global frequencies, flat frequencies (lib/Bzip2.js:835-837)
  for (u32 i = tid; i < A; i += HF_THREADS) { s.freq[0][i] = freq0[(size_t)blk * HUFF_MAXSYM + i]; s.freq[1][i] = 1; }
  __syncthreads();  // build_tables reads the seed frequencies across threads
  u32 ng = 2;
  build_tables(s, ng, A);
  while (ng < target) {
    assign_selectors(s, nar, hmask, m, nsel, ng, any_hi);
    // which table is used most? (first maximum, lib/Bzip2.js:699)
    if (tid < HUFF_MAXGROUPS) s.gcount[tid] = 0;
    for (u32 i = tid; i < 1024; i += HF_THREADS) s.chist[i] = 0;
    __syncthreads();
    {
      u32 l0 = 0, l1 = 0, l2 = 0, l3 = 0, l4 = 0, l5 = 0;
      for (u32 g = tid; g < nsel; g += HF_THREADS) {
        const u32 v = s.sel[g];
        l0 += v == 0; l1 += v == 1; l2 += v == 2; l3 += v == 3; l4 += v == 4; l5 += v == 5;
      }
      if (l0) atomicAdd(&s.gcount[0], l0);
      if (l1) atomicAdd(&s.gcount[1], l1);
      if (l2) atomicAdd(&s.gcount[2], l2);
      if (l3) atomicAdd(&s.gcount[3], l3);
      if (l4) atomicAdd(&s.gcount[4], l4);
      if (l5) atomicAdd(&s.gcount[5], l5);
    }
    __syncthreads();
    u32 which = 0;
    for (u32 t = 1; t < ng; t++) if (s.gcount[t] > s.gcount[which]) which = t;
    const u32 cntw = s.gcount[which];
    // histogram of the costs of the groups coded by `which`
    for (u32 g = tid; g < nsel; g += HF_THREADS) if (s.sel[g] == which) atomicAdd(&s.chist[s.cost[g]], 1u);
    __syncthreads();
    // stable sort by cost, upper half [cntw>>1, cntw) moves to the new table (lib/Bzip2.js:710-714):
    // threshold cost cstar: below = #(cost < cstar) <= half < #(cost <= cstar)
    if (tid == 0) {
      const u32 half = cntw >> 1;
      u32 cum = 0, cstar = 0;
      for (u32 cv = 0; cv < 1024; cv++) {
        if (cum + s.chist[cv] > half) { cstar = cv; break; }
        cum += s.chist[cv];
      }
      s.misc[0] = cstar;
      s.misc[1] = half - cum;  // how many of the groups with cost == cstar stay (the first ones in index order)
    }
    __syncthreads();
    const u32 cstar = s.misc[0], keep_eq = s.misc[1];
    {
      // ordered prefix count of (sel == which && cost == cstar) over groups in index order
      const u32 per = (nsel + HF_THREADS - 1) / HF_THREADS;
      const u32 ga = tid * per, gb = min(nsel, ga + per);
      u32 eq = 0;
      for (u32 g = ga; g < gb; g++) eq += (s.sel[g] == which && s.cost[g] == cstar) ? 1u : 0u;
      u32 tot;
      u32 ex = block_excl_add<HF_THREADS, u32>(eq, s.ws, &tot);
      for (u32 g = ga; g < gb; g++) {
        if (s.sel[g] != which) continue;
        const u32 cg = s.cost[g];
        bool move;
        if (cg > cstar) move = true;
        else if (cg < cstar) move = false;
        else { move = ex >= keep_eq; ex++; }
        if (move) s.sel[g] = (u8)ng;
      }
    }
    __syncthreads();
    ng++;
    recount(s, nar, hmask, m, nsel, ng, any_hi);
    build_tables(s, ng, A);
  }
  assign_selectors(s, nar, hmask, m, nsel, ng, any_hi);  // lib/Bzip2.js:843
  write_block(s, blk, m, alpha, nsel, ng, used, sel_out, selmtf_out, hb, goff_out);
}

// ---- libbz2 flavor (bzlib 1.0.3+ compress.c sendMTFValues, huffman.c BZ2_hbMakeCodeLengths) ----------------------
// Initial tables from a partition of the symbol frequencies, then four rounds of assign + recount + rebuild; the
// selectors of the 4th assignment and the tables built after it are written.  The assign and recount passes are those
// of the compressjs search (lengths <= 17 and the initial 0 / 15 fit the packed 5-bit lookup); the tables of a round are
// built side by side, one thread per table running the heap builder.
struct LbHeap {                        // BZ2_hbMakeCodeLengths of one table (nodes 1..A leaves, A+1.. internal)
  u32 weight[2 * HUFF_MAXSYM];         // freq << 8 | depth
  u16 parent[2 * HUFF_MAXSYM];         // LB_ROOT: none
  u16 heap[HUFF_MAXSYM + 2];           // 1-based min-heap of node numbers, heap[0] = sentinel node 0 (weight 0)
};
#define LB_ROOT 0xffffu
#define LB_MAXLEN 17
struct HuffSmemL {
  u8 tile[HF_TILE_BYTES + 16];
  u16 cost[SEL_STRIDE];
  u8 sel[SEL_STRIDE];
  u32 tbl[HUFF_MAXSYM][HF_COPIES];
  u32 freq[HUFF_MAXGROUPS][HUFF_MAXSYM + 2];
  u8 len[HUFF_MAXGROUPS][HUFF_MAXSYM + 6];
  union {
    LbHeap hp[HUFF_MAXGROUPS];
    u32 chist[2 * HF_THREADS];         // write_block's selector scan, after the last build
  };
  u32 ws[HF_THREADS / 32 + 1];
};
// 114 KB with write_block's reduction: two CTAs per SM, as k_huffman
static_assert(sizeof(HuffSmemL) + 64 <= 115 * 1024, "two libbz2 Huffman CTAs per SM");

__device__ __forceinline__ void lb_up(LbHeap& h, u32 z) {
  const u32 tmp = h.heap[z];
  while (h.weight[tmp] < h.weight[h.heap[z >> 1]]) { h.heap[z] = h.heap[z >> 1]; z >>= 1; }
  h.heap[z] = (u16)tmp;
}
__device__ __forceinline__ void lb_down(LbHeap& h, u32 z, u32 nHeap) {
  const u32 tmp = h.heap[z];
  for (;;) {
    u32 y = z << 1;
    if (y > nHeap) break;
    if (y < nHeap && h.weight[h.heap[y + 1]] < h.weight[h.heap[y]]) y++;
    if (h.weight[tmp] < h.weight[h.heap[y]]) break;
    h.heap[z] = h.heap[y];
    z = y;
  }
  h.heap[z] = (u16)tmp;
}
// code lengths of one table (one thread): Huffman by the heap above, depth in the weights' low byte as tie-break; while
// a length exceeds 17 every frequency f becomes 1 + f / 2 and the tree is built again
__device__ void lb_make_lengths(LbHeap& h, const u32* freq, u8* len, u32 A) {
  for (u32 i = 0; i < A; i++) h.weight[i + 1] = (freq[i] ? freq[i] : 1u) << 8;
  for (;;) {
    u32 nNodes = A, nHeap = 0;
    h.heap[0] = 0; h.weight[0] = 0;
    for (u32 i = 1; i <= A; i++) {
      h.parent[i] = LB_ROOT;
      h.heap[++nHeap] = (u16)i;
      lb_up(h, nHeap);
    }
    while (nHeap > 1) {
      const u32 n1 = h.heap[1];
      h.heap[1] = h.heap[nHeap--];
      lb_down(h, 1, nHeap);
      const u32 n2 = h.heap[1];
      h.heap[1] = h.heap[nHeap--];
      lb_down(h, 1, nHeap);
      nNodes++;
      h.parent[n1] = h.parent[n2] = (u16)nNodes;
      const u32 w1 = h.weight[n1], w2 = h.weight[n2];
      h.weight[nNodes] = ((w1 & 0xffffff00u) + (w2 & 0xffffff00u)) | (1u + max(w1 & 0xffu, w2 & 0xffu));
      h.parent[nNodes] = LB_ROOT;
      h.heap[++nHeap] = (u16)nNodes;
      lb_up(h, nHeap);
    }
    bool too_long = false;
    for (u32 i = 1; i <= A; i++) {
      u32 j = 0;
      for (u32 k = i; h.parent[k] != LB_ROOT; k = h.parent[k]) j++;
      len[i - 1] = (u8)j;
      too_long |= j > LB_MAXLEN;
    }
    if (!too_long) return;
    for (u32 i = 1; i <= A; i++) h.weight[i] = (1u + (h.weight[i] >> 8) / 2) << 8;
  }
}

// s.cost[g] = the bits of group g under the table it selected (the 4th assignment costed it under the tables before)
__device__ void cost_selected(HuffSmemL& s, const u8* nar, const unsigned long long* hmask, u32 m, u32 nsel, bool any_hi) {
  const u32 tid = threadIdx.x, lane = tid % HF_COPIES;
  TileRegs tr;
  tile_fetch(tr, nar, hmask, 0, nsel, any_hi);
  for (u32 g0 = 0; g0 < nsel; g0 += HF_TILE_GROUPS) {
    tile_store(tr, s.tile);
    const unsigned long long hm = tr.hm;
    __syncthreads();
    if (g0 + HF_TILE_GROUPS < nsel) tile_fetch(tr, nar, hmask, g0 + HF_TILE_GROUPS, nsel, any_hi);
    const u32 g = g0 + tid;
    if (g < nsel) {
      const u32 sh = 5 * s.sel[g];
      u32 c = 0;
      for_group(s.tile, min(50u, m - 50u * g), hm, [&](u32 sy) { c += (s.tbl[sy][lane] >> sh) & 31u; });
      s.cost[g] = (u16)c;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(HF_THREADS, 2)
k_huffman_libbz2(const u8* __restrict__ sym_lo, const unsigned long long* __restrict__ sym_hi, const u32* __restrict__ any_hi_arr,
                 const u32* __restrict__ m_arr, const u32* __restrict__ freq0, const u32* __restrict__ used, u8* __restrict__ sel_out,
                 u8* __restrict__ selmtf_out, HuffBlk* __restrict__ hb_out, u32* __restrict__ goff_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  HuffSmemL& s = *reinterpret_cast<HuffSmemL*>(smem_raw);
  const u32 tid = threadIdx.x;
  const u32 blk = blockIdx.x;
  const u32 m = m_arr[blk];
  HuffBlk* hb = hb_out + blk;
  if (m == 0) {
    if (tid == 0) { hb->ngroups = 0; hb->nsel = 0; hb->alpha = 0; hb->m = 0; hb->body_bits = 0; }
    return;
  }
  u32 alpha = 0;
  for (int k = 0; k < 8; k++) alpha += __popc(used[blk * 8 + k]);
  const u32 A = alpha + 2;
  const u32 nsel = (m + HUFF_GROUP - 1) / HUFF_GROUP;
  const u8* nar = sym_lo + ((size_t)blk << SEG_SHIFT);
  const unsigned long long* hmask = sym_hi + (size_t)blk * SEL_STRIDE;
  const bool any_hi = any_hi_arr[blk] != 0;
  u32 ng;
  if (m < 200) ng = 2; else if (m < 600) ng = 3; else if (m < 1200) ng = 4; else if (m < 2400) ng = 5; else ng = 6;
  // initial tables: table nPart-1 codes the symbols gs..ge of a run of about remF / nPart of the frequency in 0 bits,
  // everything else in 15
  if (tid == 0) {
    const u32* mf = freq0 + (size_t)blk * HUFF_MAXSYM;
    u32 remF = m, gs = 0;
    for (u32 nPart = ng; nPart > 0; nPart--) {
      const u32 tFreq = remF / nPart;
      int ge = (int)gs - 1;
      u32 aFreq = 0;
      while (aFreq < tFreq && ge < (int)A - 1) aFreq += mf[++ge];
      if (ge > (int)gs && nPart != ng && nPart != 1 && ((ng - nPart) & 1)) aFreq -= mf[ge--];
      for (u32 v = 0; v < A; v++) s.len[nPart - 1][v] = ((int)v >= (int)gs && (int)v <= ge) ? 0 : 15;
      gs = (u32)(ge + 1);
      remF -= aFreq;
    }
  }
  __syncthreads();
  pack_lengths(s, ng, A);
  for (int it = 0; it < 4; it++) {
    assign_selectors(s, nar, hmask, m, nsel, ng, any_hi);
    recount(s, nar, hmask, m, nsel, ng, any_hi);
    if (tid < ng) lb_make_lengths(s.hp[tid], s.freq[tid], s.len[tid], A);
    __syncthreads();
    pack_lengths(s, ng, A);
  }
  cost_selected(s, nar, hmask, m, nsel, any_hi);
  write_block(s, blk, m, alpha, nsel, ng, used, sel_out, selmtf_out, hb, goff_out);
}

void huffman_batch(Ctx& c, const NarrowSyms& sym, const u32* d_m, const u32* d_freq, const u32* d_used, u32 nblk, u8* d_sel, u8* d_selmtf,
                   HuffBlk* d_hb, u32* d_goff) {
  static bool attr = false;
  if (!attr) {
    CUDA_CHECK(cudaFuncSetAttribute(k_huffman, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HuffSmem)));
    CUDA_CHECK(cudaFuncSetAttribute(k_huffman_libbz2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HuffSmemL)));
    attr = true;
  }
  if (c.bz_flavor == B2_BZ2_LIBBZ2) {
    k_huffman_libbz2<<<nblk, HF_THREADS, sizeof(HuffSmemL), c.stream>>>(sym.lo, sym.hi, sym.any_hi, d_m, d_freq, d_used, d_sel, d_selmtf, d_hb,
                                                                        d_goff);
    KLAUNCH(c); KCHECK();
    return;
  }
  k_huffman<<<nblk, HF_THREADS, sizeof(HuffSmem), c.stream>>>(sym.lo, sym.hi, sym.any_hi, d_m, d_freq, d_used, d_sel, d_selmtf, d_hb, d_goff);
  KLAUNCH(c); KCHECK();
}
