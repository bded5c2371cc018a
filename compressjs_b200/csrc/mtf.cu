// mtf.cu -- symbol map, move-to-front and zero-run (RUNA/RUNB) coding of the BWT output.
//
// Reference: lib/Bzip2.js:743-815 (compressBlock: used[] map, MTF list M, RLE2 emit) and
// lib/Bzip2.js:53-60 (mtf()).  The reference walks the block byte by byte with a linear
// search in M.  Parallel form:
//   k_used        : 256-bit "byte occurs in block" map per block
//   k_mtf_lastpos : per 4 KiB chunk (one warp each), last position of every byte value inside the chunk
//   k_mtf_prefix  : per block, running max over the chunks -> last occurrence BEFORE each chunk;
//                   the MTF list at a chunk start is "bytes by most recent occurrence, then the
//                   not-yet-seen used bytes in ascending order" (the initial list M)
//   k_mtf_ranks   : one warp per chunk, 32 bytes per step: every byte value carries a recency key
//                   (255 - rank at the chunk start, found by a register bitonic sort, or 256 + position
//                   of its last occurrence inside the chunk); the rank of a byte is the number of live
//                   keys above its own, counted through a bucketed live-key bitmap with suffix sums, and
//                   the bytes of one step that precede each other are settled with a ballot radix compare
//                   The same pass summarises the chunk for the zero-run coder: leading / trailing zeros and the number
//                   of symbols its non-zero ranks and interior runs will emit.
//   k_rle2_scan   : one warp per block walks the chunk summaries: output offset and carried-in run length of every chunk
//                   (a run belongs to the chunk that holds the non-zero rank ending it); final run + EOB + m
//   k_rle2        : zero ranks form runs -> bijective base-2 RUNA/RUNB digits (lib/Bzip2.js:783-794); every chunk knows
//                   its offsets, so there is no chain between tiles; symbols in one byte each (NarrowSyms, enc.h) +
//                   histogram
#include "enc.h"

#define MTF_CHUNK 4096

__global__ void __launch_bounds__(256) k_used(const u8* __restrict__ U, const u32* __restrict__ seg_n, u32 tiles_per_seg, u32* __restrict__ used) {
  __shared__ u32 f[8];
  if (threadIdx.x < 8) f[threadIdx.x] = 0;
  __syncthreads();
  const u32 seg = blockIdx.x / tiles_per_seg, lt = blockIdx.x % tiles_per_seg;
  const u32 n = seg_n[seg];
  const u32 start = lt * (256 * 64);
  if (start >= n) return;
  const u8* p = U + ((size_t)seg << SEG_SHIFT);
  u32 loc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (u32 i = start + threadIdx.x; i < min(n, start + 256 * 64); i += 256) {
    u8 c = p[i];
    loc[c >> 5] |= 1u << (c & 31);
  }
#pragma unroll
  for (int k = 0; k < 8; k++)
    if (loc[k]) atomicOr(&f[k], loc[k]);
  __syncthreads();
  if (threadIdx.x < 8 && f[threadIdx.x]) atomicOr(&used[seg * 8 + threadIdx.x], f[threadIdx.x]);
}

__global__ void __launch_bounds__(256) k_used_from_hist(const u32* __restrict__ hist, u32* __restrict__ used) {
  const u32 bal = __ballot_sync(FULL_MASK, hist[blockIdx.x * 256 + threadIdx.x] != 0);
  if ((threadIdx.x & 31) == 0) used[blockIdx.x * 8 + (threadIdx.x >> 5)] = bal;
}

// lastpos[(seg*cps + chunk)*256 + c] = (last position of byte c inside the chunk) + 1, 0 if none.
// One warp per chunk; every lane reads 16 bytes at a time and folds them into the warp's table with shared atomicMax.
#define LP_WARPS 8
__global__ void __launch_bounds__(LP_WARPS * 32)
k_mtf_lastpos(const u8* __restrict__ U, const u32* __restrict__ seg_n, u32 cps, u32 nchunks, u32* __restrict__ lastpos) {
  __shared__ __align__(16) u32 last[LP_WARPS][256];
  const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const u32 gchunk = blockIdx.x * LP_WARPS + w;
  if (gchunk >= nchunks) return;
  u32* L = last[w];
  uint4* L4 = reinterpret_cast<uint4*>(L);
  L4[2 * lane] = make_uint4(0, 0, 0, 0);
  L4[2 * lane + 1] = make_uint4(0, 0, 0, 0);
  __syncwarp();
  const u32 seg = gchunk / cps, ch = gchunk % cps;
  const u32 n = seg_n[seg];
  const u32 start = ch * MTF_CHUNK;
  if (start < n) {
    const u8* p = U + ((size_t)seg << SEG_SHIFT);
    const u32 end = min(n, start + MTF_CHUNK);
    for (u32 i0 = start + lane * 16; i0 < end; i0 += 512) {
      const uint4 x = *reinterpret_cast<const uint4*>(p + i0);  // inside the 1 MiB slot; bytes past n are skipped
      const u32 xw[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int j = 0; j < 16; j++)
        if (i0 + j < end) atomicMax(&L[(xw[j >> 2] >> (8 * (j & 3))) & 255u], i0 + j + 1);
    }
  }
  __syncwarp();
  uint4* out = reinterpret_cast<uint4*>(lastpos + (size_t)gchunk * 256);
  out[2 * lane] = L4[2 * lane];
  out[2 * lane + 1] = L4[2 * lane + 1];
}

// in place: lastpos[chunk] := max over earlier chunks (exclusive).  The loads of 16 chunks are issued together, so the
// walk over a block's ~220 chunks waits for memory 14 times instead of 220.
#define MP_BATCH 16
__global__ void __launch_bounds__(256) k_mtf_prefix(const u32* __restrict__ seg_n, u32 cps, u32* __restrict__ lastpos) {
  const u32 seg = blockIdx.x;
  const u32 n = seg_n[seg];
  const u32 nch = (n + MTF_CHUNK - 1) / MTF_CHUNK;
  u32* p = lastpos + (size_t)seg * cps * 256 + threadIdx.x;
  u32 run = 0;
  for (u32 ch0 = 0; ch0 < nch; ch0 += MP_BATCH) {
    u32 t[MP_BATCH];
#pragma unroll
    for (int j = 0; j < MP_BATCH; j++) t[j] = ch0 + j < nch ? p[(size_t)(ch0 + j) * 256] : 0u;
#pragma unroll
    for (int j = 0; j < MP_BATCH; j++) {
      if (ch0 + j < nch) p[(size_t)(ch0 + j) * 256] = run;
      run = max(run, t[j]);
    }
  }
}

#define MR_WARPS 8
#define MB_BUCKETS 36   // recency keys live in [0, 256 + 4096): 34 buckets of 128 values (+ slack), two per lane
struct MtfWarp {
  u16 K[256];                       // recency key of every byte value (larger = used more recently)
  __align__(16) u32 bm[MB_BUCKETS][4];  // bitmap of the key values that are currently somebody's key
  u32 nz[MTF_CHUNK / 32];           // bit i of word s: rank 32 s + i of the chunk is not zero
};
// MTF rank of a byte = number of byte values used more recently than it.  Every byte value carries
// a 13-bit recency key: (list position at the chunk start, 0 = back of the list) until it is used inside
// the chunk, 256 + (position inside the chunk) afterwards.  A warp ranks 32 bytes per step:
//   * first use of a byte in the window: r0_i = #{keys alive before the window that are > its key}
//     (bucket suffix sums + bitmap) -- its rank at the window start
//   * T_i = time of the previous use of lane i's byte on a 9-bit scale that keeps the order of those times:
//     255 - r0_i for a first use, 256 + prev_i for a byte an earlier lane prev_i of the window holds
//   * rank_i = (r0_i for a first use) + #{k in (prev_i, i) : T_k < T_i}   (bytes first used after T_i inside the
//     window), with the T_k < T_i lane mask built by a 9-round ballot radix compare, low bit first (no equal-so-far
//     mask to carry)
//   * only the last use of a byte inside the window rewrites its key.
// The zero-run summary of the chunk is not kept step by step: every step stores the ballot of its non-zero ranks, and
// the warp reads the chunk's 4096 bits once at the end.
__global__ void __launch_bounds__(MR_WARPS * 32)
k_mtf_ranks(const u8* __restrict__ U, const u32* __restrict__ seg_n, u32 cps, const u32* __restrict__ lastpos,
            const u32* __restrict__ used, u8* __restrict__ R, u32 nblk, uint4* __restrict__ rsum) {
  __shared__ MtfWarp sm[MR_WARPS];
  const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const u32 gchunk = blockIdx.x * MR_WARPS + w;
  const u32 seg = gchunk / cps, ch = gchunk % cps;
  // (every warp of the grid maps to a valid (seg, chunk) pair or exits as a whole)
  if (seg >= nblk) return;
  const u32 n = seg_n[seg];
  const u32 start = ch * MTF_CHUNK;
  if (start >= n) return;
  const u32 count = min((u32)MTF_CHUNK, n - start);
  MtfWarp& s = sm[w];
  const uint4* bm4 = reinterpret_cast<const uint4*>(&s.bm[0][0]);
  // ---- list position of every byte value at the chunk start ----
  // The list is: bytes seen before the chunk, most recent first; then the used bytes not seen yet, ascending; then the
  // bytes the block never holds.  Sort keys carry the byte value in their low 8 bits and are all distinct:
  //   seen 2^30 | lastpos << 8 | c,   not seen yet 2^29 | (255 - c) << 8 | c,   never held (255 - c) << 8 | c.
  // A bitonic sort of the 256 keys, 8 per lane in lane-major order, puts them in ascending order; the sorted index of
  // a byte is then its list position counted from the back.
  u32 v[8];
  {
    const uint4* lp4 = reinterpret_cast<const uint4*>(lastpos + (size_t)gchunk * 256 + lane * 8);
    const uint4 l0 = lp4[0], l1 = lp4[1];
    const u32 l[8] = {l0.x, l0.y, l0.z, l0.w, l1.x, l1.y, l1.z, l1.w};
    const u32 uw = used[seg * 8 + (lane >> 2)] >> ((lane & 3) * 8);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const u32 c = lane * 8 + i;
      if (l[i]) v[i] = 0x40000000u | (l[i] << 8) | c;
      else v[i] = (((uw >> i) & 1u) << 29) | ((255u - c) << 8) | c;
    }
  }
#pragma unroll
  for (u32 k = 2; k <= 256; k <<= 1) {
#pragma unroll
    for (u32 j = k >> 1; j > 0; j >>= 1) {
      if (j >= 8) {  // partner in lane ^ (j / 8), same register
        const bool lower = !(lane & (j >> 3));
        const bool asc = !((lane * 8) & k);
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const u32 o = __shfl_xor_sync(FULL_MASK, v[i], j >> 3);
          v[i] = (lower == asc) ? min(v[i], o) : max(v[i], o);
        }
      } else {       // partner in the same lane, register i ^ j
#pragma unroll
        for (int i = 0; i < 8; i++) {
          if (i & j) continue;
          const bool asc = !((lane * 8 + i) & k);
          const u32 a = v[i], b = v[i | j];
          v[i] = asc ? min(a, b) : max(a, b);
          v[i | j] = asc ? max(a, b) : min(a, b);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; i++) s.K[v[i] & 255u] = (u16)(lane * 8 + i);
  // all 256 start keys 0..255 are alive: buckets 0 and 1 full, the rest empty
  for (u32 i = lane; i < MB_BUCKETS * 4; i += 32) (&s.bm[0][0])[i] = (i < 8) ? 0xffffffffu : 0u;
  __syncwarp();
  const u8* src = U + ((size_t)seg << SEG_SHIFT) + start;
  u8* dst = R + ((size_t)seg << SEG_SHIFT) + start;
  for (u32 base = 0; base < count; base += 32) {
    const bool valid = base + lane < count;
    const u32 c = valid ? (u32)src[base + lane] : (256u + lane);
    // ---- bucket suffix sums of the keys alive before this window: lane l holds buckets 2l and 2l+1 ----
    u32 spair;  // (S[2l] << 16) | S[2l+1], S[b] = number of live keys in buckets above b
    {
      u32 ca = 0, cb = 0;
      if (lane < MB_BUCKETS / 2) {
        const uint4 a = bm4[2 * lane], b = bm4[2 * lane + 1];
        ca = __popc(a.x) + __popc(a.y) + __popc(a.z) + __popc(a.w);
        cb = __popc(b.x) + __popc(b.y) + __popc(b.z) + __popc(b.w);
      }
      u32 x = ca + cb;  // inclusive suffix sum over lanes (high lanes first)
#pragma unroll
      for (int o = 1; o < MB_BUCKETS / 2; o <<= 1) { const u32 t = __shfl_down_sync(FULL_MASK, x, o); if (lane + o < 32) x += t; }
      spair = ((x - ca) << 16) | (x - ca - cb);
    }
    // ---- who used my byte last? ----
    const u32 m = __match_any_sync(FULL_MASK, c);
    const u32 pm = m & lanemask_lt();
    const int prev = pm ? (31 - __clz(pm)) : -1;
    const bool is_last = (m >> lane) <= 1u;  // no higher lane holds the same byte
    const u32 tb = 256u + base;
    const u32 q = valid ? (u32)s.K[c] : 0u;
    const u32 b = q >> 7;
    const u32 sb = __shfl_sync(FULL_MASK, spair, b >> 1);
    // ---- r0: keys alive before the window and more recent than q (only for the first use of a byte) ----
    u32 rank = 0, T = 256u + (u32)prev;
    if (prev < 0) {
      if (valid) {
        const u32 off = q & 127u, wi = off >> 5;
        const uint4 bw = bm4[b];
        rank = (b & 1) ? (sb & 0xffffu) : (sb >> 16);
        const u32 cur = wi == 0 ? bw.x : (wi == 1 ? bw.y : (wi == 2 ? bw.z : bw.w));
        rank += __popc(cur & ((0xfffffffeu) << (off & 31u)));
        if (wi < 1) rank += __popc(bw.y);
        if (wi < 2) rank += __popc(bw.z);
        if (wi < 3) rank += __popc(bw.w);
      }
      T = 255u - rank;
    }
    // ---- bytes first used after T_i inside the window: k in (prev_i, i) with T_k < T_i ----
    {
      // after bits 0..b: lt = lanes whose T is below mine in those bits.  Where my bit is 1, every lane with a 0 there
      // is below me; where it is 0, only lanes that were below and have a 0 there stay below.
      u32 lt = 0;
#pragma unroll
      for (int bit = 0; bit <= 8; bit++) {
        const bool one = T & (1u << bit);
        const u32 nB = ~__ballot_sync(FULL_MASK, one);
        lt = one ? (lt | nB) : (lt & nB);
      }
      rank += __popc(lt & lanemask_lt() & (FULL_MASK << (u32)(prev + 1)));
    }
    if (valid) dst[base + lane] = (u8)rank;
    {
      const u32 nzm = __ballot_sync(FULL_MASK, valid && rank != 0);
      if (lane == 0) s.nz[base >> 5] = nzm;
    }
    // ---- the last use of every byte in the window rewrites its key ----
    if (valid && is_last) {
      atomicAnd(&s.bm[q >> 7][(q & 127u) >> 5], ~(1u << (q & 31u)));
      s.K[c] = (u16)(tb + lane);
    }
    const u32 newbits = __ballot_sync(FULL_MASK, valid && is_last);
    // windows are 32-aligned and every old key is below tb: this word is ours alone
    if (lane == 0) s.bm[tb >> 7][(tb & 127u) >> 5] = newbits;
    __syncwarp();
  }
  // ---- zero-run summary: leading zeros, trailing zeros, symbols emitted by the non-zero ranks and interior runs ----
  // Lane l reads the bits of ranks [128 l, 128 l + 128).  A non-zero rank emits itself and, unless it is the first of
  // the chunk (the run in front of that one is carried in by the block scan), the digits of the zero run before it.
  {
    u32 nzw[4], mylast = 0;  // mylast: position + 1 of the lane's last non-zero rank, 0 if none
    const u32 nw = (count + 31) >> 5;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      nzw[k] = lane * 4 + k < nw ? s.nz[lane * 4 + k] : 0u;
      if (nzw[k]) mylast = lane * 128 + 32 * k + 32 - __clz(nzw[k]);
    }
    const u32 inc = warp_incl_max(mylast);
    u32 pp = __shfl_up_sync(FULL_MASK, inc, 1);  // position + 1 of the last non-zero rank before the lane's bits
    if (lane == 0) pp = 0;
    u32 acc = 0, lead = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const u32 x = nzw[k], p0 = lane * 128 + 32 * k;
      acc += __popc(x);
      // non-zero ranks with a zero rank right in front of them (or, at p0 = 0, the chunk start)
      u32 y = x & ~((x << 1) | (pp == p0 ? 1u : 0u));
      while (y) {
        const u32 bit = __ffs(y) - 1;
        y &= y - 1;
        const u32 low = x & ((1u << bit) - 1u);
        const u32 q = low ? p0 + 32 - __clz(low) : pp;
        if (q == 0) lead = p0 + bit;
        else acc += 31 - __clz(p0 + bit - q + 1);
      }
      if (x) pp = p0 + 32 - __clz(x);
    }
    const u32 inner = warp_reduce_add(acc);
    const u32 last = __shfl_sync(FULL_MASK, inc, 31);
    lead = warp_reduce_max(lead);
    if (lane == 0) rsum[gchunk] = last ? make_uint4(lead, count - last, inner, 0u) : make_uint4(count, count, 0u, 1u);
  }
}

// One warp per block: walk the chunk summaries in order (lib/Bzip2.js:783-794 flushes a run when the next non-zero
// rank arrives, so the run is charged to the chunk holding that rank).  plan[chunk] = (output offset, zeros carried in).
__global__ void __launch_bounds__(32)
k_rle2_scan(const uint4* __restrict__ rsum, const u32* __restrict__ seg_n, u32 cps, const u32* __restrict__ used, uint2* __restrict__ plan,
            u8* __restrict__ A, unsigned long long* __restrict__ hi, u32* __restrict__ any_hi, u32* __restrict__ m_out,
            u32* __restrict__ freq) {
  const u32 seg = blockIdx.x, lane = threadIdx.x;
  const u32 n = seg_n[seg];
  if (n == 0) return;
  const u32 nch = (n + MTF_CHUNK - 1) / MTF_CHUNK;
  u32 carry = 0, o = 0;
  for (u32 c0 = 0; c0 < nch; c0 += 32) {
    const u32 k = c0 + lane;
    uint4 v = make_uint4(0, 0, 0, 1);
    if (k < nch) v = rsum[(size_t)seg * cps + k];
    u32 my_o = 0, my_c = 0;
    const u32 lim = min(32u, nch - c0);
    for (u32 j = 0; j < lim; j++) {
      const u32 lead = __shfl_sync(FULL_MASK, v.x, j), trail = __shfl_sync(FULL_MASK, v.y, j);
      const u32 inner = __shfl_sync(FULL_MASK, v.z, j), allz = __shfl_sync(FULL_MASK, v.w, j);
      if (lane == j) { my_o = o; my_c = carry; }
      if (allz) carry += lead;
      else {
        const u32 r = carry + lead;
        o += (r ? 31 - __clz(r + 1) : 0) + inner;
        carry = trail;
      }
    }
    if (k < nch) plan[(size_t)seg * cps + k] = make_uint2(my_o, my_c);
  }
  if (lane == 0) {
    u8* a = A + ((size_t)seg << SEG_SHIFT);
    u32* fq = freq + (size_t)seg * HUFF_MAXSYM;
    u32 L = carry, f0 = 0, f1 = 0;
    while (L) {  // the run still open at the end of the block
      if (L & 1) { a[o++] = 0; f0++; L -= 1; }
      else { a[o++] = 1; f1++; L -= 2; }
      L >>= 1;
    }
    u32 alpha = 0;
    for (int k = 0; k < 8; k++) alpha += __popc(used[seg * 8 + k]);
    a[o] = (u8)(alpha + 1);  // end of block symbol
    if (alpha + 1 >= 256) {
      atomicOr(&hi[(size_t)seg * SEL_STRIDE + o / HUFF_GROUP], 1ull << (o % HUFF_GROUP));
      any_hi[seg] = 1;
    }
    if (f0) atomicAdd(&fq[0], f0);
    if (f1) atomicAdd(&fq[1], f1);
    atomicAdd(&fq[alpha + 1], 1u);
    m_out[seg] = o + 1;
  }
}

// The masks of the slots whose flag the previous batch set go back to zero (the masks of all other slots are zero).
__global__ void __launch_bounds__(256) k_clear_hi(const u32* __restrict__ any_hi, unsigned long long* __restrict__ hi) {
  if (!any_hi[blockIdx.x]) return;
  uint4* h = reinterpret_cast<uint4*>(hi + (size_t)blockIdx.x * SEL_STRIDE);
  for (u32 i = threadIdx.x; i < SEL_STRIDE / 2; i += 256) h[i] = make_uint4(0, 0, 0, 0);
}

// ---- RLE2 ---------------------------------------------------------------------------------
#define R2_THREADS 256
#define R2_ITEMS 16
#define R2_TILE (R2_THREADS * R2_ITEMS)   // == MTF_CHUNK: one tile per chunk summary

__global__ void __launch_bounds__(R2_THREADS)
k_rle2(const u8* __restrict__ R, const u32* __restrict__ seg_n, u32 tps, const uint2* __restrict__ plan, u8* __restrict__ A,
       unsigned long long* __restrict__ hi, u32* __restrict__ any_hi, u32* __restrict__ freq) {
  __shared__ u32 hist[HUFF_MAXSYM];
  __shared__ uint4 wrec[R2_THREADS / 32];
  // the tile's symbols are staged here at the alignment (mod 16 symbols = 16 bytes) they have in global memory, then
  // copied out in 16-byte pieces: at most one symbol per rank plus the digits of the run that was carried in
  __shared__ __align__(16) u8 stage[R2_TILE + 48];
  const u32 tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const u32 seg = blockIdx.x / tps, lt = blockIdx.x % tps;
  const u32 n = seg_n[seg];
  const u32 start = lt * R2_TILE;
  if (start >= n) return;
  for (u32 i = tid; i < HUFF_MAXSYM; i += R2_THREADS) hist[i] = 0;
  const uint2 pl = plan[(size_t)seg * tps + lt];
  const u8* r = R + ((size_t)seg << SEG_SHIFT);
  u8* a = A + ((size_t)seg << SEG_SHIFT);
  const u32 p0 = start + tid * R2_ITEMS;
  const uint4 rv = *reinterpret_cast<const uint4*>(r + p0);  // inside the 1 MiB slot; bytes past n are ignored below
  const u32 xw[4] = {rv.x, rv.y, rv.z, rv.w};
#define R2_RANK(j) ((xw[(j) >> 2] >> (8 * ((j) & 3))) & 255u)
  // A non-zero rank flushes the zero run in front of it (floor(log2(L + 1)) digits for L zeros), then writes itself.
  // Per thread: first and last non-zero position (+1, 0 if none) and the symbols of its items, but for the digits of
  // the run in front of its first non-zero, which reaches back into earlier threads.
  u32 fnz = 0, lnz = 0, own = 0;
#pragma unroll
  for (int j = 0; j < R2_ITEMS; j++) {
    const u32 p = p0 + j;
    if (p < n && R2_RANK(j) != 0) {
      if (lnz) { const u32 L = p - lnz; own += 1 + (L ? 31 - __clz(L + 1) : 0); }
      else { own += 1; fnz = p + 1; }
      lnz = p + 1;
    }
  }
  // inside the warp: position after the last non-zero of the lanes below (0 if none)
  const u32 inc = warp_incl_max(lnz);
  u32 exw = __shfl_up_sync(FULL_MASK, inc, 1);
  if (lane == 0) exw = 0;
  // per warp: (position after its last non-zero, its first non-zero + 1, its symbols but for the digits of the run in
  // front of its first non-zero); a warp's run comes in from the warps below, which one barrier hands over
  {
    const u32 s = warp_reduce_add((fnz && exw) ? own + (31 - __clz(fnz - exw)) : own);  // fnz - 1 - exw zeros in front
    const u32 fm = __ballot_sync(FULL_MASK, fnz != 0);
    const u32 F = __shfl_sync(FULL_MASK, fnz, fm ? __ffs(fm) - 1 : 0);
    const u32 Lw = __shfl_sync(FULL_MASK, inc, 31);
    if (lane == 0) wrec[w] = make_uint4(Lw, F, s, 0u);
  }
  __syncthreads();
  // walk the warps' records: position after the last non-zero in front of this warp, its output offset, the tile's
  u32 run = start - pl.y, woff = 0, tot_off = 0, wrun = 0;  // (pl.y zeros were carried into the tile)
#pragma unroll
  for (u32 k = 0; k < R2_THREADS / 32; k++) {
    const uint4 rec = wrec[k];
    if (k == w) { wrun = run; woff = tot_off; }
    tot_off += rec.y ? rec.z + (31 - __clz(rec.y - run)) : rec.z;
    if (rec.x) run = rec.x;
  }
  u32 rs = max(wrun, exw);  // position after the last non-zero in front of this thread's items
  const u32 mine = fnz ? own + (31 - __clz(fnz - rs)) : own;
  const u32 first = pl.x & 15u;
  u32 o = first + woff + warp_incl_add(mine) - mine;  // index into `stage`
#pragma unroll
  for (int j = 0; j < R2_ITEMS; j++) {
    const u32 p = p0 + j;
    const u32 v = R2_RANK(j);
    if (p < n && v != 0) {
      u32 L = p - rs;
      rs = p + 1;
      while (L) {  // lib/Bzip2.js:783-794 emitLastRun
        if (L & 1) { stage[o++] = 0; atomicAdd(&hist[0], 1u); L -= 1; }
        else { stage[o++] = 1; atomicAdd(&hist[1], 1u); L -= 2; }
        L >>= 1;
      }
      const u32 sy = v + 1;
      if (sy == 256) {  // rank 255: a rare mask bit (a group can straddle two tiles, hence the atomic)
        const u32 og = pl.x - first + o;
        atomicOr(&hi[(size_t)seg * SEL_STRIDE + og / HUFF_GROUP], 1ull << (og % HUFF_GROUP));
        any_hi[seg] = 1;
      }
      stage[o++] = (u8)sy;
      atomicAdd(&hist[sy], 1u);
    }
  }
#undef R2_RANK
  __syncthreads();
  {
    const u32 last = first + tot_off;
    u8* ag = a + (pl.x - first);  // 16-byte aligned: the slot base is, and (pl.x - first) is a multiple of 16 symbols
    for (u32 c16 = tid * 16u; c16 < last; c16 += R2_THREADS * 16u) {
      if (c16 >= first && c16 + 16u <= last) {
        *reinterpret_cast<uint4*>(ag + c16) = *reinterpret_cast<const uint4*>(stage + c16);
      } else {
        const u32 e = min(c16 + 16u, last);
        for (u32 x = max(c16, first); x < e; x++) ag[x] = stage[x];
      }
    }
  }
  for (u32 i = tid; i < HUFF_MAXSYM; i += R2_THREADS)
    if (hist[i]) atomicAdd(&freq[(size_t)seg * HUFF_MAXSYM + i], hist[i]);
}

void mtf_rle2_batch(Ctx& c, const u8* d_T, const u8* d_U, const u32* d_n, const u32* h_n, u32 nblk, const NarrowSyms& sym, u32* d_m,
                    u32* d_freq, u32* d_used, const u32* d_bytehist) {
  (void)d_T;
  u32 n_max = 0;
  for (u32 b = 0; b < nblk; b++) n_max = h_n[b] > n_max ? h_n[b] : n_max;
  if (n_max == 0) return;
  const u32 utiles = (n_max + 256 * 64 - 1) / (256 * 64);
  CUDA_CHECK(cudaMemsetAsync(d_used, 0, (size_t)nblk * 8 * 4, c.stream));
  CUDA_CHECK(cudaMemsetAsync(d_freq, 0, (size_t)nblk * HUFF_MAXSYM * 4, c.stream));
  CUDA_CHECK(cudaMemsetAsync(d_m, 0, (size_t)nblk * 4, c.stream));
  k_clear_hi<<<nblk, 256, 0, c.stream>>>(sym.any_hi, sym.hi);
  KLAUNCH(c); KCHECK();
  CUDA_CHECK(cudaMemsetAsync(sym.any_hi, 0, (size_t)nblk * 4, c.stream));
  if (d_bytehist) k_used_from_hist<<<nblk, 256, 0, c.stream>>>(d_bytehist, d_used);  // the BWT column is a permutation of the block
  else k_used<<<utiles * nblk, 256, 0, c.stream>>>(d_U, d_n, utiles, d_used);
  KLAUNCH(c); KCHECK();
  const u32 cps = (n_max + MTF_CHUNK - 1) / MTF_CHUNK;
  DBuf<u32> lastpos(c, (size_t)nblk * cps * 256);
  DBuf<u8> R(c, (size_t)nblk << SEG_SHIFT);
  DBuf<uint4> rsum(c, (size_t)nblk * cps);
  DBuf<uint2> plan(c, (size_t)nblk * cps);
  k_mtf_lastpos<<<(cps * nblk + LP_WARPS - 1) / LP_WARPS, LP_WARPS * 32, 0, c.stream>>>(d_U, d_n, cps, cps * nblk, lastpos);
  KLAUNCH(c); KCHECK();
  k_mtf_prefix<<<nblk, 256, 0, c.stream>>>(d_n, cps, lastpos);
  KLAUNCH(c); KCHECK();
  {
    const u32 chunks = cps * nblk;
    k_mtf_ranks<<<(chunks + MR_WARPS - 1) / MR_WARPS, MR_WARPS * 32, 0, c.stream>>>(d_U, d_n, cps, lastpos, d_used, R, nblk, rsum);
    KLAUNCH(c); KCHECK();
  }
  k_rle2_scan<<<nblk, 32, 0, c.stream>>>(rsum, d_n, cps, d_used, plan, sym.lo, sym.hi, sym.any_hi, d_m, d_freq);
  KLAUNCH(c); KCHECK();
  static_assert(R2_TILE == MTF_CHUNK, "one zero-run tile per MTF chunk");
  k_rle2<<<cps * nblk, R2_THREADS, 0, c.stream>>>(R, d_n, cps, plan, sym.lo, sym.hi, sym.any_hi, d_freq);
  KLAUNCH(c); KCHECK();
}
