// bwt_msd.cu -- forward cyclic BWT for batches whose short prefixes rarely collide (near-uniform data such as
// BASELINE config 2): ONE most-significant-digit pass over HBM + a shared-memory sort of every (block, first byte)
// bucket, instead of four least-significant-digit passes (radix.cuh).
//
//   k_byte_hist (bwt.cu)   block byte histograms = bucket sizes
//   k_msd_prep             bucket offsets, dense symbol ranks, the scale that spreads 4-symbol keys over 32 bits
//   k_msd_scatter          text tile -> records (key32 = symbols 1..4 of the rotation as a scaled mixed-radix number,
//                          byte before the rotation, position) scattered into their first-byte bucket.  An MSD pass
//                          may be unstable, so ranks come from shared-memory atomics and bucket space from one global
//                          atomic per (tile, digit): no look-back chain, no warp match.  The tile arrives by bulk copy.
//   k_msd_bucket           persistent CTAs: the next bucket streams into shared memory by bulk copy (mbarrier) while
//                          the current one is sorted: interpolation cells (key >> 18) counted with shared-memory atomics,
//                          scanned, scattered in place, then every record ranks itself inside its cell.  The sorted
//                          order is only used to write the BWT column (the byte travels in the record) and pidx; equal
//                          keys (rotations that share 5 bytes) go to the tie list for k_resolve_direct (bwt.cu).
//
// Contract: lib/BWT.js:372-417 (bwtransform2), same result as the LSD path.  Algorithmic HBM bytes per text byte:
// 1 (histogram) + 1 + 8 (scatter) + 8 + 1 (bucket sort) = 19.
#include <cstdlib>
#include <type_traits>
#include "ctx.h"
#include "tma.cuh"
#include "bwt_msd.h"

// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_msd_prep(const u32* __restrict__ hist, u32* __restrict__ bstart, u32* __restrict__ cursor, u8* __restrict__ lut, MsdBlk* __restrict__ blk,
           uint4* __restrict__ work, u32* ctl) {
  __shared__ u32 ws[9];
  __shared__ u32 s_base;
  const u32 b = blockIdx.x, d = threadIdx.x;
  const u32 h = hist[b * 256 + d];
  u32 tot;
  const u32 ex = block_excl_add<256, u32>(h, ws, &tot);
  bstart[b * 256 + d] = ex;
  cursor[b * 256 + d] = ex;
  const u32 r = block_excl_add<256, u32>(h ? 1u : 0u, ws, &tot);  // tot = symbols in use
  lut[b * 256 + d] = (u8)r;
  if (h > MB_CAP) atomicOr(&ctl[2], 1u);  // a bucket that does not fit the shared-memory sort: LSD path for this batch
  if (d == 0) {
    const u64 a = tot, a4 = a * a * a * a;
    MsdBlk m;
    m.a = (u32)a;
    m.a2 = (u32)(a * a);
    // key * S >> 32 is strictly increasing in key as long as S >= 2^32 (a <= 255); 256 symbols: the key is the 4 raw bytes
    m.S = a4 >= (1ull << 32) ? (1ull << 32) : (a4 ? 0xffffffffffffffffull / a4 : 0ull);
    blk[b] = m;
    s_base = atomicAdd(&ctl[3], (u32)a);  // the block's non-empty buckets take consecutive entries of the work list
  }
  __syncthreads();
  if (h) work[s_base + r] = make_uint4(b * 256 + d, ex, h, 0u);  // (bucket id, first row inside the block, records)
}

// ---------------------------------------------------------------------------------------
struct MsdScatterSmem {
  __align__(16) u8 raw[16 + MSD_TILE + 16];  // raw[15] = byte before the tile, raw[16..] the tile, then 4 bytes of look-ahead
  __align__(16) u8 rk[MSD_TILE + 16];        // dense symbol ranks of raw[16..]
  u32 key[MSD_TILE];  // the staged records as two 32-bit planes: a warp's stores in digit order meet fewer bank conflicts
  u32 low[MSD_TILE];  // than 64-bit stores
  u32 cnt[256];
  int gdst[256];
  u8 lut[256];
  u32 ws[9];
  __align__(8) u64 bar;
};

__device__ __forceinline__ u32 lut4(const u8* lut, u32 w) {
  return (u32)lut[w & 0xff] | ((u32)lut[(w >> 8) & 0xff] << 8) | ((u32)lut[(w >> 16) & 0xff] << 16) | ((u32)lut[w >> 24] << 24);
}

template <int CTAS>
__global__ void __launch_bounds__(MSD_THREADS, CTAS)
k_msd_scatter(const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 tps, const u8* __restrict__ lut, const MsdBlk* __restrict__ blk,
              u32* __restrict__ cursor, u64* __restrict__ rec_out, const u32* __restrict__ ctl) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MsdScatterSmem& s = *reinterpret_cast<MsdScatterSmem*>(smem_raw);
  if (ctl[2]) return;
  const u32 b = blockIdx.x / tps, lt = blockIdx.x - b * tps;
  const u32 n = seg_n[b];
  const u32 start = lt * MSD_TILE;
  if (start >= n) return;
  const u32 count = min((u32)MSD_TILE, n - start);
  const u8* Tb = T + ((size_t)b << SEG_SHIFT);
  const u32 tid = threadIdx.x;
  if (tid == 0) {
    // the whole tile in one bulk copy (a short last tile reads on into the unused rest of the 1 MiB slot)
    mbar_init(&s.bar, 1); mbar_fence_init();
    mbar_expect_tx(&s.bar, MSD_TILE);
    bulk_g2s(s.raw + 16, Tb + start, MSD_TILE, &s.bar);
  }
  // everything else this tile needs from global memory is requested now, while the copy is in flight
  const MsdBlk mb = blk[b];
  const u8 lutv = lut[b * 256 + tid];
  u8 edge = 0;  // tid 32: the byte before the tile; tid 0..3: look-ahead of the last rotations (cyclic)
  if (tid == 32) edge = start ? Tb[start - 1] : Tb[n - 1];
  if (tid < 4) edge = Tb[(start + count + tid) % n];
  s.lut[tid] = lutv;
  s.cnt[tid] = 0;
  __syncthreads();  // also publishes the barrier initialisation to the waiting threads
  mbar_wait(&s.bar, 0);
  if (tid == 32) s.raw[15] = edge;
  if (tid < 4) s.raw[16 + count + tid] = edge;
  __syncthreads();
  const u32 a = mb.a, a2 = mb.a2, S_lo = (u32)mb.S, S_hi = (u32)(mb.S >> 32);
  // the rest twice: full tiles (all but the last of a block) carry no per-record bounds checks
  auto body = [&](auto full_c) {
  constexpr bool full = decltype(full_c)::value;
  // ---- dense ranks of the own 16 bytes, and their slots among the tile's records of the same digit (the digit is
  // the byte itself, so the tile's digit counts are known before any key is computed) ----
  const uint4 rv = *reinterpret_cast<const uint4*>(s.raw + 16 + tid * 16);
  const u32 rw[4] = {rv.x, rv.y, rv.z, rv.w};
  u32 slot[MSD_ITEMS / 2];
  {
    uint4 kv;
    kv.x = lut4(s.lut, rv.x); kv.y = lut4(s.lut, rv.y); kv.z = lut4(s.lut, rv.z); kv.w = lut4(s.lut, rv.w);
    *reinterpret_cast<uint4*>(s.rk + tid * 16) = kv;
    if (tid < 4) s.rk[count + tid] = s.lut[s.raw[16 + count + tid]];  // look-ahead ranks (same value as the owner's store, if any)
#pragma unroll
    for (int j = 0; j < MSD_ITEMS; j++) {
      const u32 d = (rw[j >> 2] >> (8 * (j & 3))) & 0xffu;
      u32 sl = 0;
      if (full || tid * MSD_ITEMS + j < count) sl = atomicAdd(&s.cnt[d], 1u);
      if (j & 1) slot[j >> 1] |= sl << 16; else slot[j >> 1] = sl;
    }
  }
  __syncthreads();
  // ---- per digit: space in the block's bucket (any order: the bucket is sorted afterwards).  The global atomic is
  // issued here and its result is first needed after the keys are computed and staged. ----
  u32 g, ex;
  {
    const u32 c = s.cnt[tid];
    u32 tot;
    ex = block_excl_add<MSD_THREADS, u32>(c, s.ws, &tot);
    g = c ? atomicAdd(&cursor[b * 256 + tid], c) : 0u;
    s.cnt[tid] = ex;
  }
  __syncthreads();
  // ---- keys, staged in digit order as two 32-bit planes (key, low word); the low word carries (byte before, digit,
  // position inside the tile) for now ----
  {
    const uint4 k0 = *reinterpret_cast<const uint4*>(s.rk + tid * 16);
    const u32 k1 = *reinterpret_cast<const u32*>(s.rk + tid * 16 + 16);
    const u32 kw[5] = {k0.x, k0.y, k0.z, k0.w, k1};
    u32 rr[20];
#pragma unroll
    for (int j = 0; j < 20; j++) rr[j] = (kw[j >> 2] >> (8 * (j & 3))) & 0xffu;
    u32 v2[19];  // two symbols starting at j
#pragma unroll
    for (int j = 1; j < 19; j++) v2[j] = rr[j] * a + rr[j + 1];
    u32 prev = s.raw[15 + tid * 16];
#pragma unroll
    for (int j = 0; j < MSD_ITEMS; j++) {
      const u32 d = (rw[j >> 2] >> (8 * (j & 3))) & 0xffu;
      if (full || tid * MSD_ITEMS + j < count) {
        const u32 k = v2[j + 1] * a2 + v2[j + 3];          // symbols j+1 .. j+4 as a base-a number
        const u32 sl = (j & 1) ? (slot[j >> 1] >> 16) : (slot[j >> 1] & 0xffffu);
        const u32 at = s.cnt[d] + sl;
        s.key[at] = k * S_hi + __umulhi(k, S_lo);           // spread over 32 bits (order preserving, injective)
        s.low[at] = (prev << SEG_SHIFT) | (d << 12) | (tid * MSD_ITEMS + j);
      }
      prev = d;
    }
  }
  s.gdst[tid] = (int)g - (int)ex;
  __syncthreads();
  u64* out = rec_out + ((size_t)b << SEG_SHIFT);
#pragma unroll
  for (int k = 0; k < MSD_ITEMS; k++) {
    const u32 p = k * MSD_THREADS + tid;
    if (full || p < count) {
      const u32 lw = s.low[p];
      const u32 low = (lw & 0x0ff00000u) | (start + (lw & 0xfffu));
      out[(int)p + s.gdst[(lw >> 12) & 0xffu]] = ((u64)s.key[p] << 32) | low;
    }
  }
  };
  if (count == MSD_TILE) body(std::true_type{}); else body(std::false_type{});
}

// ---------------------------------------------------------------------------------------
// Phase probe of k_msd_bucket, off by default (tools/msd_phases.py builds the library with -DB2_MSD_PROBE and prints
// it): thread 0 of every CTA adds the clock64() cycles from one phase boundary to the next over all of its buckets,
// and at the end adds its sums and its bucket count to g_msd_probe.  A boundary is where thread 0 leaves a barrier, so a
// phase's cycles are those of the CTA's slowest warp in it.  The sums live in shared memory, not in registers, so the
// probe build keeps the default build's registers and does not spill.
#define MB_PHASES 6  // wait for the bucket, histogram, scan + queue, scatter, ordering, write-out
#ifdef B2_MSD_PROBE
__device__ unsigned long long g_msd_probe[MB_PHASES + 1];
#define MB_STAMP(k) do { if (tid == 0) { const long long t_ = clock64(); s.ph[k] += t_ - s.ph[MB_PHASES + 1]; s.ph[MB_PHASES + 1] = t_; } } while (0)
extern "C" __attribute__((visibility("default"))) int b2_msd_probe(unsigned long long* out) {
  // out: MB_PHASES cycle sums and the number of buckets, summed over every launch since the last call; resets them
  unsigned long long zero[MB_PHASES + 1] = {};
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, g_msd_probe, sizeof(zero)) != cudaSuccess ||
      cudaMemcpyToSymbol(g_msd_probe, zero, sizeof(zero)) != cudaSuccess) return -1;
  return MB_PHASES;
}
#else
#define MB_STAMP(k) do { } while (0)
#endif

struct MsdBucketSmem {
  __align__(16) u64 buf[2][MB_BUF];
  __align__(16) u32 cnt[MB_CELLS / 2];  // two 16-bit cell counters per word
  __align__(16) u8 outb[MB_BUF + 16];   // the bucket's slice of the BWT column, at the alignment (mod 16) it has in global memory
  u32 multi[MB_BUF / 2];                // queued cells, four lists (2, 3, 4, more records): first row | size << 16
  __align__(8) u64 ws64[MB_THREADS / 32];
  __align__(8) u64 bar[2];
  u32 w[2], M[2], off[2], st[2];
  u32 nl[4];  // queued cells of 2, 3, 4 records / of more
#ifdef B2_MSD_PROBE
  long long ph[MB_PHASES + 2];  // phase sums, buckets, clock64() at the last boundary
#endif
};

static_assert(sizeof(MsdBucketSmem) <= 227 * 1024, "bucket sort state must fit the 227 KiB of shared memory a CTA can have");


__device__ __forceinline__ u32 cell_of(u32 key) { return key >> (32 - MB_CELL_BITS); }

// K records of one cell, starting at row `lo` of the bucket: order them (odd-even transposition network), write their
// bytes to the column slice, report runs of equal keys (rotations that share their first 5 bytes) to the resolver
// (bwt.cu k_resolve_direct).
template <int K>
__device__ __forceinline__ void small_cell(const u64* __restrict__ buf, u32 lo, u8* __restrict__ ob, u32 base, u32 urow, u32* __restrict__ pidx,
                                           u32* __restrict__ tie_head, u32* __restrict__ tie_idx, u32* ctl) {
  u64 v[K];
#pragma unroll
  for (int i = 0; i < K; i++) v[i] = buf[lo + i];
#pragma unroll
  for (int round = 0; round < K; round++) {
#pragma unroll
    for (int i = round & 1; i + 1 < K; i += 2) {
      const u64 a = v[i], b = v[i + 1];
      const bool sw = a > b;
      v[i] = sw ? b : a;
      v[i + 1] = sw ? a : b;
    }
  }
  bool any_tie = false;
#pragma unroll
  for (int i = 0; i < K; i++) {
    const u32 lw = (u32)v[i];
    ob[lo + i] = (u8)(lw >> SEG_SHIFT);
    if ((lw & SEG_MASK) == 0) pidx[base >> SEG_SHIFT] = urow + lo + i;
    if (i + 1 < K) any_tie |= (u32)(v[i] >> 32) == (u32)(v[i + 1] >> 32);
  }
  if (any_tie) {
    int run0 = 0;
#pragma unroll
    for (int i = 0; i < K; i++) {
      if (i + 1 == K || (u32)(v[i + 1] >> 32) != (u32)(v[i] >> 32)) {
        const int run = i + 1 - run0;
        if (run > 1) {
          u32 t = atomicAdd(&ctl[0], (u32)run);
          const u32 head = base | (urow + lo + run0);
#pragma unroll
          for (int z = 0; z < K; z++)
            if (z >= run0 && z <= i) { tie_head[t] = head; tie_idx[t] = base | ((u32)v[z] & SEG_MASK); t++; }
        }
        run0 = i + 1;
      }
    }
  }
}

// A cell of `size` records handled by one warp: every record counts the records of the cell that sort before it (full
// 64-bit compare: key, then the unique low word), which is its row; rows of equal keys are reported as tie runs by the
// first record of the run.  rank: per-cell scratch (one u16 per record: row -> index of the record that landed there).
__device__ __forceinline__ void big_cell(const u64* __restrict__ cb, u32 size, u32 lo, u8* __restrict__ ob, u32 base, u32 urow,
                                         u32* __restrict__ pidx, u32* __restrict__ tie_head, u32* __restrict__ tie_idx, u32* ctl,
                                         u16* __restrict__ rank) {
  const u32 lane = threadIdx.x & 31u;
  for (u32 e0 = 0; e0 < size; e0 += 32) {
    const u32 e = e0 + lane;
    if (e < size) {
      const u64 x = cb[e];
      u32 less = 0;
      for (u32 q = 0; q < size; q++) less += cb[q] < x ? 1u : 0u;
      const u32 lw = (u32)x;
      ob[lo + less] = (u8)(lw >> SEG_SHIFT);
      if ((lw & SEG_MASK) == 0) pidx[base >> SEG_SHIFT] = urow + lo + less;
      rank[less] = (u16)e;
    }
  }
  __syncwarp();
  // tie runs: walk the rows in order (lane 0 only: ties are rare and short)
  if (lane == 0) {
    u32 run0 = 0;
    for (u32 r = 0; r < size; r++) {
      const u32 kr = (u32)(cb[rank[r]] >> 32);
      if (r + 1 == size || (u32)(cb[rank[r + 1]] >> 32) != kr) {
        const u32 run = r + 1 - run0;
        if (run > 1) {
          u32 t = atomicAdd(&ctl[0], run);
          const u32 head = base | (urow + lo + run0);
          for (u32 z = run0; z <= r; z++) { tie_head[t] = head; tie_idx[t] = base | ((u32)cb[rank[z]] & SEG_MASK); t++; }
        }
        run0 = r + 1;
      }
    }
  }
  __syncwarp();
}

// Exclusive add scan over the CTA's 1024 threads with ONE barrier: every warp publishes its total, then every warp scans
// the 32 totals itself.  `ws` (32 entries) is not reused before the next barrier of the caller.
__device__ __forceinline__ u64 scan_excl_1barrier(u64 v, u64* ws, u64* total) {
  static_assert(MB_THREADS == 1024, "one lane per warp total");
  const u64 inc = warp_incl_add(v);
  const u32 w = threadIdx.x >> 5, l = threadIdx.x & 31u;
  if (l == 31) ws[w] = inc;
  __syncthreads();
  const u64 x = ws[l];
  const u64 xi = warp_incl_add(x);
  const u64 before = __shfl_sync(FULL_MASK, xi - x, (int)w);
  *total = __shfl_sync(FULL_MASK, xi, 31);
  return before + inc - v;
}

__global__ void __launch_bounds__(MB_THREADS, 1)
k_msd_bucket(const u64* __restrict__ rec, const uint4* __restrict__ work, u8* __restrict__ U, u32* __restrict__ pidx,
             u32* __restrict__ tie_head, u32* __restrict__ tie_idx, u32* ctl) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MsdBucketSmem& s = *reinterpret_cast<MsdBucketSmem*>(smem_raw);
  if (ctl[2]) return;
  const u32 tid = threadIdx.x;
  const u32 nw = ctl[3];
  // Thread 0 is the producer.  Work descriptors are fetched one round ahead of their use, so that the only global
  // latency on its path is already covered when the bulk copy of the next bucket is issued.
  auto issue = [&](u32 i, uint4 d) {
    const u32 w = d.x, st = d.y, M = d.z, off = st & 1u;
    s.w[i] = w; s.M[i] = M; s.off[i] = off; s.st[i] = st;
    if (!M) return;  // end of this CTA's list
    const u32 recs = (M + off + 1u) & ~1u;  // 16-byte granules: at most one foreign record on each side
    mbar_expect_tx(&s.bar[i], recs * 8u);
    bulk_g2s(s.buf[i], rec + (((size_t)(w >> 8)) << SEG_SHIFT) + (st - off), recs * 8u, &s.bar[i]);
  };
  uint4 dnext = make_uint4(0, 0, 0, 0);
  u32 inext = blockIdx.x + gridDim.x;
  if (tid == 0) {
    mbar_init(&s.bar[0], 1); mbar_init(&s.bar[1], 1); mbar_fence_init();
    issue(0, blockIdx.x < nw ? work[blockIdx.x] : dnext);
    if (inext < nw) dnext = work[inext];
  }
  auto clear_cells = [&]() {
    const uint4 z = make_uint4(0, 0, 0, 0);
    uint4* c4 = reinterpret_cast<uint4*>(s.cnt);
#pragma unroll
    for (u32 k = 0; k < MB_CELLS / 8 / MB_THREADS; k++) c4[tid + k * MB_THREADS] = z;
  };
  clear_cells();
  __syncthreads();
#ifdef B2_MSD_PROBE
  if (tid == 0) {
    for (int k = 0; k <= MB_PHASES; k++) s.ph[k] = 0;
    s.ph[MB_PHASES + 1] = clock64();
  }
#endif
  for (u32 it = 0;; it++) {
    const u32 i = it & 1u;
    if (s.M[i] == 0) break;
    const u32 w = s.w[i];
    if (tid == 0) {  // the other buffer was released by the barrier that ended the last round
      issue(i ^ 1u, dnext);
      inext += gridDim.x;
      dnext = inext < nw ? work[inext] : make_uint4(0, 0, 0, 0);
    }
    const u32 M = s.M[i], off = s.off[i], ust = s.st[i], blockb = w >> 8;
    u64* buf = s.buf[i];
    mbar_wait(&s.bar[i], (it >> 1) & 1u);
    u64 r[MB_ITEMS];
#pragma unroll
    for (int k = 0; k < MB_ITEMS; k++) {
      const u32 p = tid + k * MB_THREADS;
      r[k] = p < M ? buf[off + p] : 0ull;
    }
    MB_STAMP(0);
    // ---- cell histogram (the counters were cleared behind the barrier that ended the last round) ----
#pragma unroll
    for (int k = 0; k < MB_ITEMS; k++) {
      const u32 p = tid + k * MB_THREADS;
      if (p < M) {
        const u32 c = cell_of((u32)(r[k] >> 32));
        atomicAdd(&s.cnt[c >> 1], 1u << ((c & 1u) * 16u));
      }
    }
    __syncthreads();
    MB_STAMP(1);
    // ---- exclusive scan of the cell counts (each thread owns 8 words = 16 cells, two 16-bit counts per word, handled
    // two at a time without branches: counts are < 2^14, so "count >= k" is bit 15 of count + (0x8000 - k) in both halves
    // at once).  Cells of one record are flagged (bit 15 of their start): their record is final when it is scattered.
    // Cells of 2, 3, 4 and of more records are queued in four lists for the ordering passes. ----
    u8* ob = s.outb + (ust & 15u);
    {
      uint4* c4 = reinterpret_cast<uint4*>(s.cnt) + tid * 2;
      uint4 x0 = c4[0], x1 = c4[1];
      u32 wv[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
      const u32 H = 0x00010001u;
      u32 sum = 0, a2 = 0, a3 = 0, a4 = 0, a5 = 0, mm = 0;  // a_k: cells with >= k records, per half; mm: bit k / 16 + k = cell of word k queued
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const u32 w = wv[k];
        sum += (w & 0xffffu) + (w >> 16);
        const u32 ge2 = ((w + 0x7ffe7ffeu) >> 15) & H;
        a2 += ge2;
        a3 += ((w + 0x7ffd7ffdu) >> 15) & H;
        a4 += ((w + 0x7ffc7ffcu) >> 15) & H;
        a5 += ((w + 0x7ffb7ffbu) >> 15) & H;
        mm |= ge2 << k;
      }
      const u32 g2 = (a2 & 0xffffu) + (a2 >> 16), g3 = (a3 & 0xffffu) + (a3 >> 16), g4 = (a4 & 0xffffu) + (a4 >> 16), g5 = (a5 & 0xffffu) + (a5 >> 16);
      // records | cells of 2 << 14 | cells of 3 << 27 | cells of 4 << 39 | larger cells << 51
      u64 tot;
      const u64 ex = scan_excl_1barrier((u64)sum | ((u64)(g2 - g3) << 14) | ((u64)(g3 - g4) << 27) | ((u64)(g4 - g5) << 39) | ((u64)g5 << 51),
                                        s.ws64, &tot);
      const u32 t2 = (u32)(tot >> 14) & 0x1fffu, t3 = (u32)(tot >> 27) & 0xfffu, t4 = (u32)(tot >> 39) & 0xfffu, tN = (u32)(tot >> 51);
      if (tid == 0) { s.nl[0] = t2; s.nl[1] = t3; s.nl[2] = t4; s.nl[3] = tN; }
      u32 run = (u32)ex & 0x3fffu;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const u32 w = wv[k];
        const u32 s1 = run + (w & 0xffffu);
        // exactly one record: >= 1 and not >= 2
        const u32 one = (((w + 0x7fff7fffu) >> 15) & H) & ~((w + 0x7ffe7ffeu) >> 15);
        wv[k] = (run | (s1 << 16)) | (one << 15);
        run = s1 + (w >> 16);
      }
      c4[0] = make_uint4(wv[0], wv[1], wv[2], wv[3]);
      c4[1] = make_uint4(wv[4], wv[5], wv[6], wv[7]);
      __syncwarp();  // the starts are read back below through a differently typed pointer: keep the order
      // queue the own cells that hold two or more records (two on average); starts are read back from shared memory
      u32 i2 = (u32)(ex >> 14) & 0x1fffu, i3 = t2 + ((u32)(ex >> 27) & 0xfffu), i4 = t2 + t3 + ((u32)(ex >> 39) & 0xfffu),
          iN = t2 + t3 + t4 + (u32)(ex >> 51);
      const u16* cst = reinterpret_cast<const u16*>(s.cnt) + tid * 16;
      while (mm) {
        const u32 b = __ffs(mm) - 1;
        mm &= mm - 1;
        const u32 c = 2 * (b & 15u) + (b >> 4);          // cell inside the thread's 16
        const u32 st = cst[c] & 0x3fffu;
        const u32 nx = c == 15 ? run : (cst[c + 1] & 0x3fffu);
        const u32 size = nx - st;
        const u32 at = size == 2 ? i2++ : (size == 3 ? i3++ : (size == 4 ? i4++ : iN++));
        s.multi[at] = st | (size << 16);
      }
    }
    __syncthreads();
    MB_STAMP(2);
    // ---- scatter (every record of the bucket sits in a register by now).  A record alone in its cell is final: its
    // byte goes straight to the column slice; the others are stored in cell order for the ordering passes. ----
#pragma unroll
    for (int k = 0; k < MB_ITEMS; k++) {
      const u32 p = tid + k * MB_THREADS;
      if (p < M) {
        const u32 c = cell_of((u32)(r[k] >> 32));
        const u32 sh = (c & 1u) * 16u;
        const u32 half = (atomicAdd(&s.cnt[c >> 1], 1u << sh) >> sh) & 0xffffu;
        const u32 pos = half & 0x7fffu;
        if (half & 0x8000u) {
          const u32 lw = (u32)r[k];
          ob[pos] = (u8)(lw >> SEG_SHIFT);
          if ((lw & SEG_MASK) == 0) pidx[blockb] = ust + pos;
        } else {
          buf[pos] = r[k];
        }
      }
    }
    __syncthreads();
    MB_STAMP(3);
    // ---- ordering passes.  Cells of 2, 3 and 4 records: one thread per cell, a fixed compare-exchange network in
    // registers (the rarer sizes go to the high thread numbers so that no warp collects all the long jobs); larger cells
    // (a handful per bucket on uniform data, the rule on skewed data): one WARP per cell, every lane ranks its records
    // by counting. ----
    {
      const u32 n2 = s.nl[0], n3 = s.nl[1], n4 = s.nl[2], nN = s.nl[3];
      const u32 base = (blockb << SEG_SHIFT), urow = ust;
      const u32 rt = MB_THREADS - 1 - tid;
      for (u32 j = rt >> 5; j < nN; j += MB_THREADS / 32) {
        const u32 mmv = s.multi[n2 + n3 + n4 + j], lo = mmv & 0xffffu, size = mmv >> 16;
        if (size > MB_MAXCELL) { if ((tid & 31u) == 0) atomicOr(&ctl[1], 1u); continue; }  // far from uniform after all: the LSD path redoes the batch
        big_cell(buf + lo, size, lo, ob, base, urow, pidx, tie_head, tie_idx, ctl, reinterpret_cast<u16*>(s.cnt) + lo);  // the cell counters are free by now
      }
      for (u32 j = rt; j < n4; j += MB_THREADS) small_cell<4>(buf, s.multi[n2 + n3 + j] & 0xffffu, ob, base, urow, pidx, tie_head, tie_idx, ctl);
      for (u32 j = (tid + MB_THREADS / 2) & (MB_THREADS - 1); j < n3; j += MB_THREADS)
        small_cell<3>(buf, s.multi[n2 + j] & 0xffffu, ob, base, urow, pidx, tie_head, tie_idx, ctl);
      for (u32 j = tid; j < n2; j += MB_THREADS) small_cell<2>(buf, s.multi[j] & 0xffffu, ob, base, urow, pidx, tie_head, tie_idx, ctl);
    }
    __syncthreads();
    MB_STAMP(4);
    // ---- the column slice goes out in 16-byte pieces ----
    {
      const u32 first = ust & 15u, last = first + M;
      u8* Ug = U + ((size_t)blockb << SEG_SHIFT) + (ust - first);  // 16-byte aligned
      for (u32 c16 = tid * 16u; c16 < last; c16 += MB_THREADS * 16u) {
        if (c16 >= first && c16 + 16u <= last) {
          *reinterpret_cast<uint4*>(Ug + c16) = *reinterpret_cast<const uint4*>(s.outb + c16);
        } else {
          const u32 e = min(c16 + 16u, last);
          for (u32 x = max(c16, first); x < e; x++) Ug[x] = s.outb[x];
        }
      }
    }
    clear_cells();       // the ordering passes are done with their scratch in the counters
    fence_async_smem();  // the generic-proxy writes to this buffer are ordered before the bulk copy that refills it
    __syncthreads();
    MB_STAMP(5);
#ifdef B2_MSD_PROBE
    if (tid == 0) s.ph[MB_PHASES]++;
#endif
  }
#ifdef B2_MSD_PROBE
  if (tid == 0)
    for (int k = 0; k <= MB_PHASES; k++) atomicAdd(&g_msd_probe[k], (unsigned long long)s.ph[k]);
#endif
}

// ---------------------------------------------------------------------------------------
void bwt_msd_launch(Ctx& c, const u8* d_T, u8* d_U, const u32* d_n, u32 nblk, u32 n_max, u64 n_total, const u32* d_hist, u64* d_rec,
                    u32* d_pidx, u32* d_tie_head, u32* d_tie_idx, u32* d_ctl) {
  static int sms = 0, scatter_ctas = MSD_CTAS_PER_SM;
  if (!sms) {
    CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device));
    CUDA_CHECK(cudaFuncSetAttribute(k_msd_scatter<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MsdScatterSmem)));
    CUDA_CHECK(cudaFuncSetAttribute(k_msd_scatter<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MsdScatterSmem)));
    if (const char* e = getenv("B2_MSD_CTAS")) scatter_ctas = atoi(e) == 4 ? 4 : 5;  // tuning knob: registers (64 vs 48) against occupancy
    CUDA_CHECK(cudaFuncSetAttribute(k_msd_bucket, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MsdBucketSmem)));
  }
  DBuf<u32> bstart(c, (size_t)nblk * 256), cursor(c, (size_t)nblk * 256);
  DBuf<u8> lut(c, (size_t)nblk * 256);
  DBuf<MsdBlk> blk(c, nblk);
  DBuf<uint4> work(c, (size_t)nblk * 256);
  k_msd_prep<<<nblk, 256, 0, c.stream>>>(d_hist, bstart, cursor, lut, blk, work, d_ctl);
  KLAUNCH(c); KCHECK();
  const u32 tps = (n_max + MSD_TILE - 1) / MSD_TILE;
  {
    size_t ev = c.begin(ST_MSD_SCATTER);
    if (scatter_ctas == 4) k_msd_scatter<4><<<tps * nblk, MSD_THREADS, sizeof(MsdScatterSmem), c.stream>>>(d_T, d_n, tps, lut, blk, cursor, d_rec, d_ctl);
    else k_msd_scatter<5><<<tps * nblk, MSD_THREADS, sizeof(MsdScatterSmem), c.stream>>>(d_T, d_n, tps, lut, blk, cursor, d_rec, d_ctl);
    c.end(ev);
    KLAUNCH(c); KCHECK();
    ev = c.begin(ST_MSD_BUCKET);
    k_msd_bucket<<<(unsigned)sms, MB_THREADS, sizeof(MsdBucketSmem), c.stream>>>(d_rec, work, d_U, d_pidx, d_tie_head, d_tie_idx, d_ctl);
    c.end(ev);
    KLAUNCH(c); KCHECK();
  }
  c.stats.msd_launches++;
  c.stats.msd_scatter_bytes += n_total * 9;  // text in, records out
  c.stats.msd_bucket_bytes += n_total * 9;   // records in, column out
  c.stats.bwt_bytes += n_total * 18;
}
