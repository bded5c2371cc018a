// bwt.cu -- batched forward cyclic Burrows-Wheeler transform on the GPU.
//
// Replaces lib/BWT.js:372-417 (BWT.bwtransform2: SA-IS over the doubled block, one block
// at a time) with a segmented prefix-doubling suffix sort over MANY bzip2 blocks at once:
//
//   1. key32[g] = first 4 bytes of rotation g (cyclic), g = block<<20 | i
//   2. segmented LSD radix sort of (key32, g) per block           (radix.cuh, 4 passes)
//   3. k_rerank<INIT>: group heads -> rank[g], SA, compact the suffixes whose group is
//      not yet a singleton into (head, g) records
//   4. rounds h = 4, 8, 16, ...: for the still-unsorted suffixes only
//        key64 = head << 20 | rank[(i+h) mod n]   (k_gather)
//        flat radix sort of (key64, g)           (radix.cuh)
//        k_rerank<ROUND>: scatter back into SA[head + j], refine ranks, re-compact
//      until nothing is left or h >= n (then the remaining ties are equal rotations of a
//      periodic block, ordered by DESCENDING start index -- what sorting the doubled
//      string yields in the reference, SURVEY.md 3.5)
//   5. k_emit: U[p] = T[SA[p]-1], pidx = row of rotation 0
//
// All arrays use the slot layout g = block << 20 | position (max block 900000 < 2^20).
#include "ctx.h"
#include "radix.cuh"
#include "radix_host.cuh"
#include "bwt_msd.h"

// ---------------------------------------------------------------------------------------
// key32 = first four bytes of every rotation; hist[b][256] = byte histogram of block b (which is the
// digit histogram of EVERY pass of the 4-byte-prefix sort, because each text byte is the k-th byte of
// exactly one rotation).
#define BK_THREADS 256
#define BK_ITEMS 16
__global__ void __launch_bounds__(BK_THREADS)
k_build_keys(const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 tps, u64* __restrict__ rec, u32* __restrict__ hist, u32 koff, int sentinel) {
  __shared__ u32 h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const u32 b = blockIdx.x / tps, lt = blockIdx.x % tps;
  const u32 n = seg_n[b];
  const u32 start = lt * (BK_THREADS * BK_ITEMS);
  if (start >= n) return;
  const u8* t = T + ((size_t)b << SEG_SHIFT);
  u64* ko = rec + ((size_t)b << SEG_SHIFT);
#pragma unroll 4
  for (int k = 0; k < BK_ITEMS; k++) {
    const u32 i = start + k * BK_THREADS + threadIdx.x;
    if (i < n) {
      if (sentinel) {
        // suffixes, not rotations (lib/BWT.js:305-321): past the end the key is padded with zeros; a suffix that
        // ends inside its key ties with longer ones and is placed first by the rounds (its successor ranks 0)
        const u32 c0 = t[i], c1 = i + 1 < n ? t[i + 1] : 0u, c2 = i + 2 < n ? t[i + 2] : 0u, c3 = i + 3 < n ? t[i + 3] : 0u;
        ko[i] = ((u64)((c0 << 24) | (c1 << 16) | (c2 << 8) | c3) << 32) | (((u32)t[i ? i - 1 : n - 1] << SEG_SHIFT) | i);
        continue;
      }
      u32 i0 = i + koff; if (i0 >= n) i0 %= n;
      u32 i1 = i0 + 1; if (i1 >= n) i1 -= n;
      u32 i2 = i1 + 1; if (i2 >= n) i2 -= n;
      u32 i3 = i2 + 1; if (i3 >= n) i3 -= n;
      const u32 c0 = t[i0];
      // low word: the byte BEFORE the rotation (its BWT output, so the emit pass needs no gather) and its position;
      // the block is implied by the slot the record sits in (the sort never moves a record out of its segment)
      ko[i] = ((u64)((c0 << 24) | ((u32)t[i1] << 16) | ((u32)t[i2] << 8) | (u32)t[i3]) << 32) | (((u32)t[i ? i - 1 : n - 1] << SEG_SHIFT) | i);
      if (hist) atomicAdd(&h[c0], 1u);
    }
  }
  __syncthreads();
  if (hist && h[threadIdx.x]) atomicAdd(&hist[b * 256 + threadIdx.x], h[threadIdx.x]);
}

// Block byte histograms (bucket sizes of the MSD path, digit histogram of every LSD pass, text score): 16-byte loads,
// one private set of counters per warp.  Tiles are BH_TILE bytes of one block.
#define BH_TILE 16384
__global__ void __launch_bounds__(BK_THREADS) k_byte_hist(const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 tps, u32* __restrict__ hist) {
  __shared__ u32 h[BK_THREADS / 32][256];
  const u32 tid = threadIdx.x, w = tid >> 5;
#pragma unroll
  for (int k = 0; k < BK_THREADS / 32; k++) h[k][tid] = 0;
  __syncthreads();
  const u32 b = blockIdx.x / tps, lt = blockIdx.x % tps;
  const u32 n = seg_n[b];
  const u32 start = lt * BH_TILE;
  if (start >= n) return;
  const u8* t = T + ((size_t)b << SEG_SHIFT) + start;
  const u32 cnt = min((u32)BH_TILE, n - start);
#pragma unroll
  for (int k = 0; k < BH_TILE / 16 / BK_THREADS; k++) {
    const u32 o = (k * BK_THREADS + tid) * 16;
    if (o + 16 <= cnt) {
      const uint4 v = *reinterpret_cast<const uint4*>(t + o);
      const u32 wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; q++) {
        atomicAdd(&h[w][wv[q] & 0xff], 1u); atomicAdd(&h[w][(wv[q] >> 8) & 0xff], 1u);
        atomicAdd(&h[w][(wv[q] >> 16) & 0xff], 1u); atomicAdd(&h[w][wv[q] >> 24], 1u);
      }
    } else {
      for (u32 x = o; x < cnt; x++) atomicAdd(&h[w][t[x]], 1u);
    }
  }
  __syncthreads();
  u32 tot = 0;
#pragma unroll
  for (int k = 0; k < BK_THREADS / 32; k++) tot += h[k][tid];
  if (tot) atomicAdd(&hist[b * 256 + tid], tot);
}
// four bytes of block text starting at (i + off) mod n, big endian
__device__ __forceinline__ u32 word_at(const u8* __restrict__ t, u32 n, u32 i, u32 off) {
  u32 i0 = i + off; if (i0 >= n) i0 %= n;
  u32 i1 = i0 + 1; if (i1 >= n) i1 -= n;
  u32 i2 = i1 + 1; if (i2 >= n) i2 -= n;
  u32 i3 = i2 + 1; if (i3 >= n) i3 -= n;
  return ((u32)t[i0] << 24) | ((u32)t[i1] << 16) | ((u32)t[i2] << 8) | (u32)t[i3];
}
// 8-byte mode, between the two 4-pass sorts: the records are ordered by bytes 4..7; re-key them with
// bytes 0..3 (the stable second sort then yields the order by the first 8 bytes).
__global__ void k_rekey(const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 nslots, u64* __restrict__ rec) {
  const u32 g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nslots) return;
  const u32 b = g >> SEG_SHIFT, n = seg_n[b];
  if ((g & SEG_MASK) >= n) return;
  const u32 idx = (u32)rec[g];
  rec[g] = ((u64)word_at(T + ((size_t)b << SEG_SHIFT), n, idx & SEG_MASK, 0) << 32) | idx;
}
// text-likeness of a batch from its byte histograms: expected number of 4-byte-prefix collisions per
// suffix, n * (sum p_c^2)^4, averaged over the blocks (0.01 for uniform ASCII, >> 1 for text)
__global__ void k_text_score(const u32* __restrict__ hist, const u32* __restrict__ seg_n, u32 nblk, float* __restrict__ score) {
  __shared__ float acc[256];
  float a = 0.f;
  for (u32 b = threadIdx.x; b < nblk; b += blockDim.x) {
    const float n = (float)seg_n[b];
    if (n < 1.f) continue;
    float s2 = 0.f;
    for (u32 c = 0; c < 256; c++) { const float p = (float)hist[b * 256 + c] / n; s2 += p * p; }
    a += n * s2 * s2 * s2 * s2;
  }
  acc[threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (u32 i = 0; i < blockDim.x; i++) t += acc[i]; *score = t / (float)nblk; }
}

// ---------------------------------------------------------------------------------------
#define RR_THREADS 256
#define RR_ITEMS 8
#define RR_TILE (RR_THREADS * RR_ITEMS)

// Exclusive max over the threads before this one (0 when none). ws: RR_THREADS/32+1 entries.
__device__ __forceinline__ u32 block_excl_max_u32(u32 v, u32* ws, u32* total) {
  u32 inc = warp_incl_max(v);
  u32 exw = __shfl_up_sync(FULL_MASK, inc, 1);
  if (lane_id() == 0) exw = 0;
  const int w = threadIdx.x >> 5;
  if (lane_id() == 31) ws[w] = inc;
  __syncthreads();
  if (w == 0) {
    u32 x = (lane_id() < RR_THREADS / 32) ? ws[lane_id()] : 0u;
    u32 xi = warp_incl_max(x);
    u32 xe = __shfl_up_sync(FULL_MASK, xi, 1);
    if (lane_id() == 0) xe = 0;
    if (lane_id() < RR_THREADS / 32) ws[lane_id()] = xe;
    if (lane_id() == RR_THREADS / 32 - 1) ws[RR_THREADS / 32] = xi;
  }
  __syncthreads();
  u32 c = ws[w];
  *total = ws[RR_THREADS / 32];
  __syncthreads();
  return exw > c ? exw : c;
}

// One kernel for both "after the initial sort" (INIT: records live in the slot layout, key =
// 4-byte prefix, every block is one old group) and "after a doubling round" (records are the
// flat sorted (key64 = head<<20|r2, g) array).
template <bool INIT>
__global__ void __launch_bounds__(RR_THREADS)
k_rerank(const u32* __restrict__ key32, const u64* __restrict__ key64, const u32* __restrict__ vals,
         const u32* __restrict__ seg_n, u32 total, u32* __restrict__ SA, u32* __restrict__ rank,
         u32* __restrict__ next_head, u32* __restrict__ next_idx, u32* next_count, u32* ticket, u64* st_first,
         u64* st_new, u64* st_cnt, u32 ntiles) {
  __shared__ u64 sk[RR_TILE + 2];      // composite keys, sk[0] = predecessor of the tile, sk[TILE+1] = successor
  __shared__ u8 sv[RR_TILE + 2];       // validity of the same
  __shared__ u32 ws[RR_THREADS / 32 + 1];
  __shared__ u32 s_tile, s_cf, s_cn, s_cc;
  const u32 tid = threadIdx.x;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 tile = s_tile;
  const u32 q0 = tile * RR_TILE;
  // ---- stage composite keys (with a halo of one on each side) ----
  for (u32 j = tid; j < RR_TILE + 2; j += RR_THREADS) {
    long long q = (long long)q0 + (long long)j - 1;
    u64 ck = 0; u8 v = 0;
    if (q >= 0 && q < (long long)total) {
      if (INIT) {
        u32 b = (u32)q >> SEG_SHIFT, i = (u32)q & SEG_MASK;
        if (i < seg_n[b]) { v = 1; ck = ((u64)(b + 1) << 32) | key32[q]; }
      } else {
        v = 1; ck = key64[q];
      }
    }
    sk[j] = ck; sv[j] = v;
  }
  __syncthreads();
  // ---- per item flags ----
  u32 vf[RR_ITEMS], vn[RR_ITEMS], nc[RR_ITEMS];
  u32 mf = 0, mn = 0, cs = 0;
#pragma unroll
  for (int j = 0; j < RR_ITEMS; j++) {
    const u32 l = tid * RR_ITEMS + j + 1;  // index into sk
    const u32 q = q0 + tid * RR_ITEMS + j;
    const bool valid = sv[l];
    const u64 ck = sk[l];
    bool hc, nh, single;
    if (INIT) {
      hc = (q & SEG_MASK) == 0;
      nh = !sv[l - 1] || sk[l - 1] != ck;
    } else {
      hc = !sv[l - 1] || (sk[l - 1] >> SEG_SHIFT) != (ck >> SEG_SHIFT);
      nh = !sv[l - 1] || sk[l - 1] != ck;
    }
    single = nh && (!sv[l + 1] || sk[l + 1] != ck);
    vf[j] = (valid && hc) ? q + 1 : 0;
    vn[j] = (valid && nh) ? q + 1 : 0;
    nc[j] = (valid && !single) ? 1u : 0u;
    mf = max(mf, vf[j]); mn = max(mn, vn[j]); cs += nc[j];
  }
  // ---- block scans of the thread aggregates ----
  u32 tot_f, tot_n, tot_c;
  u32 ex_f = block_excl_max_u32(mf, ws, &tot_f);
  u32 ex_n = block_excl_max_u32(mn, ws, &tot_n);
  u32 ex_c = block_excl_add<RR_THREADS, u32>(cs, ws, &tot_c);
  // ---- chained scans across tiles: warps 0,1,2 each run one look-back ----
  {
    const u32 w = tid >> 5;
    if (w == 0) { u32 r = lookback_warp(st_first, tile, tot_f, OpMax()); if (lane_id() == 0) s_cf = r; }
    else if (w == 1) { u32 r = lookback_warp(st_new, tile, tot_n, OpMax()); if (lane_id() == 0) s_cn = r; }
    else if (w == 2) { u32 r = lookback_warp(st_cnt, tile, tot_c, OpAdd()); if (lane_id() == 0) s_cc = r; }
  }
  __syncthreads();
  u32 run_f = max(s_cf, ex_f), run_n = max(s_cn, ex_n), run_c = s_cc + ex_c;
  if (tile == ntiles - 1 && tid == 0) *next_count = s_cc + tot_c;
  // ---- outputs ----
#pragma unroll
  for (int j = 0; j < RR_ITEMS; j++) {
    const u32 l = tid * RR_ITEMS + j + 1;
    const u32 q = q0 + tid * RR_ITEMS + j;
    run_f = max(run_f, vf[j]);
    run_n = max(run_n, vn[j]);
    if (sv[l]) {
      const u32 firstq = run_f - 1, lastnew = run_n - 1;
      const u32 g = vals[q];
      u32 ghead;
      if (INIT) ghead = q & ~SEG_MASK; else ghead = (u32)(sk[l] >> SEG_SHIFT);
      const u32 newhead = ghead + (lastnew - firstq);
      if (!INIT) SA[ghead + (q - firstq)] = g;  // INIT: SA is the sorted value array itself
      rank[g] = newhead & SEG_MASK;
      if (nc[j]) { next_head[run_c] = newhead; next_idx[run_c] = g; }
    }
    run_c += nc[j];
  }
}

// Specialised "after the initial sort" variant: tiles never straddle blocks, invalid slots are skipped,
// 32-bit keys staged in padded shared memory (conflict-free blocked reads).  Group head chain per
// block, compaction offsets as one flat chain over all tiles.
#define RI_PAD(j) ((j) + ((j) >> 5))
template <bool WIDE>
__global__ void __launch_bounds__(RR_THREADS)
k_rerank_init(const u64* __restrict__ rec, const u8* __restrict__ T, u32* __restrict__ SA, const u32* __restrict__ seg_n, u32 tps, u32* __restrict__ rank,
              u32* __restrict__ next_head, u32* __restrict__ next_idx, u32* next_count, u32* ticket, u64* st_new, u64* st_cnt, u32 ntiles) {
  __shared__ u32 sk[RR_TILE + RR_TILE / 32 + 2];
  __shared__ u32 sg[RR_TILE + RR_TILE / 32 + 2];
  __shared__ u32 s2[WIDE ? RR_TILE + RR_TILE / 32 + 2 : 1];   // bytes 4..7 of every suffix (8-byte mode)
  __shared__ u32 ws[RR_THREADS / 32 + 1];
  __shared__ u32 s_tile, s_cn, s_cc, s_prev, s_next, s_prev2, s_next2;
  const u32 tid = threadIdx.x;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 tile = s_tile;
  const u32 b = tile / tps, lt = tile - b * tps;
  const u32 n = seg_n[b];
  const u32 start = lt * RR_TILE;
  const u32 cnt = start < n ? min((u32)RR_TILE, n - start) : 0u;
  const size_t base = ((size_t)b << SEG_SHIFT) + start;
  for (u32 j = tid; j < cnt; j += RR_THREADS) {
    const u64 rv = rec[base + j];
    sk[RI_PAD(j)] = (u32)(rv >> 32);
    sg[RI_PAD(j)] = (u32)rv;
    SA[base + j] = (u32)rv;
    if (WIDE) s2[RI_PAD(j)] = word_at(T + ((size_t)b << SEG_SHIFT), n, (u32)rv & SEG_MASK, 4);
  }
  if (tid == 0 && cnt) {
    s_prev = start ? (u32)(rec[base - 1] >> 32) : 0u;
    s_next = (start + cnt < n) ? (u32)(rec[base + cnt] >> 32) : 0u;
    if (WIDE) {
      s_prev2 = start ? word_at(T + ((size_t)b << SEG_SHIFT), n, (u32)rec[base - 1] & SEG_MASK, 4) : 0u;
      s_next2 = (start + cnt < n) ? word_at(T + ((size_t)b << SEG_SHIFT), n, (u32)rec[base + cnt] & SEG_MASK, 4) : 0u;
    }
  }
  __syncthreads();
  u32 vn[RR_ITEMS], nc[RR_ITEMS];
  u32 mn = 0, cs = 0;
#pragma unroll
  for (int j = 0; j < RR_ITEMS; j++) {
    const u32 p = tid * RR_ITEMS + j;
    vn[j] = 0; nc[j] = 0;
    if (p < cnt) {
      const u32 k = sk[RI_PAD(p)];
      const bool hasprev = p > 0 || start > 0;
      const u32 kp = p > 0 ? sk[RI_PAD(p - 1)] : s_prev;
      const bool hasnext = (p + 1 < cnt) || (start + cnt < n);
      const u32 kn = (p + 1 < cnt) ? sk[RI_PAD(p + 1)] : s_next;
      bool eqp = kp == k, eqn = kn == k;
      if (WIDE) {
        const u32 k2 = s2[RI_PAD(p)];
        eqp = eqp && (p > 0 ? s2[RI_PAD(p - 1)] : s_prev2) == k2;
        eqn = eqn && ((p + 1 < cnt) ? s2[RI_PAD(p + 1)] : s_next2) == k2;
      }
      const bool nh = !hasprev || !eqp;
      const bool single = nh && (!hasnext || !eqn);
      vn[j] = nh ? start + p + 1 : 0u;
      nc[j] = single ? 0u : 1u;
      mn = max(mn, vn[j]); cs += nc[j];
    }
  }
  u32 tot_n, tot_c;
  const u32 ex_n = block_excl_max_u32(mn, ws, &tot_n);
  const u32 ex_c = block_excl_add<RR_THREADS, u32>(cs, ws, &tot_c);
  {
    const u32 w = tid >> 5;
    if (w == 0 && cnt) { u32 r = lookback_warp(st_new + (size_t)b * tps, lt, tot_n, OpMax()); if (lane_id() == 0) s_cn = r; }
    else if (w == 1) { u32 r = lookback_warp(st_cnt, tile, tot_c, OpAdd()); if (lane_id() == 0) s_cc = r; }
  }
  __syncthreads();
  if (tile == ntiles - 1 && tid == 0) *next_count = s_cc + tot_c;
  if (cnt == 0) return;
  u32 run_n = max(s_cn, ex_n), run_c = s_cc + ex_c;
#pragma unroll
  for (int j = 0; j < RR_ITEMS; j++) {
    const u32 p = tid * RR_ITEMS + j;
    if (p < cnt) {
      run_n = max(run_n, vn[j]);
      const u32 lastnew = run_n - 1;  // position (inside the block) of this suffix's group head
      const u32 g = (b << SEG_SHIFT) | (sg[RI_PAD(p)] & SEG_MASK);
      rank[g] = lastnew;
      if (nc[j]) { next_head[run_c] = (b << SEG_SHIFT) | lastnew; next_idx[run_c] = g; }
      run_c += nc[j];
    }
  }
}

// Sparse-tie path (batches whose 4-byte prefixes rarely collide): one pass over the sorted records emits the
// BWT column for every position AND compacts the few suffixes that still share their prefix with a neighbour
// (in sorted order, with their group head) -- no rank array, no SA.  k_resolve_direct then orders each small
// group by comparing the rotations' next bytes and rewrites the group's slice of the column.
__global__ void __launch_bounds__(RR_THREADS)
k_emit_detect(const u64* __restrict__ rec, const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 tps, u8* __restrict__ U,
              u32* __restrict__ pidx, u32* __restrict__ next_head, u32* __restrict__ next_idx, u32* next_count, u32* ticket, u64* st_new,
              u64* st_cnt, u32 ntiles) {
  __shared__ u32 sk[RR_TILE + RR_TILE / 32 + 2];
  __shared__ u32 sg[RR_TILE + RR_TILE / 32 + 2];
  __shared__ u32 ws[RR_THREADS / 32 + 1];
  __shared__ u32 s_tile, s_cn, s_cc, s_prev, s_next;
  const u32 tid = threadIdx.x;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 tile = s_tile;
  const u32 b = tile / tps, lt = tile - b * tps;
  const u32 n = seg_n[b];
  const u32 start = lt * RR_TILE;
  const u32 cnt = start < n ? min((u32)RR_TILE, n - start) : 0u;
  const size_t base = ((size_t)b << SEG_SHIFT) + start;
  for (u32 j = tid; j < cnt; j += RR_THREADS) {
    const u64 rv = rec[base + j];
    sk[RI_PAD(j)] = (u32)(rv >> 32);
    sg[RI_PAD(j)] = (u32)rv;
    U[base + j] = (u8)((u32)rv >> SEG_SHIFT);  // the byte before the rotation travels in the record
    if (((u32)rv & SEG_MASK) == 0) pidx[b] = start + j;
  }
  if (tid == 0 && cnt) {
    s_prev = start ? (u32)(rec[base - 1] >> 32) : 0u;
    s_next = (start + cnt < n) ? (u32)(rec[base + cnt] >> 32) : 0u;
  }
  __syncthreads();
  u32 vn[RR_ITEMS], nc[RR_ITEMS];
  u32 mn = 0, cs = 0;
#pragma unroll
  for (int j = 0; j < RR_ITEMS; j++) {
    const u32 p = tid * RR_ITEMS + j;
    vn[j] = 0; nc[j] = 0;
    if (p < cnt) {
      const u32 k = sk[RI_PAD(p)];
      const bool hasprev = p > 0 || start > 0;
      const u32 kp = p > 0 ? sk[RI_PAD(p - 1)] : s_prev;
      const bool hasnext = (p + 1 < cnt) || (start + cnt < n);
      const u32 kn = (p + 1 < cnt) ? sk[RI_PAD(p + 1)] : s_next;
      const bool nh = !hasprev || kp != k;
      const bool single = nh && (!hasnext || kn != k);
      vn[j] = nh ? start + p + 1 : 0u;
      nc[j] = single ? 0u : 1u;
      mn = max(mn, vn[j]); cs += nc[j];
    }
  }
  u32 tot_n, tot_c;
  const u32 ex_n = block_excl_max_u32(mn, ws, &tot_n);
  const u32 ex_c = block_excl_add<RR_THREADS, u32>(cs, ws, &tot_c);
  {
    const u32 w = tid >> 5;
    if (w == 0 && cnt) { u32 r = lookback_warp(st_new + (size_t)b * tps, lt, tot_n, OpMax()); if (lane_id() == 0) s_cn = r; }
    else if (w == 1) { u32 r = lookback_warp(st_cnt, tile, tot_c, OpAdd()); if (lane_id() == 0) s_cc = r; }
  }
  __syncthreads();
  if (tile == ntiles - 1 && tid == 0) *next_count = s_cc + tot_c;
  if (cnt == 0) return;
  u32 run_n = max(s_cn, ex_n), run_c = s_cc + ex_c;
#pragma unroll
  for (int j = 0; j < RR_ITEMS; j++) {
    const u32 p = tid * RR_ITEMS + j;
    if (p < cnt) {
      run_n = max(run_n, vn[j]);
      if (nc[j]) { next_head[run_c] = (b << SEG_SHIFT) | (run_n - 1); next_idx[run_c] = (b << SEG_SHIFT) | (sg[RI_PAD(p)] & SEG_MASK); }
      run_c += nc[j];
    }
  }
}

#define RD_MAXGROUP 16  // larger groups and rotations equal over RD_DEPTH more bytes go to the doubling rounds
#define RD_DEPTH 64
#define RD_FAIL_GROUP 1u  // *fail bits: a group larger than RD_MAXGROUP,
#define RD_FAIL_DEPTH 2u  // two rotations equal over h0 + RD_DEPTH bytes
__global__ void k_resolve_direct(const u32* __restrict__ head, const u32* __restrict__ idx, u32 M, const u8* __restrict__ T,
                                 const u32* __restrict__ seg_n, u32 h0, u8* __restrict__ U, u32* __restrict__ pidx, u32* fail) {
  const u32 q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= M) return;
  const u32 hd = head[q];
  if (q > 0 && head[q - 1] == hd) return;  // one thread per group: its first member
  u32 mem[RD_MAXGROUP];
  u32 cnt = 0;
  while (q + cnt < M && head[q + cnt] == hd) {
    if (cnt == RD_MAXGROUP) { atomicOr(fail, RD_FAIL_GROUP); return; }
    mem[cnt] = idx[q + cnt] & SEG_MASK;
    cnt++;
  }
  const u32 b = hd >> SEG_SHIFT, n = seg_n[b];
  const u8* Tb = T + ((size_t)b << SEG_SHIFT);
  // insertion sort; rotations compare by their bytes from h0 on (the first h0 bytes are equal inside a group)
  for (u32 a = 1; a < cnt; a++) {
    const u32 x = mem[a];
    u32 pos = a;
    while (pos > 0) {
      const u32 y = mem[pos - 1];
      int less = -1;  // x < y ?
      for (u32 d = h0; d < h0 + RD_DEPTH; d += 4) {
        const u32 wx = word_at(Tb, n, x, d), wy = word_at(Tb, n, y, d);
        if (wx != wy) { less = wx < wy ? 1 : 0; break; }
      }
      if (less < 0) { atomicOr(fail, RD_FAIL_DEPTH); return; }
      if (!less) break;
      mem[pos] = y;
      pos--;
    }
    mem[pos] = x;
  }
  const u32 p0 = hd & SEG_MASK;
  for (u32 r = 0; r < cnt; r++) {
    const u32 i = mem[r];
    U[((size_t)b << SEG_SHIFT) + p0 + r] = Tb[i ? i - 1 : n - 1];
    if (i == 0) pidx[b] = p0 + r;
  }
}

// key64 = head << 20 | rank of the rotation h further on (or n-1-i for the final tie-break).
__global__ void k_gather(const u32* __restrict__ head, const u32* __restrict__ idx, u32 M, const u32* __restrict__ rank,
                         const u32* __restrict__ seg_n, u32 h, int tiebreak, u64* __restrict__ key_out, u32* __restrict__ val_out,
                         int sentinel) {
  u32 q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= M) return;
  const u32 g = idx[q];
  const u32 b = g >> SEG_SHIFT, i = g & SEG_MASK, n = seg_n[b];
  u32 r2;
  if (tiebreak) r2 = n - 1 - i;
  else if (sentinel) r2 = i + h < n ? rank[(b << SEG_SHIFT) | (i + h)] + 1 : 0u;  // the empty suffix sorts first
  else r2 = rank[(b << SEG_SHIFT) | ((i + h) % n)];
  key_out[q] = ((u64)head[q] << SEG_SHIFT) | r2;
  val_out[q] = g;
}

__global__ void k_emit(const u32* __restrict__ SA, const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 nslots,
                       u8* __restrict__ U, u32* __restrict__ pidx) {
  u32 q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nslots) return;
  const u32 b = q >> SEG_SHIFT, p = q & SEG_MASK, n = seg_n[b];
  if (p >= n) return;
  const u32 i = SA[q] & SEG_MASK;
  U[q] = T[((size_t)b << SEG_SHIFT) | (i ? i - 1 : n - 1)];
  if (i == 0) pidx[b] = p;
}

// Sentinel mode outputs: the suffix array itself (lib/BWT.js:305-321) and the BWT of lib/BWT.js:328-350:
// U[0] = T[n-1], then the characters before the suffixes in order with suffix 0 left out; pidx = its rank + 1.
__global__ void k_emit_sa(const u32* __restrict__ SA, const u32* __restrict__ seg_n, u32 nslots, u32* __restrict__ sa_out, u32* __restrict__ pidx) {
  u32 q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nslots) return;
  const u32 b = q >> SEG_SHIFT, p = q & SEG_MASK, n = seg_n[b];
  if (p >= n) return;
  const u32 i = SA[q] & SEG_MASK;
  if (sa_out) sa_out[q] = i;
  if (i == 0) pidx[b] = p + 1;
}
__global__ void k_emit_sentinel(const u32* __restrict__ SA, const u8* __restrict__ T, const u32* __restrict__ seg_n, u32 nslots,
                                const u32* __restrict__ pidx, u8* __restrict__ U) {
  u32 q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nslots) return;
  const u32 b = q >> SEG_SHIFT, p = q & SEG_MASK, n = seg_n[b];
  if (p >= n) return;
  const size_t base = (size_t)b << SEG_SHIFT;
  const u32 i = SA[q] & SEG_MASK, r0 = pidx[b] - 1;
  if (p == 0) U[base] = T[base + n - 1];
  if (i != 0) U[base + p + 1 - (p > r0 ? 1u : 0u)] = T[base + i - 1];
}

// host side: radix_sort<> lives in radix_host.cuh
// why a direct finish gave up (b2_stats.bwt_msd_fallback_why / bwt_direct_fallback_why)
enum : u32 { WHY_BUCKET = 1, WHY_CELL = 2, WHY_TIES = 4, WHY_GROUP = 8, WHY_DEPTH = 16 };
static u32 resolve_why(u32 fail) { return (fail & RD_FAIL_GROUP ? WHY_GROUP : 0u) | (fail & RD_FAIL_DEPTH ? WHY_DEPTH : 0u); }
static u32 bits_for(u32 maxval) {  // number of bits needed to represent values 0..maxval
  u32 b = 0;
  while (maxval) { b++; maxval >>= 1; }
  return b;
}

// Forward cyclic BWT of `nblk` blocks in the slot layout.  d_T/d_U: u8[nblk << 20];
// d_n: device u32[nblk]; h_n: host copy; d_pidx: device u32[nblk].
void bwt_forward_batch(Ctx& c, const u8* d_T, u8* d_U, const u32* d_n, const u32* h_n, u32 nblk, u32* d_pidx, bool sentinel, u32* d_sa_out,
                       u32* d_hist_out) {
  if (nblk == 0) return;
  u32 n_max = 0; u64 n_total = 0;
  for (u32 b = 0; b < nblk; b++) { n_max = h_n[b] > n_max ? h_n[b] : n_max; n_total += h_n[b]; }
  if (n_total == 0) return;
  const u32 nslots = nblk << SEG_SHIFT;
  DBuf<u64> recA(c, nslots), recB(c, nslots);
  DBuf<u32> saBuf(c, nslots), rank(c, nslots);
  DBuf<u32> headA(c, n_total), idxA(c, n_total), cnt(c, 4), ticket(c, 1);
  const u32 rr_tiles_init = (nslots + RR_TILE - 1) / RR_TILE;
  DBuf<u64> st(c, (size_t)3 * rr_tiles_init);
  u64 *kin = recA, *kout = recB;
  u32 *vin = nullptr, *vout = nullptr;

  // block byte histograms: in the caller's buffer when it wants them (the MTF stage derives its symbol map from them)
  DBuf<u32> bytehist_own;
  if (!d_hist_out) bytehist_own.alloc(c, (size_t)nblk * 256);
  u32* const bytehist = d_hist_out ? d_hist_out : bytehist_own.p;
  DBuf<float> dscore(c, 1);
  CUDA_CHECK(cudaMemsetAsync(bytehist, 0, (size_t)nblk * 256 * 4, c.stream));
  const u32 bk_tps = (n_max + BK_THREADS * BK_ITEMS - 1) / (BK_THREADS * BK_ITEMS);
  // The block byte histograms come first: they are the digit histogram of every pass of the 4-byte-prefix sort, the
  // bucket sizes of the MSD path and the input of the text-likeness score that picks the mode of the batch.
  if (!sentinel) {
    const u32 bh_tps = (n_max + BH_TILE - 1) / BH_TILE;
    k_byte_hist<<<bh_tps * nblk, BK_THREADS, 0, c.stream>>>(d_T, d_n, bh_tps, bytehist);
    KLAUNCH(c); KCHECK();
    c.stats.bwt_bytes += n_total;
  }
  k_text_score<<<1, 256, 0, c.stream>>>(bytehist, d_n, nblk, dscore);  // sentinel mode: zero histogram, score 0
  KLAUNCH(c); KCHECK();
  // Text-like batches (many 4-byte-prefix collisions) sort on the first EIGHT bytes before the doubling
  // rounds start: bytes 4..7 first, then a stable sort on bytes 0..3 -- two cheap keys-only sorts replace
  // the h=4 round over nearly all suffixes.  The first batch of a call reads its own score (one small sync);
  // later batches follow the score of the batch before them (B2_BWT_PREFIX8 forces the mode).
  if (!sentinel && !c.bwt_wide_forced && !c.bwt_mode_known) {
    float sc = 0.f;
    c.to_host(&sc, dscore, 4);
    c.sync();
    c.bwt_wide = sc > 0.5f;
    c.bwt_mode_known = true;
  }
  const bool wide = sentinel ? false : c.bwt_wide;
  if (wide) c.stats.bwt_wide_batches++;
  if (!wide && !sentinel && c.bwt_msd) {
    // sparse-tie batches: one MSD pass + shared-memory bucket sorts (bwt_msd.cu); ties on 5 bytes are ordered directly
    CUDA_CHECK(cudaMemsetAsync(cnt, 0, 16, c.stream));
    bwt_msd_launch(c, d_T, d_U, d_n, nblk, n_max, n_total, bytehist, recA, d_pidx, headA, idxA, cnt);
    u32 h_ctl[4] = {0, 0, 0, 0};
    float score = 0.f;
    c.to_host(h_ctl, cnt, 16);
    c.to_host(&score, dscore, 4);
    c.sync();
    if (!c.bwt_wide_forced) c.bwt_wide = score > 0.5f;  // next batch of this call
    u32 why = (h_ctl[2] ? WHY_BUCKET : 0u) | (h_ctl[1] ? WHY_CELL : 0u);
    if (!why) {
      const u32 Mt = h_ctl[0];
      u32 failed = 0;
      if (Mt > n_total / 8) why = WHY_TIES;
      else if (Mt) {
        k_resolve_direct<<<(Mt + 127) / 128, 128, 0, c.stream>>>(headA, idxA, Mt, d_T, d_n, 5, d_U, d_pidx, cnt.p + 1);
        KLAUNCH(c); KCHECK();
        c.stats.bwt_bytes += (u64)Mt * 80;
        c.to_host(&failed, cnt.p + 1, 4);
        c.sync();
        why = resolve_why(failed);
      }
      if (!why) { c.stats.bwt_msd_done++; return; }
    }
    c.stats.bwt_msd_fallback_why |= why;
    // an oversized bucket or long repeats after all: the LSD path below redoes the batch
  }
  k_build_keys<<<bk_tps * nblk, BK_THREADS, 0, c.stream>>>(d_T, d_n, bk_tps, kin, nullptr, wide ? 4u : 0u, sentinel ? 1 : 0);
  KLAUNCH(c); KCHECK();
  c.stats.bwt_bytes += n_total * 9;
  // keys-only sort of the packed records on their upper 32 bits
  // (sentinel mode: the zero padding breaks the "byte histogram = digit histogram" identity, so the sort counts its own)
  radix_sort<u64, false>(c, kin, vin, kout, vout, d_n, nblk, SEG_SHIFT, n_max, 32, 4, false, n_total, sentinel ? nullptr : bytehist);
  if (wide) {
    k_rekey<<<(nslots + 255) / 256, 256, 0, c.stream>>>(d_T, d_n, nslots, kin);
    KLAUNCH(c); KCHECK();
    c.stats.bwt_bytes += n_total * 20;
    radix_sort<u64, false>(c, kin, vin, kout, vout, d_n, nblk, SEG_SHIFT, n_max, 32, 4, false, n_total, bytehist);
  }
  u32* SA = saBuf;
  const u32 ri_tps = (n_max + RR_TILE - 1) / RR_TILE;
  const u32 ri_tiles = ri_tps * nblk;  // <= rr_tiles_init
  if (!wide && !sentinel) {
    // sparse-tie path: emit the column straight from the sorted records and order the few tied groups directly
    CUDA_CHECK(cudaMemsetAsync(st, 0, (size_t)3 * rr_tiles_init * 8, c.stream));
    CUDA_CHECK(cudaMemsetAsync(ticket, 0, 4, c.stream));
    CUDA_CHECK(cudaMemsetAsync(cnt, 0, 8, c.stream));  // cnt[0] = tied suffixes, cnt[1] = "needs the rounds" flag
    k_emit_detect<<<ri_tiles, RR_THREADS, 0, c.stream>>>(kin, d_T, d_n, ri_tps, d_U, d_pidx, headA, idxA, cnt, ticket, st.p, st.p + rr_tiles_init,
                                                         ri_tiles);
    KLAUNCH(c); KCHECK();
    c.stats.bwt_bytes += n_total * (8 + 2);
    u32 Mt = 0;
    float score = 0.f;
    c.to_host(&Mt, cnt, 4);
    c.to_host(&score, dscore, 4);
    c.sync();
    if (!c.bwt_wide_forced) c.bwt_wide = score > 0.5f;  // next batch of this call
    u32 failed = 0, why = 0;
    if (Mt > n_total / 8) why = WHY_TIES;
    else if (Mt) {
      k_resolve_direct<<<(Mt + 127) / 128, 128, 0, c.stream>>>(headA, idxA, Mt, d_T, d_n, 4, d_U, d_pidx, cnt.p + 1);
      KLAUNCH(c); KCHECK();
      c.stats.bwt_bytes += (u64)Mt * 80;
      c.to_host(&failed, cnt.p + 1, 4);
      c.sync();
      why = resolve_why(failed);
    }
    if (!why) { c.stats.bwt_direct_done++; return; }
    c.stats.bwt_direct_fallback_why |= why;
    // long repeats after all: fall through to the rank-based rounds (the sorted records are still intact)
  }
  c.stats.bwt_rounds_batches++;
  CUDA_CHECK(cudaMemsetAsync(st, 0, (size_t)3 * rr_tiles_init * 8, c.stream));
  CUDA_CHECK(cudaMemsetAsync(ticket, 0, 4, c.stream));
  CUDA_CHECK(cudaMemsetAsync(cnt, 0, 4, c.stream));
  {
    if (wide)
      k_rerank_init<true><<<ri_tiles, RR_THREADS, 0, c.stream>>>(kin, d_T, SA, d_n, ri_tps, rank, headA, idxA, cnt, ticket, st.p, st.p + rr_tiles_init, ri_tiles);
    else
      k_rerank_init<false><<<ri_tiles, RR_THREADS, 0, c.stream>>>(kin, d_T, SA, d_n, ri_tps, rank, headA, idxA, cnt, ticket, st.p, st.p + rr_tiles_init, ri_tiles);
    KLAUNCH(c); KCHECK();
  }
  c.stats.bwt_bytes += n_total * (8 + 4 + 4);
  u32 M = 0;
  float score = 0.f;
  c.to_host(&M, cnt, 4);
  c.to_host(&score, dscore, 4);
  c.sync();
  if (!c.bwt_wide_forced) c.bwt_wide = score > 0.5f;  // next batch of this call

  if (M > 0) {
    // the initial-sort key buffers are free now; the rounds need 64-bit keys for at most M records
    DBuf<u64> k64A(c, M), k64B(c, M);
    DBuf<u32> v64A(c, M), v64B(c, M), headB(c, M), idxB(c, M);
    u32 *hcur = headA, *icur = idxA, *hnext = headB, *inext = idxB;
    const u32 keybits = SEG_SHIFT + bits_for(nslots - 1);
    const u32 npass = (keybits + RADIX_BITS - 1) / RADIX_BITS;
    DBuf<u32> dM(c, 1);
    u32 h = wide ? 8 : 4, rounds = 0;
    while (M > 0) {
      const int tiebreak = h >= n_max ? 1 : 0;
      rounds++;
      u64* kin64 = k64A; u64* kout64 = k64B; u32* vin64 = v64A; u32* vout64 = v64B;
      k_gather<<<(M + 255) / 256, 256, 0, c.stream>>>(hcur, icur, M, rank, d_n, h, tiebreak, kin64, vin64, sentinel ? 1 : 0);
      KLAUNCH(c); KCHECK();
      c.stats.bwt_bytes += (u64)M * (8 + 4 + 12);
      c.to_device(dM, &M, 4);
      radix_sort<u64>(c, kin64, vin64, kout64, vout64, dM, 1, 31, M, 0, npass, false, M);
      const u32 tiles = (M + RR_TILE - 1) / RR_TILE;
      CUDA_CHECK(cudaMemsetAsync(st, 0, (size_t)3 * rr_tiles_init * 8, c.stream));
      CUDA_CHECK(cudaMemsetAsync(ticket, 0, 4, c.stream));
      CUDA_CHECK(cudaMemsetAsync(cnt, 0, 4, c.stream));
      k_rerank<false><<<tiles, RR_THREADS, 0, c.stream>>>(nullptr, kin64, vin64, d_n, M, SA, rank, hnext, inext, cnt, ticket, st.p,
                                                         st.p + rr_tiles_init, st.p + 2 * (size_t)rr_tiles_init, tiles);
      KLAUNCH(c); KCHECK();
      c.stats.bwt_bytes += (u64)M * (12 + 4 + 4 + 8);
      u32 Mn = 0;
      c.to_host(&Mn, cnt, 4);
      c.sync();
      if (tiebreak && Mn != 0) throw B2Error{-200, "internal error: suffix sort did not converge"};
      M = Mn;
      std::swap(hcur, hnext);
      std::swap(icur, inext);
      if (h < (1u << 30)) h <<= 1;
    }
    if (rounds > c.stats.bwt_rounds) c.stats.bwt_rounds = rounds;
  }
  if (sentinel) {
    k_emit_sa<<<(nslots + 255) / 256, 256, 0, c.stream>>>(SA, d_n, nslots, d_sa_out, d_pidx);
    KLAUNCH(c); KCHECK();
    if (d_U) {
      k_emit_sentinel<<<(nslots + 255) / 256, 256, 0, c.stream>>>(SA, d_T, d_n, nslots, d_pidx, d_U);
      KLAUNCH(c); KCHECK();
    }
    return;
  }
  k_emit<<<(nslots + 255) / 256, 256, 0, c.stream>>>(SA, d_T, d_n, nslots, d_U, d_pidx);
  KLAUNCH(c); KCHECK();
  c.stats.bwt_bytes += n_total * 6;
}
