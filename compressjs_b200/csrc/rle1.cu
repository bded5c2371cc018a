// rle1.cu -- bzip2 initial run-length encoding, block cutting and per-block CRC32 on the GPU.
//
// Reference: lib/Bzip2.js:636-667 (readBlock) + lib/CRC32.js:72-103.  The reference is a
// byte-serial state machine whose run state resets at every block boundary, and the boundary
// is measured in OUTPUT bytes.  Parallel form used here:
//
//   w(i) = RLE1 bytes emitted when raw byte i is consumed = 1,1,1,2,0,0,... for run phases
//          1,2,3,4,5..255 (the 4th byte also emits the count byte), phases restart every 255.
//   A  k_rle_summary : per 4 KiB raw tile, assuming maximal runs: first/last byte, leading /
//                      trailing run length, sum of w behind the leading run.
//   B  k_rle_scan    : one CTA scans the tile summaries -> per tile the run length carried in
//                      (mod 255) and W(tile start) = total output before the tile.
//   C  k_rle_blocks  : one CTA walks the blocks: a block that starts in the middle of a run
//                      re-phases that run (fresh state), everything behind it follows W; the
//                      end is found by a 256-ary search over W(tile) plus one in-tile scan.
//   D  k_rle_emit    : all blocks in parallel: every raw byte computes its output position and
//                      writes its literal (+ count byte) into the slot layout.
//   CRC k_crc_pieces : 256-byte pieces, pure polynomial remainders shifted by x^(8*bytes after)
//                      and XOR-combined per block (CRC is linear), then the init/final XOR.
#include <algorithm>
#include <cstdlib>
#include "enc.h"

#define RT_THREADS 256
#define RT_PER 16  // RLE_TILE / RT_THREADS

struct TileSum {
  u32 lead, trail, rest;
  u8 fc, lc, allsame, pad;
};

// RLE1 bytes produced by c bytes of one run consumed from a fresh state.
__host__ __device__ __forceinline__ u64 outfresh(u64 c) {
  u64 q = c / 255, r = c % 255;
  return 5 * q + (r <= 3 ? r : 5);
}
// smallest c with outfresh(c) >= target (target >= 1)
__host__ __device__ __forceinline__ u64 cneed(u64 target) {
  u64 q = (target - 1) / 5, rem = target - 5 * q;  // rem in 1..5
  return 255 * q + (rem <= 3 ? rem : 4);
}
__device__ __forceinline__ u32 w_of_dist(u32 d) {
  u32 r = d % 255 + 1;
  return r <= 3 ? 1u : (r == 4 ? 2u : 0u);
}

// Per-thread view of one raw tile under maximal-run phases.
struct TileView {
  u8 by[RT_PER];
  u8 w[RT_PER];
  u32 cnt;    // valid bytes of this thread
  u32 excl;   // sum of w over the tile positions before this thread's first byte
  u32 total;  // sum of w over the tile
  u32 first_start;  // smallest position > 0 that starts a run (tile length when none)
  u32 last_start;   // largest position that starts a run (0 when the tile is one run)
  u32 len;          // valid bytes in the tile
};

struct TileScratch {
  u32 ws[RT_THREADS / 32 + 1];
  u8 lastb[RT_THREADS];
  u32 red[RT_THREADS / 32];
};

__device__ __forceinline__ u32 block_excl_max256(u32 v, u32* ws) {
  u32 inc = warp_incl_max(v);
  u32 exw = __shfl_up_sync(FULL_MASK, inc, 1);
  if (lane_id() == 0) exw = 0;
  const int w = threadIdx.x >> 5;
  if (lane_id() == 31) ws[w] = inc;
  __syncthreads();
  if (w == 0) {
    u32 x = (lane_id() < RT_THREADS / 32) ? ws[lane_id()] : 0u;
    u32 xi = warp_incl_max(x);
    u32 xe = __shfl_up_sync(FULL_MASK, xi, 1);
    if (lane_id() == 0) xe = 0;
    if (lane_id() < RT_THREADS / 32) ws[lane_id()] = xe;
  }
  __syncthreads();
  u32 c = ws[w];
  __syncthreads();
  return exw > c ? exw : c;
}
__device__ __forceinline__ u32 block_min256(u32 v, u32* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(FULL_MASK, v, o));
  if (lane_id() == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  u32 r = red[0];
#pragma unroll
  for (int i = 1; i < RT_THREADS / 32; i++) r = min(r, red[i]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ u32 block_max256(u32 v, u32* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(FULL_MASK, v, o));
  if (lane_id() == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  u32 r = red[0];
#pragma unroll
  for (int i = 1; i < RT_THREADS / 32; i++) r = max(r, red[i]);
  __syncthreads();
  return r;
}

// Whole CTA (RT_THREADS threads).  carry = run length (mod 255) entering the tile.
__device__ void tile_view(const u8* __restrict__ in, u64 N, u64 tstart, u32 carry, TileScratch& sc, TileView& v) {
  const u32 tid = threadIdx.x;
  const u64 remain = N - tstart;
  v.len = remain < RLE_TILE ? (u32)remain : RLE_TILE;
  const u32 pos0 = tid * RT_PER;
  v.cnt = pos0 >= v.len ? 0 : min((u32)RT_PER, v.len - pos0);
  const u8* p = in + tstart + pos0;
  if (v.cnt == RT_PER && (((size_t)p) & 15) == 0) {
    uint4 q = *reinterpret_cast<const uint4*>(p);
    u32 a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < RT_PER; j++) v.by[j] = (u8)(a[j >> 2] >> ((j & 3) * 8));
  } else {
#pragma unroll
    for (int j = 0; j < RT_PER; j++) v.by[j] = (j < (int)v.cnt) ? p[j] : 0;
  }
  sc.lastb[tid] = v.by[RT_PER - 1];
  __syncthreads();
  const u8 prev0 = tid ? sc.lastb[tid - 1] : 0;
  // run starts inside the tile (position 0 always counts as one; its phase comes from `carry`)
  u32 smask = 0, last_local = 0, first_local = 0xffffffffu;
#pragma unroll
  for (int j = 0; j < RT_PER; j++) {
    if (j < (int)v.cnt) {
      const u32 pos = pos0 + j;
      const u8 pb = j ? v.by[j - 1] : prev0;
      const bool st = (pos == 0) || (v.by[j] != pb);
      if (st) {
        smask |= 1u << j;
        last_local = pos + 1;
        if (pos > 0 && first_local == 0xffffffffu) first_local = pos;
      }
    }
  }
  const u32 ex = block_excl_max256(last_local, sc.ws);  // (last start before this thread) + 1
  u32 rs = ex ? ex - 1 : 0;
  u32 sum = 0;
#pragma unroll
  for (int j = 0; j < RT_PER; j++) {
    u32 ww = 0;
    if (j < (int)v.cnt) {
      const u32 pos = pos0 + j;
      if (smask & (1u << j)) rs = pos;
      const u32 d = pos - rs + (rs == 0 ? carry : 0);
      ww = w_of_dist(d);
    }
    v.w[j] = (u8)ww;
    sum += ww;
  }
  u32 total;
  v.excl = block_excl_add<RT_THREADS, u32>(sum, sc.ws, &total);
  v.total = total;
  u32 fs = block_min256(first_local, sc.red);
  v.first_start = fs == 0xffffffffu ? v.len : fs;
  u32 ls = block_max256(last_local, sc.red);
  v.last_start = ls ? ls - 1 : 0;
}

// ---- A ---------------------------------------------------------------------------------
// Fast path: a tile that contains no four equal consecutive bytes (looking 3 bytes back into the
// previous tile) emits exactly one output byte per input byte, so its summary needs no scans.
__global__ void __launch_bounds__(RT_THREADS) k_rle_summary(const u8* __restrict__ in, u64 N, TileSum* __restrict__ sums, u8* __restrict__ plain) {
  __shared__ TileScratch sc;
  __shared__ u32 lastw[RT_THREADS];
  const u64 t = blockIdx.x;
  const u64 tstart = t * RLE_TILE;
  const u32 tid = threadIdx.x;
  const u64 remain = N - tstart;
  const u32 len = remain < RLE_TILE ? (u32)remain : RLE_TILE;
  const u8* p = in + tstart + tid * RT_PER;
  if (len == RLE_TILE && ((((size_t)in) + tstart) & 15) == 0) {
    const uint4 q = *reinterpret_cast<const uint4*>(p);
    lastw[tid] = q.w;
    __syncthreads();
    u32 prevw;  // the 4 bytes before this thread's 16 (only 3 are used)
    if (tid) prevw = lastw[tid - 1];
    else if (tstart >= 4) prevw = ((u32)in[tstart - 1] << 24) | ((u32)in[tstart - 2] << 16) | ((u32)in[tstart - 3] << 8);
    else {
      // near the start of the input: bytes that do not exist must not look equal
      prevw = 0;
      for (int k = 1; k <= 3; k++) {
        const u32 b = (tstart >= (u64)k) ? in[tstart - k] : (u32)((u8)(~q.x) + k);
        prevw |= b << (8 * (4 - k));
      }
    }
    // x_i == x_{i-1} for every byte, via word-wise compare of the stream shifted by one byte
    const u32 a[5] = {prevw, q.x, q.y, q.z, q.w};
    u32 any4 = 0;
#pragma unroll
    for (int wv = 1; wv < 5; wv++) {
      const u32 cur = a[wv], sh1 = __funnelshift_l(a[wv - 1], cur, 8);   // bytes shifted by one position
      const u32 sh2 = __funnelshift_l(a[wv - 1], cur, 16), sh3 = __funnelshift_l(a[wv - 1], cur, 24);
      const u32 e = __vcmpeq4(cur, sh1) & __vcmpeq4(cur, sh2) & __vcmpeq4(cur, sh3);
      any4 |= e;
    }
    if (!__syncthreads_or(any4 != 0)) {
      if (tid == 0) {
        TileSum s;
        s.fc = in[tstart];
        s.lc = in[tstart + len - 1];
        u32 lead = 1;
        while (lead < 4 && in[tstart + lead] == s.fc) lead++;
        u32 trail = 1;
        while (trail < 4 && in[tstart + len - 1 - trail] == s.lc) trail++;
        s.lead = lead; s.trail = trail; s.allsame = 0; s.rest = len - lead; s.pad = 0;
        sums[t] = s;
        plain[t] = 1;
      }
      return;
    }
  }
  TileView v;
  tile_view(in, N, tstart, 0, sc, v);
  if (threadIdx.x == 0) {
    plain[t] = 0;
    TileSum s;
    s.fc = in[tstart];
    s.lc = in[tstart + v.len - 1];
    s.lead = v.first_start;
    s.allsame = v.first_start == v.len;
    s.trail = v.len - v.last_start;
    // total was computed with carry 0, so its leading run contributed outfresh(lead)
    s.rest = v.total - (u32)outfresh(v.first_start);
    s.pad = 0;
    sums[t] = s;
  }
}

// ---- B ---------------------------------------------------------------------------------
// scan state: bit 63 nonempty | bit 62 allsame | fc<<24 | lc<<16 | trail255<<8 | len255
__device__ __forceinline__ u64 rs_make(bool allsame, u32 fc, u32 lc, u32 trail, u32 len) {
  return (1ull << 63) | ((u64)allsame << 62) | ((u64)fc << 24) | ((u64)lc << 16) | ((u64)trail << 8) | (u64)len;
}
__device__ __forceinline__ u64 rs_combine(u64 A, u64 B) {
  if (!(A >> 63)) return B;
  if (!(B >> 63)) return A;
  const bool Aall = (A >> 62) & 1, Ball = (B >> 62) & 1;
  const u32 Afc = (A >> 24) & 255, Alc = (A >> 16) & 255, Atr = (A >> 8) & 255, Alen = A & 255;
  const u32 Bfc = (B >> 24) & 255, Blc = (B >> 16) & 255, Btr = (B >> 8) & 255, Blen = B & 255;
  const bool join = Alc == Bfc;
  const u32 trail = (Ball && join) ? (Atr + Blen) % 255 : Btr;
  return rs_make(Aall && Ball && join, Afc, Blc, trail, (Alen + Blen) % 255);
}

#define RS_THREADS 1024
__global__ void __launch_bounds__(RS_THREADS)
k_rle_scan(const TileSum* __restrict__ sums, u64 ntiles, u64 N, u32* __restrict__ carry, u64* __restrict__ prefix, u64 st0, u64 W0,
           u64* __restrict__ agg_out) {
  __shared__ u64 sa[RS_THREADS], sb[RS_THREADS];
  const u32 tid = threadIdx.x;
  const u64 per = (ntiles + RS_THREADS - 1) / RS_THREADS;
  const u64 t0 = (u64)tid * per, t1 = min(ntiles, t0 + per);
  // 1. aggregate of this thread's tiles
  u64 agg = 0;
  for (u64 t = t0; t < t1; t++) {
    const TileSum s = sums[t];
    const u64 tl = min((u64)RLE_TILE, N - t * RLE_TILE);
    agg = rs_combine(agg, rs_make(s.allsame, s.fc, s.lc, s.trail % 255, (u32)(tl % 255)));
  }
  // 2. exclusive scan over threads (Hillis-Steele, operator is not commutative)
  sa[tid] = agg;
  __syncthreads();
  u64* src = sa; u64* dst = sb;
  for (u32 o = 1; o < RS_THREADS; o <<= 1) {
    u64 x = src[tid];
    if (tid >= o) x = rs_combine(src[tid - o], x);
    dst[tid] = x;
    __syncthreads();
    u64* tmp = src; src = dst; dst = tmp;
  }
  u64 st = rs_combine(st0, tid ? src[tid - 1] : 0);  // st0: run state entering the buffer (a share of a larger input)
  if (tid == 0 && agg_out) *agg_out = src[RS_THREADS - 1];
  __syncthreads();
  // 3. carries + per-tile output sums (stored in prefix[] for now)
  u64 mysum = 0;
  for (u64 t = t0; t < t1; t++) {
    const TileSum s = sums[t];
    const u64 tl = min((u64)RLE_TILE, N - t * RLE_TILE);
    u32 c = 0;
    if ((st >> 63) && ((st >> 16) & 255) == s.fc) c = (st >> 8) & 255;
    carry[t] = c;
    const u64 S = outfresh((u64)c + s.lead) - outfresh(c) + s.rest;
    prefix[t] = S;
    mysum += S;
    st = rs_combine(st, rs_make(s.allsame, s.fc, s.lc, s.trail % 255, (u32)(tl % 255)));
  }
  // 4. exclusive add scan of the thread sums
  sa[tid] = mysum;
  __syncthreads();
  src = sa; dst = sb;
  for (u32 o = 1; o < RS_THREADS; o <<= 1) {
    u64 x = src[tid];
    if (tid >= o) x += src[tid - o];
    dst[tid] = x;
    __syncthreads();
    u64* tmp = src; src = dst; dst = tmp;
  }
  u64 run = W0 + (tid ? src[tid - 1] : 0);
  const u64 grand = W0 + src[RS_THREADS - 1];
  for (u64 t = t0; t < t1; t++) {
    const u64 S = prefix[t];
    prefix[t] = run;
    run += S;
  }
  if (tid == 0) prefix[ntiles] = grand;
}

// Multi-CTA version of the same scan for inputs of many tiles (one CTA per RG_TILES tiles, five small launches):
//   g1: per group, the aggregate run state                    g2: exclusive scan of the group aggregates (one CTA)
//   g3: per tile carry + output size S (in prefix[]), group sums   g4: exclusive scan of the group sums (one CTA)
//   g5: prefix[t] = group base + exclusive scan of S inside the group
#define RG_THREADS 256
#define RG_PER 8
#define RG_TILES (RG_THREADS * RG_PER)
__device__ __forceinline__ u64 rg_tile_state(const TileSum& s, u64 t, u64 N) {
  const u64 tl = min((u64)RLE_TILE, N - t * RLE_TILE);
  return rs_make(s.allsame, s.fc, s.lc, s.trail % 255, (u32)(tl % 255));
}
// exclusive scan over the CTA's threads with the (non commutative) state operator; *total = combination of all
__device__ __forceinline__ u64 rg_block_excl_state(u64 v, u64* sa, u64* sb, u64* total) {
  const u32 tid = threadIdx.x;
  sa[tid] = v;
  __syncthreads();
  u64* src = sa; u64* dst = sb;
  for (u32 o = 1; o < RG_THREADS; o <<= 1) {
    u64 x = src[tid];
    if (tid >= o) x = rs_combine(src[tid - o], x);
    dst[tid] = x;
    __syncthreads();
    u64* tmp = src; src = dst; dst = tmp;
  }
  const u64 ex = tid ? src[tid - 1] : 0;
  *total = src[RG_THREADS - 1];
  __syncthreads();
  return ex;
}
__global__ void __launch_bounds__(RG_THREADS)
k_rle_scan_g1(const TileSum* __restrict__ sums, u64 ntiles, u64 N, u64* __restrict__ group_agg) {
  __shared__ u64 sa[RG_THREADS], sb[RG_THREADS];
  const u64 t0 = (u64)blockIdx.x * RG_TILES + (u64)threadIdx.x * RG_PER;
  u64 agg = 0;
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    if (t < ntiles) agg = rs_combine(agg, rg_tile_state(sums[t], t, N));
  }
  u64 total;
  rg_block_excl_state(agg, sa, sb, &total);
  if (threadIdx.x == 0) group_agg[blockIdx.x] = total;
}
// one CTA: exclusive scan of ngroups values (state operator when STATE, plain addition otherwise); out[ngroups] = total
template <bool STATE>
__global__ void __launch_bounds__(RS_THREADS)
k_rle_scan_groups(const u64* __restrict__ in, u32 ngroups, u64* __restrict__ out, u64 init, u64* __restrict__ agg_out) {
  __shared__ u64 sa[RS_THREADS], sb[RS_THREADS];
  const u32 tid = threadIdx.x;
  const u32 per = (ngroups + RS_THREADS - 1) / RS_THREADS;
  const u32 g0 = tid * per, g1 = min(ngroups, g0 + per);
  u64 agg = 0;
  for (u32 g = g0; g < g1; g++) agg = STATE ? rs_combine(agg, in[g]) : agg + in[g];
  sa[tid] = agg;
  __syncthreads();
  u64* src = sa; u64* dst = sb;
  for (u32 o = 1; o < RS_THREADS; o <<= 1) {
    u64 x = src[tid];
    if (tid >= o) x = STATE ? rs_combine(src[tid - o], x) : src[tid - o] + x;
    dst[tid] = x;
    __syncthreads();
    u64* tmp = src; src = dst; dst = tmp;
  }
  u64 run = tid ? src[tid - 1] : 0;
  run = STATE ? rs_combine(init, run) : init + run;
  if (tid == 0 && agg_out) *agg_out = src[RS_THREADS - 1];  // combination of all groups without `init`
  for (u32 g = g0; g < g1; g++) {
    const u64 v = in[g];
    out[g] = run;
    run = STATE ? rs_combine(run, v) : run + v;
  }
  if (tid == RS_THREADS - 1) out[ngroups] = STATE ? rs_combine(init, src[RS_THREADS - 1]) : init + src[RS_THREADS - 1];
}
__global__ void __launch_bounds__(RG_THREADS)
k_rle_scan_g3(const TileSum* __restrict__ sums, u64 ntiles, u64 N, const u64* __restrict__ group_start, u32* __restrict__ carry,
              u64* __restrict__ prefix, u64* __restrict__ group_sum) {
  __shared__ u64 sa[RG_THREADS], sb[RG_THREADS];
  __shared__ u32 ws[RG_THREADS / 32 + 1];
  const u64 t0 = (u64)blockIdx.x * RG_TILES + (u64)threadIdx.x * RG_PER;
  TileSum ts[RG_PER];
  u64 agg = 0;
#pragma unroll
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    if (t < ntiles) { ts[j] = sums[t]; agg = rs_combine(agg, rg_tile_state(ts[j], t, N)); }
  }
  u64 total;
  u64 st = rs_combine(group_start[blockIdx.x], rg_block_excl_state(agg, sa, sb, &total));
  u32 mysum = 0;  // <= 2048 tiles x 5120 bytes per group: fits 32 bits
#pragma unroll
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    if (t < ntiles) {
      const TileSum& s = ts[j];
      u32 c = 0;
      if ((st >> 63) && ((st >> 16) & 255) == s.fc) c = (st >> 8) & 255;
      carry[t] = c;
      const u64 S = outfresh((u64)c + s.lead) - outfresh(c) + s.rest;
      prefix[t] = S;
      mysum += (u32)S;
      st = rs_combine(st, rg_tile_state(s, t, N));
    }
  }
  u32 tot;
  block_excl_add<RG_THREADS, u32>(mysum, ws, &tot);
  if (threadIdx.x == 0) group_sum[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(RG_THREADS)
k_rle_scan_g5(u64 ntiles, const u64* __restrict__ group_base, u32 ngroups, u64* __restrict__ prefix) {
  __shared__ u32 ws[RG_THREADS / 32 + 1];
  const u64 t0 = (u64)blockIdx.x * RG_TILES + (u64)threadIdx.x * RG_PER;
  u32 S[RG_PER];
  u32 mysum = 0;
#pragma unroll
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    S[j] = t < ntiles ? (u32)prefix[t] : 0u;
    mysum += S[j];
  }
  u32 tot;
  u64 run = group_base[blockIdx.x] + block_excl_add<RG_THREADS, u32>(mysum, ws, &tot);
#pragma unroll
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    if (t < ntiles) { prefix[t] = run; run += S[j]; }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) prefix[ntiles] = group_base[ngroups];
}

// ---- C ---------------------------------------------------------------------------------
struct BlocksShared {
  TileScratch sc;
  u64 r64;
  u32 r32;
};

// W(x): RLE1 output of raw[0,x) under maximal phases.  Whole CTA.
__device__ u64 eval_W(const u8* in, u64 N, const u32* carry, const u64* prefix, u64 x, BlocksShared& sh) {
  const u64 t = x / RLE_TILE;
  const u32 off = (u32)(x % RLE_TILE);
  if (off == 0) return prefix[t];
  TileView v;
  tile_view(in, N, t * RLE_TILE, carry[t], sh.sc, v);
  const u32 tid = threadIdx.x;
  if (off / RT_PER == tid) {
    u32 a = v.excl;
    for (u32 j = 0; j < off % RT_PER; j++) a += v.w[j];
    sh.r64 = prefix[t] + a;
  }
  __syncthreads();
  u64 r = sh.r64;
  __syncthreads();
  return r;
}

// first position >= s whose byte differs from in[s], capped at cap.  Whole CTA.
__device__ u64 find_run_end(const u8* in, u64 s, u64 cap, BlocksShared& sh) {
  const u8 ch = in[s];
  for (u64 base = s; base < cap; base += RLE_TILE) {
    const u64 p0 = base + (u64)threadIdx.x * RT_PER;
    u32 found = 0xffffffffu;
    for (u32 j = 0; j < RT_PER; j++) {
      const u64 p = p0 + j;
      if (p < cap && in[p] != ch) { found = (u32)(p - base); break; }
    }
    const u32 f = block_min256(found, sh.sc.red);
    if (f != 0xffffffffu) return base + f;
  }
  return cap;
}

__global__ void __launch_bounds__(RT_THREADS)
k_rle_blocks(const u8* __restrict__ in, u64 N, u32 BS, const u32* __restrict__ carry, const u64* __restrict__ prefix, u64 ntiles,
             BlkInfo* __restrict__ blocks, u32* nblocks_out, u32 maxblocks, u64 u_start, u32 range_first, u32 range_count, int open_end) {
  __shared__ BlocksShared sh;
  const u32 tid = threadIdx.x;
  const u64 Wtotal = prefix[ntiles];
  if (gridDim.x > 1) {
    // parallel walk: CTA r takes its share of the blocks [range_first, range_first + range_count) that W predicts,
    // from the speculative boundary W = first*BS; the host accepts the result only if every segment ends where
    // the next one starts (then it IS the sequential walk) and repeats the walk with one CTA otherwise.
    // blocks[0] is block range_first; open_end: the last CTA goes on to the end of the input.
    const u32 P = gridDim.x, r = blockIdx.x;
    const u32 first = range_first + (u32)((u64)r * range_count / P), next = range_first + (u32)((u64)(r + 1) * range_count / P);
    u_start = (u64)first * BS;
    blocks += first - range_first;
    nblocks_out += r;
    maxblocks = (r == P - 1 && open_end) ? maxblocks - (first - range_first) : next - first;
  }
  u64 s = 0, Ws = prefix[0];
  bool Ws_valid = true;  // W(0) = 0 (or the W base of a share)
  u32 k = 0;
  if (u_start > 0) {
    // speculative start (multi-GPU range plan): the first raw position x with W(x) >= u_start, i.e. where a
    // block boundary falls if no block before it was shifted by a run-phase slip (verified by the caller)
    if (u_start > Wtotal) { if (tid == 0) *nblocks_out = 0; return; }
    u64 lo = 0, hi = ntiles;
    while (hi - lo > 1) {
      const u64 span = hi - lo;
      const u64 pi = lo + 1 + (span - 1) * (u64)tid / RT_THREADS;
      const bool valid = pi < hi && (tid == 0 || pi != lo + 1 + (span - 1) * (u64)(tid - 1) / RT_THREADS);
      const bool pr = valid && prefix[pi] < u_start;
      const u32 tr = block_max256(pr ? tid + 1 : 0, sh.sc.red);
      const u32 fl = block_min256((valid && !pr) ? tid : 0xffffffffu, sh.sc.red);
      u64 nlo = lo, nhi = hi;
      if (tr) nlo = lo + 1 + (span - 1) * (u64)(tr - 1) / RT_THREADS;
      if (fl != 0xffffffffu) nhi = lo + 1 + (span - 1) * (u64)fl / RT_THREADS;
      lo = nlo; hi = nhi;
    }
    const u64 t = lo;
    TileView v;
    tile_view(in, N, t * RLE_TILE, carry[t], sh.sc, v);
    u32 found = 0xffffffffu;
    {
      u64 acc = prefix[t] + v.excl;
      for (u32 j = 0; j < v.cnt; j++) {
        acc += v.w[j];
        if (acc >= u_start) { found = tid * RT_PER + j; break; }
      }
    }
    const u32 f = block_min256(found, sh.sc.red);
    if (f / RT_PER == tid) {
      u64 acc = prefix[t] + v.excl;
      for (u32 j = 0; j <= f % RT_PER; j++) acc += v.w[j];
      sh.r64 = acc;
    }
    __syncthreads();
    Ws = sh.r64;
    __syncthreads();
    s = t * RLE_TILE + f + 1;
    Ws_valid = true;
  }
  while (s < N && k < maxblocks) {
    BlkInfo bi;
    bi.s = s;
    const bool midrun = s > 0 && in[s - 1] == in[s];
    u64 b = s;
    if (midrun) {
      const u64 cap = min(N, s + cneed(BS));
      b = find_run_end(in, s, cap, sh);
    }
    const u64 ofs = outfresh(b - s);
    u64 e;
    if (ofs >= BS) {
      // the block fills up inside its first (re-phased) run
      e = s + cneed(BS);
      bi.e = e; bi.b = e; bi.Wb = 0; bi.ofs = 0; bi.n = BS;
      Ws_valid = false;
    } else {
      u64 Wb;
      if (midrun) Wb = eval_W(in, N, carry, prefix, b, sh);
      else Wb = Ws_valid ? Ws : eval_W(in, N, carry, prefix, s, sh);
      const u64 V = Wb + (BS - ofs);
      if (V > Wtotal) {
        e = N;
        bi.e = e; bi.b = b; bi.Wb = Wb; bi.ofs = (u32)ofs; bi.n = (u32)(ofs + (Wtotal - Wb));
        Ws_valid = false;
      } else {
        // largest tile t >= tile(b) with prefix[t] < V
        u64 lo = b / RLE_TILE, hi = ntiles;  // pred(lo) true, pred(hi) false
        {
          // W grows by ~1 per raw byte on ordinary data: try the tile that linear extrapolation predicts
          const u64 plo = prefix[lo];
          u64 tg = lo + ((V - plo) >> 12);
          if (tg >= ntiles) tg = ntiles - 1;
          const u64 pg = prefix[tg], pg1 = prefix[tg + 1];
          if (pg < V && pg1 >= V) { lo = tg; hi = tg + 1; }
          else if (pg < V) lo = tg;
          else if (tg > lo) hi = tg;
        }
        if (hi - lo > 1) {
          // narrow with a guess window first (typical data: about BS raw bytes per block)
          const u64 a = ((BS - ofs) * 4 / 5) / RLE_TILE;
          const u64 g0 = lo + (a > 1 ? a - 1 : 0);
          if (g0 < ntiles && prefix[g0] < V) {
            lo = g0;
            const u64 g1 = g0 + 4 * RT_THREADS;
            if (g1 < ntiles && !(prefix[g1] < V)) hi = g1;
          }
        }
        while (hi - lo > 1) {
          const u64 span = hi - lo;
          // probe points lo < p_i < hi, increasing in i
          const u64 pi = lo + 1 + (span - 1) * (u64)tid / RT_THREADS;
          const bool valid = pi < hi && (tid == 0 || pi != lo + 1 + (span - 1) * (u64)(tid - 1) / RT_THREADS);
          const bool pr = valid && prefix[pi] < V;
          // largest true probe -> new lo ; smallest false probe -> new hi
          const u32 tr = block_max256(pr ? tid + 1 : 0, sh.sc.red);
          const u32 fl = block_min256((valid && !pr) ? tid : 0xffffffffu, sh.sc.red);
          u64 nlo = lo, nhi = hi;
          if (tr) nlo = lo + 1 + (span - 1) * (u64)(tr - 1) / RT_THREADS;
          if (fl != 0xffffffffu) nhi = lo + 1 + (span - 1) * (u64)fl / RT_THREADS;
          lo = nlo; hi = nhi;
        }
        const u64 t = lo;
        TileView v;
        tile_view(in, N, t * RLE_TILE, carry[t], sh.sc, v);
        // smallest position whose inclusive W reaches V
        u32 found = 0xffffffffu;
        {
          u64 acc = prefix[t] + v.excl;
          for (u32 j = 0; j < v.cnt; j++) {
            acc += v.w[j];
            if (acc >= V) { found = tid * RT_PER + j; break; }
          }
        }
        const u32 f = block_min256(found, sh.sc.red);
        // f always exists: prefix[t+1] >= V
        if (f / RT_PER == tid) {
          u64 acc = prefix[t] + v.excl;
          for (u32 j = 0; j <= f % RT_PER; j++) acc += v.w[j];
          sh.r64 = acc;
        }
        __syncthreads();
        const u64 We = sh.r64;
        __syncthreads();
        e = t * RLE_TILE + f + 1;
        const u64 produced = ofs + (We - Wb);
        bi.e = e; bi.b = b; bi.Wb = Wb; bi.ofs = (u32)ofs; bi.n = (u32)min(produced, (u64)BS);
        Ws = We; Ws_valid = true;
      }
    }
    if (tid == 0) blocks[k] = bi;
    k++;
    s = e;
  }
  if (tid == 0) *nblocks_out = k;
}

// ---- D ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(RT_THREADS)
k_rle_emit(const u8* __restrict__ in, u64 N, const u32* __restrict__ carry, const u64* __restrict__ prefix, const u8* __restrict__ plain,
           const BlkInfo* __restrict__ blocks, u32 first, u32 count, const u64* __restrict__ tile_base, u8* __restrict__ T) {
  __shared__ TileScratch sc;
  __shared__ u32 s_k;
  __shared__ __align__(16) u8 stage[RLE_TILE + 32];
  // which block does this CTA work for?  tile_base[k] = first CTA of block (first+k)
  if (threadIdx.x == 0) {
    u32 lo = 0, hi = count;
    while (hi - lo > 1) {
      u32 mid = (lo + hi) >> 1;
      if (tile_base[mid] <= blockIdx.x) lo = mid; else hi = mid;
    }
    s_k = lo;
  }
  __syncthreads();
  const u32 kk = s_k;
  const BlkInfo bi = blocks[first + kk];
  const u64 t = bi.s / RLE_TILE + (blockIdx.x - tile_base[kk]);
  const u64 tstart = t * RLE_TILE;
  u8* Tb = T + ((size_t)kk << SEG_SHIFT);
  const u64 Pt = prefix[t];
  if (plain[t]) {
    // No run reaches four bytes in or into this tile: every raw byte emits itself (w = 1), whatever the phase, so the
    // tile's part of the block is a byte copy to output position (x - x0) + o0.  Staged in shared memory at the
    // destination's alignment, stored 16 bytes at a time.
    const u64 remain = N - tstart;
    const u32 len = remain < RLE_TILE ? (u32)remain : RLE_TILE;
    const u64 x0 = bi.s > tstart ? bi.s : tstart;                                    // first raw byte of the block in this tile
    const u64 x1 = (bi.e < tstart + len) ? bi.e : tstart + len;
    if (x0 >= x1) return;
    // output position of x0 (same formulas as the general path below, with w = 1 everywhere)
    const u64 o0 = x0 < bi.b ? (x0 - bi.s) : (u64)bi.ofs + (Pt + (x0 - tstart) - bi.Wb);
    if (o0 >= bi.n) return;
    const u32 cnt = (u32)min((u64)(x1 - x0), (u64)bi.n - o0);
    const u32 fo = (u32)(o0 & 15u);
    const u8* src = in + x0;
    for (u32 i = threadIdx.x * 16u; i < cnt; i += RT_THREADS * 16u) {
      if (i + 16u <= cnt && ((((size_t)src) + i) & 15u) == 0) {
        const uint4 q = *reinterpret_cast<const uint4*>(src + i);
        const u32 a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 16; j++) stage[fo + i + j] = (u8)(a[j >> 2] >> ((j & 3) * 8));
      } else {
        const u32 e = min(i + 16u, cnt);
        for (u32 x = i; x < e; x++) stage[fo + x] = src[x];
      }
    }
    __syncthreads();
    const u32 last = fo + cnt;
    u8* dst = Tb + (o0 - fo);   // 16-byte aligned
    for (u32 c16 = threadIdx.x * 16u; c16 < last; c16 += RT_THREADS * 16u) {
      if (c16 >= fo && c16 + 16u <= last) *reinterpret_cast<uint4*>(dst + c16) = *reinterpret_cast<const uint4*>(stage + c16);
      else {
        const u32 e = min(c16 + 16u, last);
        for (u32 x = max(c16, fo); x < e; x++) dst[x] = stage[x];
      }
    }
    return;
  }
  TileView v;
  tile_view(in, N, tstart, carry[t], sc, v);
  u32 run = v.excl;
  for (u32 j = 0; j < v.cnt; j++) {
    const u64 x = tstart + threadIdx.x * RT_PER + j;
    const u32 wmax = v.w[j];
    const u32 exw = run;
    run += wmax;
    if (x < bi.s || x >= bi.e) continue;
    u32 r;
    u64 opos;
    if (x < bi.b) {
      const u64 d = x - bi.s;
      r = (u32)(d % 255) + 1;
      opos = outfresh(d);
    } else {
      r = wmax == 0 ? 5u : (wmax == 2 ? 4u : 1u);  // only "literal / 4th byte / counted" matters
      opos = bi.ofs + (Pt + exw - bi.Wb);
    }
    if (r > 4 || opos >= bi.n) continue;
    const u8 ch = v.by[j];
    Tb[opos] = ch;
    if (r == 4 && opos + 1 < bi.n) {
      // count byte: how many more equal bytes does this 255-chunk take inside the block?
      u64 lim = x + 1 + 251;
      if (lim > bi.e) lim = bi.e;
      if (x < bi.b && lim > bi.b) lim = bi.b;
      u32 c = 0;
      while (x + 1 + c < lim && in[x + 1 + c] == ch) c++;
      Tb[opos + 1] = (u8)c;
    }
  }
}

// ---- CRC ---------------------------------------------------------------------------------
#define CRC_POLY 0x04c11db7u
__host__ __device__ __forceinline__ u32 gf_mulmod(u32 a, u32 b) {
  u32 r = 0;
  for (int i = 31; i >= 0; i--) {
    r = (r << 1) ^ ((r & 0x80000000u) ? CRC_POLY : 0u);
    if ((b >> i) & 1) r ^= a;
  }
  return r;
}
struct CrcConsts {
  u32 table[256];
  u32 pow[48];  // pow[i] = x^(8 * 2^i) mod P
  u32 slice[3][256];  // slice[k][i] = table value after k+1 further zero bytes: four bytes per step (slicing by 4)
};
static CrcConsts make_crc_consts() {
  CrcConsts c;
  for (u32 i = 0; i < 256; i++) {
    u32 v = i << 24;
    for (int k = 0; k < 8; k++) v = (v & 0x80000000u) ? (v << 1) ^ CRC_POLY : (v << 1);
    c.table[i] = v;
  }
  for (int k = 0; k < 3; k++)
    for (u32 i = 0; i < 256; i++) {
      const u32 prev = k ? c.slice[k - 1][i] : c.table[i];
      c.slice[k][i] = (prev << 8) ^ c.table[prev >> 24];
    }
  c.pow[0] = 0x100;  // x^8
  for (int i = 1; i < 48; i++) c.pow[i] = gf_mulmod(c.pow[i - 1], c.pow[i - 1]);
  return c;
}
__constant__ CrcConsts c_crc;
static bool g_crc_ready = false;
static void crc_setup() {
  if (g_crc_ready) return;
  CrcConsts h = make_crc_consts();
  CUDA_CHECK(cudaMemcpyToSymbol(c_crc, &h, sizeof h));
  g_crc_ready = true;
}
// x^(8*bytes) mod P
__device__ __forceinline__ u32 crc_xpow(u64 bytes) {
  u32 r = 1u;  // bit i of a register value is the coefficient of x^i, so the polynomial 1 is 0x1
  for (int i = 0; bytes; i++, bytes >>= 1)
    if (bytes & 1) r = gf_mulmod(r, c_crc.pow[i]);
  return r;
}

#define CRC_PIECE 256
// Piece j of a block is the j-th 256-byte ADDRESS-aligned window of the buffer that intersects the block's raw
// range [s,e): every full piece is read with aligned 16-byte loads.  A piece that ends inside the block ends
// on a window boundary, 256*k + (e' mod 256) bytes before the block end (e' = e + buffer misalignment), so
// acc[2k] ^= R(piece) * x^(8*256*k) and the common factor x^(8*(e' mod 256)) is applied once in k_crc_final;
// the piece that ends the block goes to acc[2k+1] unshifted.
__host__ __device__ __forceinline__ u64 crc_piece_count(u64 s, u64 e, u32 mis) {
  return e > s ? (e - 1 + mis) / CRC_PIECE - (s + mis) / CRC_PIECE + 1 : 0;
}
__global__ void __launch_bounds__(256)
k_crc_pieces(const u8* __restrict__ in, const BlkInfo* __restrict__ blocks, u32 first, u32 count, const u64* __restrict__ piece_base,
             u64 total_pieces, u32* __restrict__ acc) {
  __shared__ u32 tab[256], t1[256], t2[256], t3[256];
  tab[threadIdx.x] = c_crc.table[threadIdx.x];
  t1[threadIdx.x] = c_crc.slice[0][threadIdx.x];
  t2[threadIdx.x] = c_crc.slice[1][threadIdx.x];
  t3[threadIdx.x] = c_crc.slice[2][threadIdx.x];
  __syncthreads();
  const u64 gid = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total_pieces) return;
  u32 lo = 0, hi = count;
  while (hi - lo > 1) {
    u32 mid = (lo + hi) >> 1;
    if (piece_base[mid] <= gid) lo = mid; else hi = mid;
  }
  const BlkInfo bi = blocks[first + lo];
  const u32 mis = (u32)((size_t)in & (CRC_PIECE - 1));
  const u64 j = gid - piece_base[lo];
  const u64 A = ((bi.s + mis) / CRC_PIECE + j) * CRC_PIECE;  // window start, in misalignment-shifted offsets
  const u64 pbeg = A > bi.s + mis ? A - mis : bi.s;
  const u64 pend = A + CRC_PIECE < bi.e + mis ? A + CRC_PIECE - mis : bi.e;
  u32 crc = 0;
  const u8* p = in + pbeg;
  const u32 len = (u32)(pend - pbeg);
  if (len == CRC_PIECE) {
    for (u32 i = 0; i < CRC_PIECE; i += 16) {
      uint4 q = *reinterpret_cast<const uint4*>(p + i);
      u32 a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int w = 0; w < 4; w++) {
        // four message bytes per dependent step (the stream is MSB first: byte 0 of the little-endian word comes first)
        const u32 x = crc ^ __byte_perm(a[w], 0, 0x0123);
        crc = t3[x >> 24] ^ t2[(x >> 16) & 0xff] ^ t1[(x >> 8) & 0xff] ^ tab[x & 0xff];
      }
    }
  } else {
    for (u32 i = 0; i < len; i++) crc = (crc << 8) ^ tab[((crc >> 24) ^ p[i]) & 0xff];
  }
  if (pend == bi.e) {
    atomicXor(&acc[2 * lo + 1], crc);
  } else {
    const u64 k = (bi.e - pend) / CRC_PIECE;
    if (k) crc = gf_mulmod(crc, crc_xpow(k * CRC_PIECE));
    atomicXor(&acc[2 * lo], crc);
  }
}
__global__ void k_crc_final(const u8* __restrict__ in, const BlkInfo* __restrict__ blocks, u32 first, u32 count, const u32* __restrict__ acc,
                            u32* __restrict__ crc_out) {
  u32 k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const BlkInfo bi = blocks[first + k];
  const u64 len = bi.e - bi.s;
  const u32 mis = (u32)((size_t)in & (CRC_PIECE - 1));
  const u32 body = gf_mulmod(acc[2 * k], crc_xpow((bi.e + mis) % CRC_PIECE)) ^ acc[2 * k + 1];
  crc_out[k] = ~(body ^ gf_mulmod(0xffffffffu, crc_xpow(len)));
}

// single-buffer CRC (b2_crc32_bzip2)
u32 crc32_device(Ctx& c, const u8* d_p, size_t n) {
  crc_setup();
  BlkInfo bi;
  memset(&bi, 0, sizeof bi);
  bi.s = 0; bi.e = n; bi.b = 0; bi.n = 0;
  DBuf<BlkInfo> db(c, 1);
  DBuf<u64> pb(c, 1);
  DBuf<u32> acc(c, 2), out(c, 1);
  u64 zero = 0;
  c.to_device(db, &bi, sizeof bi);
  c.to_device(pb, &zero, 8);
  CUDA_CHECK(cudaMemsetAsync(acc, 0, 8, c.stream));
  const u64 pieces = crc_piece_count(0, n, (u32)((size_t)d_p & (CRC_PIECE - 1)));
  if (pieces) {
    k_crc_pieces<<<(unsigned)((pieces + 255) / 256), 256, 0, c.stream>>>(d_p, db, 0, 1, pb, pieces, acc);
    KLAUNCH(c); KCHECK();
  }
  k_crc_final<<<1, 32, 0, c.stream>>>(d_p, db, 0, 1, acc, out);
  KLAUNCH(c); KCHECK();
  u32 h = 0;
  c.to_host(&h, out, 4);
  c.sync();
  return h;
}

// ---- host drivers ---------------------------------------------------------------------------
// spec_first < 0: exact plan of the whole input.  Otherwise only blocks [spec_first, spec_first+spec_count) are
// walked, starting from the speculative boundary W(s) = spec_first * BS (see k_rle_blocks); plan.first_index
// records the global index of h_blocks[0] and plan.total_guess = ceil(W(N) / BS).
// length of the run the buffer starts with (in bytes, not reduced): tiles of one and the same byte, then the lead of
// the first tile that is not
__global__ void k_share_lead(const TileSum* __restrict__ sums, u64 ntiles, u64* __restrict__ out) {
  if (threadIdx.x) return;
  u64 lead = 0;
  const u8 fc = sums[0].fc;
  for (u64 t = 0; t < ntiles; t++) {
    const TileSum s = sums[t];
    if (s.fc != fc) break;
    lead += s.lead;
    if (!s.allsame) break;
  }
  *out = lead;
}

void rle1_plan_ex(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan, long long spec_first, size_t spec_count, bool tiles_only,
                  u64 st0, u64 W0, u64* agg_state) {
  crc_setup();
  plan.nblocks = 0;
  plan.h_blocks.clear();
  plan.first_index = 0;
  plan.total_guess = 0;
  if (n == 0) return;
  const u32 BS = (u32)level * 100000 - 19;  // lib/Bzip2.js:892-900
  const u64 ntiles = (n + RLE_TILE - 1) / RLE_TILE;
  if (plan.ntiles != ntiles || !plan.tile_prefix.p) {
    plan.ntiles = ntiles;
    DBuf<TileSum> sums(c, ntiles);
    DBuf<u64> dagg(c, 4);
    plan.tile_carry.alloc(c, ntiles);
    plan.tile_prefix.alloc(c, ntiles + 1);
    plan.tile_plain.alloc(c, ntiles);
    k_rle_summary<<<(unsigned)ntiles, RT_THREADS, 0, c.stream>>>(d_in, n, sums, plan.tile_plain);
    KLAUNCH(c); KCHECK();
    static const bool force_groups = getenv("B2_RLE_SCAN_GROUPS") != nullptr;  // test hook: multi-CTA scan on small inputs too
    if (ntiles <= 4 * RG_TILES && !force_groups) {
      k_rle_scan<<<1, RS_THREADS, 0, c.stream>>>(sums, ntiles, n, plan.tile_carry, plan.tile_prefix, st0, W0, dagg);
      KLAUNCH(c); KCHECK();
    } else {
      c.stats.rle_group_scans++;
      const u32 ng = (u32)((ntiles + RG_TILES - 1) / RG_TILES);
      DBuf<u64> gagg(c, ng), gstart(c, ng + 1), gsum(c, ng), gbase(c, ng + 1);
      k_rle_scan_g1<<<ng, RG_THREADS, 0, c.stream>>>(sums, ntiles, n, gagg);
      KLAUNCH(c); KCHECK();
      k_rle_scan_groups<true><<<1, RS_THREADS, 0, c.stream>>>(gagg, ng, gstart, st0, dagg);
      KLAUNCH(c); KCHECK();
      k_rle_scan_g3<<<ng, RG_THREADS, 0, c.stream>>>(sums, ntiles, n, gstart, plan.tile_carry, plan.tile_prefix, gsum);
      KLAUNCH(c); KCHECK();
      k_rle_scan_groups<false><<<1, RS_THREADS, 0, c.stream>>>(gsum, ng, gbase, W0, nullptr);
      KLAUNCH(c); KCHECK();
      k_rle_scan_g5<<<ng, RG_THREADS, 0, c.stream>>>(ntiles, gbase, ng, plan.tile_prefix);
      KLAUNCH(c); KCHECK();
    }
    if (agg_state) {
      // share summary for the multi-GPU planner: aggregate run state, length of the leading run, (W total follows below)
      k_share_lead<<<1, 32, 0, c.stream>>>(sums, ntiles, dagg.p + 1);
      KLAUNCH(c); KCHECK();
      c.to_host(agg_state, dagg, 16);
    }
  }
  u64 wtotal = 0;
  c.to_host(&wtotal, plan.tile_prefix.p + ntiles, 8);
  c.sync();
  plan.total_guess = (size_t)((wtotal + BS - 1) / BS);
  plan.w_total = wtotal;
  if (tiles_only) return;
  u32 maxblocks = (u32)(n / ((u64)BS * 4 / 5) + 2);
  u64 u_start = 0;
  if (spec_first >= 0) {
    maxblocks = (u32)std::min<size_t>(maxblocks, spec_count);
    u_start = (u64)spec_first * BS;
    plan.first_index = (size_t)spec_first;
    if (maxblocks == 0) return;
  }
  plan.blocks.alloc(c, maxblocks);
  // many blocks: walk P segments in parallel first (see k_rle_blocks)
  const u32 total = (u32)plan.total_guess;
  const bool exact = spec_first < 0;
  const u32 rfirst = exact ? 0u : (u32)spec_first, rcount = exact ? total : maxblocks;
  const u32 P = std::min<u32>(64, rcount / 8);
  if (P > 1 && (!exact || total < maxblocks)) {
    DBuf<u32> dnb(c, P);
    k_rle_blocks<<<P, RT_THREADS, 0, c.stream>>>(d_in, n, BS, plan.tile_carry, plan.tile_prefix, ntiles, plan.blocks, dnb, maxblocks, 0, rfirst, rcount,
                                                exact ? 1 : 0);
    KLAUNCH(c); KCHECK();
    std::vector<u32> cut(P);
    c.to_host(cut.data(), dnb, 4 * P);
    c.sync();
    bool ok = true;
    for (u32 r = 0; r + 1 < P && ok; r++) ok = cut[r] == (u32)((u64)(r + 1) * rcount / P) - (u32)((u64)r * rcount / P);
    const u32 last_first = (u32)((u64)(P - 1) * rcount / P);
    ok = ok && cut[P - 1] > 0;
    if (ok) {
      const u32 nb = last_first + cut[P - 1];
      plan.h_blocks.resize(nb);
      c.to_host(plan.h_blocks.data(), plan.blocks, sizeof(BlkInfo) * nb);
      c.sync();
      // exact plans must cover the input; range plans are checked against their neighbours by the caller
      ok = !exact || (plan.h_blocks[0].s == 0 && plan.h_blocks[nb - 1].e == n);
      for (u32 k = 0; k + 1 < nb && ok; k++) ok = plan.h_blocks[k].e == plan.h_blocks[k + 1].s;
      if (ok) { plan.nblocks = nb; c.stats.rle_walk_parallel++; return; }
      plan.h_blocks.clear();
    }
  }
  c.stats.rle_walk_serial++;
  DBuf<u32> dnb(c, 1);
  k_rle_blocks<<<1, RT_THREADS, 0, c.stream>>>(d_in, n, BS, plan.tile_carry, plan.tile_prefix, ntiles, plan.blocks, dnb, maxblocks, u_start, 0, 0, 0);
  KLAUNCH(c); KCHECK();
  u32 nb = 0;
  c.to_host(&nb, dnb, 4);
  c.sync();
  plan.nblocks = nb;
  plan.h_blocks.resize(nb);
  if (nb) c.to_host(plan.h_blocks.data(), plan.blocks, sizeof(BlkInfo) * nb);
  c.sync();
}
void rle1_plan(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan) { rle1_plan_ex(c, d_in, n, level, plan, -1, 0, false, 0, 0, nullptr); }
void rle1_materialize(Ctx& c, const u8* d_in, size_t n, const Rle1Plan& plan, size_t first, size_t count, u8* d_T, u32* d_n, u32* d_crc) {
  if (count == 0) return;
  std::vector<u64> tbase(count + 1), pbase(count + 1);
  std::vector<u32> hn(count);
  u64 tt = 0, pp = 0;
  for (size_t k = 0; k < count; k++) {
    const BlkInfo& bi = plan.h_blocks[first + k];
    tbase[k] = tt; pbase[k] = pp;
    tt += (bi.e - 1) / RLE_TILE - bi.s / RLE_TILE + 1;
    pp += crc_piece_count(bi.s, bi.e, (u32)((size_t)d_in & (CRC_PIECE - 1)));
    hn[k] = bi.n;
  }
  tbase[count] = tt; pbase[count] = pp;
  DBuf<u64> dtb(c, count + 1), dpb(c, count + 1);
  DBuf<u32> acc(c, 2 * count);
  c.to_device(dtb, tbase.data(), 8 * (count + 1));
  c.to_device(dpb, pbase.data(), 8 * (count + 1));
  c.to_device(d_n, hn.data(), 4 * count);
  CUDA_CHECK(cudaMemsetAsync(acc, 0, 8 * count, c.stream));
  k_rle_emit<<<(unsigned)tt, RT_THREADS, 0, c.stream>>>(d_in, n, plan.tile_carry, plan.tile_prefix, plan.tile_plain, plan.blocks, (u32)first, (u32)count, dtb, d_T);
  KLAUNCH(c); KCHECK();
  k_crc_pieces<<<(unsigned)((pp + 255) / 256), 256, 0, c.stream>>>(d_in, plan.blocks, (u32)first, (u32)count, dpb, pp, acc);
  KLAUNCH(c); KCHECK();
  k_crc_final<<<(unsigned)((count + 127) / 128), 128, 0, c.stream>>>(d_in, plan.blocks, (u32)first, (u32)count, acc, d_crc);
  KLAUNCH(c); KCHECK();
}

// CRC32 of arbitrary byte ranges [s,e) of one device buffer (decoder: per-block CRC of the output).
// h_ranges/d_ranges: only .s and .e are used.
void crc_ranges(Ctx& c, const u8* d_data, const BlkInfo* d_ranges, const std::vector<BlkInfo>& h_ranges, u32* d_crc_out) {
  crc_setup();
  const size_t count = h_ranges.size();
  if (count == 0) return;
  std::vector<u64> pbase(count + 1);
  u64 pp = 0;
  for (size_t k = 0; k < count; k++) {
    pbase[k] = pp;
    pp += crc_piece_count(h_ranges[k].s, h_ranges[k].e, (u32)((size_t)d_data & (CRC_PIECE - 1)));
  }
  pbase[count] = pp;
  DBuf<u64> dpb(c, count + 1);
  DBuf<u32> acc(c, 2 * count);
  c.to_device(dpb, pbase.data(), 8 * (count + 1));
  CUDA_CHECK(cudaMemsetAsync(acc, 0, 8 * count, c.stream));
  if (pp) {
    k_crc_pieces<<<(unsigned)((pp + 255) / 256), 256, 0, c.stream>>>(d_data, d_ranges, 0, (u32)count, dpb, pp, acc);
    KLAUNCH(c); KCHECK();
  }
  k_crc_final<<<(unsigned)((count + 127) / 128), 128, 0, c.stream>>>(d_data, d_ranges, 0, (u32)count, acc, d_crc_out);
  KLAUNCH(c); KCHECK();
  c.sync();
}
