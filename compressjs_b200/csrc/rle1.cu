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
//                      (mod 255) and W(tile start) = total output before the tile.  k_rle_scan_g1..g5 do the
//                      same in five launches for inputs of many tiles, with the same CTA scan and per-tile step.
//   C  k_rle_blocks  : one CTA walks the blocks: a block that starts in the middle of a run
//                      re-phases that run (fresh state), everything behind it follows W; the
//                      end is found by the W seek (seek_W): an extrapolated guess and a 256-ary search
//                      over W(tile), then one in-tile scan.  The libbz2 cut (k_rle_blocks_libbz2) and the
//                      share cut (k_w_to_raw) locate their W positions with the same seek.
//   D  k_rle_emit    : one CTA per span of up to 4 tiles of one block (a per-CTA map gives the block, no
//                      search): the span's raw bytes are staged in shared memory, a run of plain tiles is
//                      copied out as destination-aligned 16-byte words (funnel shifts), every raw byte of
//                      another tile computes its output position and writes its literal (+ count byte).
//                      The same pass folds the block CRC: every thread takes the pure polynomial remainder
//                      of 64 staged bytes (slicing by 4), shifts it by x^(8*bytes after it in the span),
//                      the CTA XOR-reduces them and adds the span to the block's accumulators (CRC is
//                      linear); k_crc_final applies the init/final XOR.
//   CRC k_crc_pieces : the same remainders over 256-byte pieces of arbitrary byte ranges (decoder, b2_crc32).
#include <algorithm>
#include <cstdlib>
#include <optional>
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
template <class Op>
__device__ __forceinline__ u32 block_reduce256(u32 v, u32* red, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(FULL_MASK, v, o));
  if (lane_id() == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  u32 r = red[0];
#pragma unroll
  for (int i = 1; i < RT_THREADS / 32; i++) r = op(r, red[i]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ u32 block_min256(u32 v, u32* red) { return block_reduce256(v, red, [](u32 a, u32 b) { return min(a, b); }); }
__device__ __forceinline__ u32 block_max256(u32 v, u32* red) { return block_reduce256(v, red, [](u32 a, u32 b) { return max(a, b); }); }

// Whole CTA (RT_THREADS threads).  carry = run length (mod 255) entering the tile.  PIECES: *pieces receives bit j for
// every byte j of the thread that starts a piece (phase 0 mod 255 of its maximal run: a run start, or byte 255 k of it).
template <bool PIECES = false>
__device__ void tile_view(const u8* __restrict__ in, u64 N, u64 tstart, u32 carry, TileScratch& sc, TileView& v, u32* pieces = nullptr) {
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
  u32 sum = 0, pm = 0;
#pragma unroll
  for (int j = 0; j < RT_PER; j++) {
    u32 ww = 0;
    if (j < (int)v.cnt) {
      const u32 pos = pos0 + j;
      if (smask & (1u << j)) rs = pos;
      const u32 d = pos - rs + (rs == 0 ? carry : 0);
      ww = w_of_dist(d);
      if constexpr (PIECES) pm |= (d % 255 == 0 ? 1u : 0u) << j;
    }
    v.w[j] = (u8)ww;
    sum += ww;
  }
  if constexpr (PIECES) *pieces = pm;
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

struct RsCombine {
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const { return rs_combine(a, b); }
};
struct Add64 {
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const { return a + b; }
};
// scan state of tile t on its own
__device__ __forceinline__ u64 tile_state(const TileSum& s, u64 t, u64 N) {
  const u64 tl = min((u64)RLE_TILE, N - t * RLE_TILE);
  return rs_make(s.allsame, s.fc, s.lc, s.trail % 255, (u32)(tl % 255));
}
// Exclusive Hillis-Steele scan of one value per thread over a CTA of NT threads.  op need not be commutative; 0 is its
// identity.  *total = the combination of all NT values.  sa and sb (NT entries each) are free again on return.
template <u32 NT, class Op>
__device__ __forceinline__ u64 cta_scan_excl(u64 v, u64* sa, u64* sb, Op op, u64* total) {
  const u32 tid = threadIdx.x;
  sa[tid] = v;
  __syncthreads();
  u64* src = sa; u64* dst = sb;
  for (u32 o = 1; o < NT; o <<= 1) {
    u64 x = src[tid];
    if (tid >= o) x = op(src[tid - o], x);
    dst[tid] = x;
    __syncthreads();
    u64* tmp = src; src = dst; dst = tmp;
  }
  const u64 ex = tid ? src[tid - 1] : 0;
  *total = src[NT - 1];
  __syncthreads();
  return ex;
}
// Tile t entered with run state st: carry[t] = the run length carried in (mod 255), prefix[t] = the tile's output size S
// (an add scan turns the sizes into W later).  Returns S and advances st past the tile.
__device__ __forceinline__ u64 tile_carry_step(const TileSum& s, u64 t, u64 N, u64& st, u32* carry, u64* prefix) {
  u32 c = 0;
  if ((st >> 63) && ((st >> 16) & 255) == s.fc) c = (st >> 8) & 255;
  carry[t] = c;
  const u64 S = outfresh((u64)c + s.lead) - outfresh(c) + s.rest;
  prefix[t] = S;
  st = rs_combine(st, tile_state(s, t, N));
  return S;
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
  for (u64 t = t0; t < t1; t++) agg = rs_combine(agg, tile_state(sums[t], t, N));
  // 2. exclusive scan over threads; st0: run state entering the buffer (a share of a larger input)
  u64 all;
  u64 st = rs_combine(st0, cta_scan_excl<RS_THREADS>(agg, sa, sb, RsCombine{}, &all));
  if (tid == 0 && agg_out) *agg_out = all;
  // 3. carries + per-tile output sums (stored in prefix[] for now)
  u64 mysum = 0;
  for (u64 t = t0; t < t1; t++) mysum += tile_carry_step(sums[t], t, N, st, carry, prefix);
  // 4. exclusive add scan of the thread sums
  u64 grand;
  u64 run = W0 + cta_scan_excl<RS_THREADS>(mysum, sa, sb, Add64{}, &grand);
  for (u64 t = t0; t < t1; t++) {
    const u64 S = prefix[t];
    prefix[t] = run;
    run += S;
  }
  if (tid == 0) prefix[ntiles] = W0 + grand;
}

// Multi-CTA version of the same scan for inputs of many tiles (one CTA per RG_TILES tiles, five small launches):
//   g1: per group, the aggregate run state                    g2: exclusive scan of the group aggregates (one CTA)
//   g3: per tile carry + output size S (in prefix[]), group sums   g4: exclusive scan of the group sums (one CTA)
//   g5: prefix[t] = group base + exclusive scan of S inside the group
#define RG_THREADS 256
#define RG_PER 8
#define RG_TILES (RG_THREADS * RG_PER)
__global__ void __launch_bounds__(RG_THREADS)
k_rle_scan_g1(const TileSum* __restrict__ sums, u64 ntiles, u64 N, u64* __restrict__ group_agg) {
  __shared__ u64 sa[RG_THREADS], sb[RG_THREADS];
  const u64 t0 = (u64)blockIdx.x * RG_TILES + (u64)threadIdx.x * RG_PER;
  u64 agg = 0;
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    if (t < ntiles) agg = rs_combine(agg, tile_state(sums[t], t, N));
  }
  u64 total;
  cta_scan_excl<RG_THREADS>(agg, sa, sb, RsCombine{}, &total);
  if (threadIdx.x == 0) group_agg[blockIdx.x] = total;
}
// one CTA: exclusive scan of ngroups values under Op (RsCombine for run states, Add64 for sizes); out[ngroups] = total
template <class Op>
__global__ void __launch_bounds__(RS_THREADS)
k_rle_scan_groups(const u64* __restrict__ in, u32 ngroups, u64* __restrict__ out, u64 init, u64* __restrict__ agg_out) {
  __shared__ u64 sa[RS_THREADS], sb[RS_THREADS];
  const Op op{};
  const u32 tid = threadIdx.x;
  const u32 per = (ngroups + RS_THREADS - 1) / RS_THREADS;
  const u32 g0 = tid * per, g1 = min(ngroups, g0 + per);
  u64 agg = 0;
  for (u32 g = g0; g < g1; g++) agg = op(agg, in[g]);
  u64 all;
  u64 run = op(init, cta_scan_excl<RS_THREADS>(agg, sa, sb, op, &all));
  if (tid == 0 && agg_out) *agg_out = all;  // combination of all groups without `init`
  for (u32 g = g0; g < g1; g++) {
    const u64 v = in[g];
    out[g] = run;
    run = op(run, v);
  }
  if (tid == RS_THREADS - 1) out[ngroups] = op(init, all);
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
    if (t < ntiles) { ts[j] = sums[t]; agg = rs_combine(agg, tile_state(ts[j], t, N)); }
  }
  u64 total;
  u64 st = rs_combine(group_start[blockIdx.x], cta_scan_excl<RG_THREADS>(agg, sa, sb, RsCombine{}, &total));
  u32 mysum = 0;  // <= 2048 tiles x 5120 bytes per group: fits 32 bits
#pragma unroll
  for (u32 j = 0; j < RG_PER; j++) {
    const u64 t = t0 + j;
    if (t < ntiles) mysum += (u32)tile_carry_step(ts[j], t, N, st, carry, prefix);
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

// The largest tile t >= lo with prefix[t] < V.  Whole CTA; see seek_W for the precondition.  Kept out of line: inlined
// twice into k_rle_blocks it made ptxas spill there, and a call per block costs nothing next to the probes' barriers.
__device__ __noinline__ u64 find_tile(const u64* prefix, u64 ntiles, u64 lo, u64 V, BlocksShared& sh) {
  const u32 tid = threadIdx.x;
  u64 hi = ntiles;  // prefix[lo] < V <= prefix[hi]
  {
    // W grows by ~1 per raw byte on ordinary data: try the tile that linear extrapolation predicts
    u64 tg = lo + ((V - prefix[lo]) >> 12);
    if (tg >= ntiles) tg = ntiles - 1;
    const u64 pg = prefix[tg], pg1 = prefix[tg + 1];
    if (pg < V && pg1 >= V) { lo = tg; hi = tg + 1; }
    else if (pg < V) lo = tg;
    else if (tg > lo) hi = tg;
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
  return lo;
}

// W seek: the smallest raw position f with W(f + 1) >= V, and *Wf = W(f + 1).  Whole CTA.  Requires
// prefix[lo] < V <= prefix[ntiles]: then f lies in the tile find_tile returns, and that tile ends at W >= V.
__device__ u64 seek_W(const u8* in, u64 N, const u32* carry, const u64* prefix, u64 ntiles, u64 lo, u64 V, BlocksShared& sh, u64* Wf) {
  const u64 t = find_tile(prefix, ntiles, lo, V, sh);
  TileView v;
  tile_view(in, N, t * RLE_TILE, carry[t], sh.sc, v);
  u32 found = 0xffffffffu;
  u64 acc = prefix[t] + v.excl;
  for (u32 j = 0; j < v.cnt; j++) {
    acc += v.w[j];
    if (acc >= V) { found = threadIdx.x * RT_PER + j; break; }
  }
  const u32 f = block_min256(found, sh.sc.red);
  if (found == f) sh.r64 = acc;  // the thread that owns f
  __syncthreads();
  *Wf = sh.r64;
  __syncthreads();
  return t * RLE_TILE + f;
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
    s = seek_W(in, N, carry, prefix, ntiles, 0, u_start, sh, &Ws) + 1;
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
        u64 We;
        e = seek_W(in, N, carry, prefix, ntiles, b / RLE_TILE, V, sh, &We) + 1;
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

// ---- C (libbz2 flavor) --------------------------------------------------------------------
// libbz2 1.0.8 (bzlib.c add_char_to_block) keeps its run state across blocks, so the pieces it reads -- stretches of
// one byte value, at most 255 long, the 255-chunks of a maximal run -- are those of the whole input, which are exactly
// the phases W is scanned under.  A block holds whole pieces and closes right after the first piece that brings its
// RLE1 size to >= blockSize.  So every block starts on a piece start with W(s) known from the block before: no run is
// re-phased (b == s, ofs == 0), and k_rle_emit writes the block unchanged.  One CTA walks the blocks: per block one
// W seek for the byte whose W reaches W(s) + blockSize, then the end of that byte's piece.
__global__ void __launch_bounds__(RT_THREADS)
k_rle_blocks_libbz2(const u8* __restrict__ in, u64 N, u32 BS, const u32* __restrict__ carry, const u64* __restrict__ prefix, u64 ntiles,
                    BlkInfo* __restrict__ blocks, u32* nblocks_out, u32 maxblocks) {
  __shared__ BlocksShared sh;
  const u32 tid = threadIdx.x;
  const u64 Wtotal = prefix[ntiles];
  u64 s = 0, Ws = prefix[0];
  u32 k = 0;
  while (s < N && k < maxblocks) {
    BlkInfo bi;
    bi.s = s; bi.b = s; bi.Wb = Ws; bi.ofs = 0;
    const u64 V = Ws + BS;
    u64 e, We;
    if (V > Wtotal) {
      e = N; We = Wtotal;
    } else {
      u64 Wf;
      const u64 f = seek_W(in, N, carry, prefix, ntiles, s / RLE_TILE, V, sh, &Wf);
      const u64 t = f / RLE_TILE, tstart = t * RLE_TILE;
      const u32 fo = (u32)(f - tstart);
      // phase of f inside its maximal run: the last byte change at or before f in the tile, else the carry
      u32 ls = 0;
      for (u32 j = 0; j < RT_PER; j++) {
        const u32 pos = tid * RT_PER + j;
        if (pos >= 1 && pos <= fo && in[tstart + pos] != in[tstart + pos - 1]) ls = pos + 1;
      }
      ls = block_max256(ls, sh.sc.red);
      const u32 d = ls ? fo - (ls - 1) : fo + carry[t];
      const u32 r = d % 255 + 1;  // f is byte r of its piece
      const u32 room = 255 - r;   // bytes the piece can still take
      const u8 ch = in[f];
      const u64 p = f + 1 + tid;
      const u32 stop = block_min256((tid < room && p < N && in[p] != ch) ? tid : 0xffffffffu, sh.sc.red);
      e = min(N, f + 1 + (stop == 0xffffffffu ? room : stop));
      const u32 L = r + (u32)(e - f - 1);  // length of the closing piece
      We = Wf - outfresh(r) + outfresh(L);
    }
    bi.e = e; bi.n = (u32)(We - Ws);
    if (tid == 0) blocks[k] = bi;
    k++;
    s = e; Ws = We;
  }
  if (tid == 0) *nblocks_out = k;
}

// ---- E (libbz2 flavor, sharded input) ---------------------------------------------------------
// The libbz2 cut in W space: block k + 1 starts at S(k+1) = next(S(k) + M), M = blockSize, where next(x) is the first
// piece start at or after W position x.  A piece holds at most 5 RLE1 bytes, so next(x) - x is 0..4, and the drift
// S(k) - k M grows by at most 4 a block.  A share that does not know the blocks in front of it walks this chain once
// for every drift its first block can have (b2_bzip2_share_cut_table), over a bitmap of the piece starts of share +
// halo in W space; the host then chains the shares and each walks its own entry again (b2_bzip2_plan_share_flavor).
//
// Probe: bit p of `bits` is set when a piece starts at W position W0 + p (W0 = the buffer's W base, prefix[0]).  One
// CTA per tile; the tile's bits are gathered in shared memory, its interior words stored and the two edge words, which
// it may share with its neighbours, OR-ed.  `bits` is zeroed by the caller.  *wshare = W(share_len) - W0 if
// share_len < N (the caller presets W(N) - W0).
#define PROBE_WORDS (RLE_TILE * 5 / 4 / 32 + 2)
__global__ void __launch_bounds__(RT_THREADS)
k_piece_probe(const u8* __restrict__ in, u64 N, const u32* __restrict__ carry, const u64* __restrict__ prefix, u64 share_len,
              u32* __restrict__ bits, u64* __restrict__ wshare) {
  __shared__ TileScratch sc;
  __shared__ u32 sm[PROBE_WORDS];
  const u32 tid = threadIdx.x;
  const u64 t = blockIdx.x, tstart = t * RLE_TILE;
  const u64 base = prefix[t] - prefix[0], end = prefix[t + 1] - prefix[0];
  for (u32 i = tid; i < PROBE_WORDS; i += RT_THREADS) sm[i] = 0;
  TileView v;
  u32 pm;
  tile_view<true>(in, N, tstart, carry[t], sc, v, &pm);  // its first barrier orders the clearing above
  u32 a = (u32)(base & 31) + v.excl;  // bit of sm[] at the thread's first byte
  for (u32 j = 0; j < v.cnt; j++) {
    if ((pm >> j) & 1) atomicOr(&sm[a >> 5], 1u << (a & 31));
    if (tstart + tid * RT_PER + j == share_len) *wshare = (base & ~(u64)31) + a;
    a += v.w[j];
  }
  __syncthreads();
  const u64 w0 = base >> 5;
  const u32 nw = (u32)(((end + 31) >> 5) - w0);
  for (u32 i = tid; i < nw; i += RT_THREADS) {
    const u32 x = sm[i];
    if (i == 0 || i == nw - 1) { if (x) atomicOr(&bits[w0 + i], x); }
    else bits[w0 + i] = x;
  }
}

// next(x) inside the buffer: the first piece start in [x, x + 4] (W positions relative to W0), or CUT_NONE when there
// is none before wbuf (the piece that holds x goes on past the buffer, or x is past it).  bits has wbuf / 32 + 2 words.
#define CUT_NONE (~0ull)
__device__ __forceinline__ u64 next_piece(const u32* __restrict__ bits, u64 wbuf, u64 x) {
  if (x >= wbuf) return CUT_NONE;
  const u64 wi = x >> 5;
  const u64 two = (u64)bits[wi] | ((u64)bits[wi + 1] << 32);
  const u64 m = (two >> (x & 31)) & 0x1f;
  return m ? x + (u64)(__ffsll((long long)m) - 1) : CUT_NONE;  // no piece starts at wbuf or later
}
__device__ __forceinline__ bool is_piece(const u32* __restrict__ bits, u64 p) { return (bits[p >> 5] >> (p & 31)) & 1; }

// One thread per entry drift d in [0, dmax]: the first block at or after the share's W start w_in with drift d is
// block k = ceil((w_in - d) / M) (0 if d >= w_in), starting at S = k M + d.  The walk counts the blocks that start in
// the share (S - w_in < wshare) and stops at the first one that does not.  Row d = {k, blocks, drift of the block
// after them, flags} (include/b2bz.h, B2_CUT_*).
__global__ void k_cut_table(const u32* __restrict__ bits, u64 wbuf, u64 wshare, u64 w_in, u32 M, u64 dmax, uint4* __restrict__ table) {
  const u64 d = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (d > dmax) return;
  const u64 k = w_in > d ? (w_in - d + M - 1) / M : 0;
  u64 S = k * M + d - w_in;
  u32 flags = 0, cnt = 0;
  if (S < wbuf && !is_piece(bits, S)) flags |= B2_CUT_NOT_PIECE;
  while (S < wshare) {
    cnt++;
    const u64 nx = next_piece(bits, wbuf, S + M);
    if (cnt == 1 && nx == S + M) flags |= B2_CUT_STEP_EXACT;
    if (nx == CUT_NONE) { flags |= B2_CUT_BUF_END; break; }
    S = nx;
  }
  const u32 exit_d = (flags & B2_CUT_BUF_END) ? 0u : (u32)(w_in + S - (k + cnt) * M);
  table[d] = make_uint4((u32)k, cnt, exit_d, flags);
}

// The chain of one entry: starts[0] = S0, starts[i + 1] = next(starts[i] + M) for up to `count` blocks; a block whose
// next start lies past the buffer ends at the buffer's end (wbuf), and the walk stops there.  *ncut = blocks walked.
__global__ void k_cut_chain(const u32* __restrict__ bits, u64 wbuf, u64 S0, u32 M, u64 count, u64* __restrict__ starts, u64* __restrict__ ncut) {
  u64 S = S0, i = 0;
  starts[0] = S;
  if (S < wbuf && is_piece(bits, S)) {
    while (i < count) {
      u64 nx = next_piece(bits, wbuf, S + M);
      if (nx == CUT_NONE) nx = wbuf;
      starts[++i] = nx;
      S = nx;
      if (S == wbuf) break;
    }
  }
  *ncut = i;
}

// One CTA per W position S = W0 + starts[i]: raw[i] = the raw position of the piece that starts there (the smallest
// position whose inclusive W exceeds S), N for S >= W(N).
__global__ void __launch_bounds__(RT_THREADS)
k_w_to_raw(const u8* __restrict__ in, u64 N, const u32* __restrict__ carry, const u64* __restrict__ prefix, u64 ntiles,
           const u64* __restrict__ starts, u64* __restrict__ raw) {
  __shared__ BlocksShared sh;
  const u64 S = prefix[0] + starts[blockIdx.x];
  u64 f = N, Wf;
  if (S < prefix[ntiles]) f = seek_W(in, N, carry, prefix, ntiles, 0, S + 1, sh, &Wf);
  if (threadIdx.x == 0) raw[blockIdx.x] = f;
}

// ---- CRC constants ---------------------------------------------------------------------------
// The block CRC is linear: the pure polynomial remainder R (no init, no final XOR) of a byte string is the XOR of the
// remainders of its pieces, each multiplied by x^(8 * bytes after the piece); leading zero bytes add nothing.
#define CRC_POLY 0x04c11db7u
__host__ __device__ __forceinline__ u32 gf_mulmod(u32 a, u32 b) {
  u32 r = 0;
  for (int i = 31; i >= 0; i--) {
    r = (r << 1) ^ ((r & 0x80000000u) ? CRC_POLY : 0u);
    if ((b >> i) & 1) r ^= a;
  }
  return r;
}
#define EMIT_TILES 4                       // raw tiles of one block per k_rle_emit CTA
#define EMIT_SPAN (EMIT_TILES * RLE_TILE)
#define EMIT_SEG 64                        // raw bytes of the span whose remainder one emit thread computes
static_assert(EMIT_SEG * RT_THREADS == EMIT_SPAN, "every emit thread takes one segment of the span");
// x^(8 * RLE_TILE * k) for every k a block can need.  RLE1 turns at most 51 raw bytes into one output byte (a run of
// 255 equal bytes, the costliest, emits 5), and a block's output stops at most one count byte past blockSize, so at
// level 9 a block spans at most 51 * 899982 = 45,899,082 raw bytes, and e / RLE_TILE - s / RLE_TILE <= 11206 tile
// edges.  rle1_materialize checks every block against the table's size.
#define CRC_TILE_POWS 11264
struct CrcConsts {
  u32 slice[4][256];  // slice[0] = byte table; slice[k][i] = slice[k-1][i] after one more zero byte (slicing by 4)
  u32 pow[48];        // pow[i] = x^(8 * 2^i) mod P
  u32 pow_byte[EMIT_SEG + 1];            // x^(8 * r), r = 0..EMIT_SEG
  u32 pow_seg[EMIT_SPAN / EMIT_SEG];     // x^(8 * EMIT_SEG * m)
  u32 pow_tile[CRC_TILE_POWS];           // x^(8 * RLE_TILE * k)
};
static void make_crc_consts(CrcConsts& c) {
  for (u32 i = 0; i < 256; i++) {
    u32 v = i << 24;
    for (int k = 0; k < 8; k++) v = (v & 0x80000000u) ? (v << 1) ^ CRC_POLY : (v << 1);
    c.slice[0][i] = v;
  }
  for (int k = 1; k < 4; k++)
    for (u32 i = 0; i < 256; i++) {
      const u32 prev = c.slice[k - 1][i];
      c.slice[k][i] = (prev << 8) ^ c.slice[0][prev >> 24];
    }
  c.pow[0] = 0x100;  // x^8
  for (int i = 1; i < 48; i++) c.pow[i] = gf_mulmod(c.pow[i - 1], c.pow[i - 1]);
  c.pow_byte[0] = 1u;  // bit i of a register value is the coefficient of x^i, so the polynomial 1 is 0x1
  for (int r = 1; r <= EMIT_SEG; r++) c.pow_byte[r] = gf_mulmod(c.pow_byte[r - 1], c.pow[0]);
  c.pow_seg[0] = 1u;
  for (int m = 1; m < EMIT_SPAN / EMIT_SEG; m++) c.pow_seg[m] = gf_mulmod(c.pow_seg[m - 1], c.pow_byte[EMIT_SEG]);
  const u32 xtile = c.pow[12];  // 2^12 = RLE_TILE bytes
  c.pow_tile[0] = 1u;
  for (int k = 1; k < CRC_TILE_POWS; k++) c.pow_tile[k] = gf_mulmod(c.pow_tile[k - 1], xtile);
}
static_assert(RLE_TILE == 1 << 12, "pow_tile is built from pow[12]");
// in global memory: the tables are read at per-thread indices, which constant memory would serialise
__device__ CrcConsts g_crc;
static bool g_crc_ready = false;
static void crc_setup() {
  if (g_crc_ready) return;
  static CrcConsts h;
  make_crc_consts(h);
  CUDA_CHECK(cudaMemcpyToSymbol(g_crc, &h, sizeof h));
  g_crc_ready = true;
}
// x^(8*bytes) mod P
__device__ __forceinline__ u32 crc_xpow(u64 bytes) {
  u32 r = 1u;
  for (int i = 0; bytes; i++, bytes >>= 1)
    if (bytes & 1) r = gf_mulmod(r, g_crc.pow[i]);
  return r;
}
// every thread of the CTA copies the four slicing tables to shared memory (blockDim.x == 256)
__device__ __forceinline__ void crc_load_tables(u32 (*tab)[256]) {
#pragma unroll
  for (int k = 0; k < 4; k++) tab[k][threadIdx.x] = g_crc.slice[k][threadIdx.x];
}
// four message bytes per dependent step: w holds them little-endian, and the stream is MSB first
__device__ __forceinline__ u32 crc_step4(u32 crc, u32 w, const u32 (*tab)[256]) {
  const u32 x = crc ^ __byte_perm(w, 0, 0x0123);
  return tab[3][x >> 24] ^ tab[2][(x >> 16) & 0xff] ^ tab[1][(x >> 8) & 0xff] ^ tab[0][x & 0xff];
}
__device__ __forceinline__ u32 crc_step1(u32 crc, u32 byte, const u32 (*tab)[256]) { return (crc << 8) ^ tab[0][((crc >> 24) ^ byte) & 0xff]; }

// ---- D ---------------------------------------------------------------------------------
// One CTA per span of up to EMIT_TILES tiles of one block; map[CTA] = (block, span index inside the block).
// The span's raw bytes are staged in shared memory, 16 per word: word w (span offset 16 w, w >= -8) lives at
// stage[emit_sw(w)].  The swizzle keeps both access patterns free of bank conflicts: eight threads reading eight
// consecutive words, and eight threads reading word j of eight consecutive EMIT_SEG-byte segments.
#define EMIT_STAGE_WORDS (EMIT_SPAN / 16 + 16)
__device__ __forceinline__ u32 emit_sw(int w) {
  const u32 v = (u32)(w + 8);
  return v ^ ((v >> 3) & 3);
}
__device__ __forceinline__ u32 stage_byte(const uint4* stage, u32 p) {
  return reinterpret_cast<const u8*>(stage)[16 * emit_sw((int)(p >> 4)) + (p & 15)];
}
// 16 raw bytes at `off` (zero past N), with aligned 16-byte loads when the buffer allows them
__device__ __forceinline__ uint4 load16(const u8* __restrict__ in, u64 N, u64 off) {
  const u8* p = in + off;
  if (off + 16 <= N && (((size_t)p) & 15) == 0) return *reinterpret_cast<const uint4*>(p);
  u32 a[4] = {0, 0, 0, 0};
  for (u32 j = 0; j < 16 && off + j < N; j++) a[j >> 2] |= (u32)p[j] << (8 * (j & 3));
  return make_uint4(a[0], a[1], a[2], a[3]);
}
// A run of plain tiles: raw span bytes [ra, ra + cnt) go to output bytes [o0, o0 + cnt) of Tb.  Every thread builds
// destination-aligned 16-byte words from two staged words with funnel shifts; only the two edge words go byte by byte.
__device__ void emit_copy(const uint4* stage, u32 ra, u64 o0, u32 cnt, u8* __restrict__ Tb) {
  const u32 fo = (u32)(o0 & 15u);
  const int delta = (int)ra - (int)fo;  // span offset of the first byte of destination word 0
  const int wq = delta >> 4;            // floor
  const u32 sh = (u32)delta & 15u, q = sh >> 2, bs = 8 * (sh & 3);
  const u32 end = fo + cnt, nw = (end + 15) >> 4;
  u8* dst = Tb + (o0 - fo);  // 16-byte aligned
  for (u32 k = threadIdx.x; k < nw; k += RT_THREADS) {
    const u32 b0 = 16 * k;
    if (b0 >= fo && b0 + 16 <= end) {
      const uint4 lo = stage[emit_sw(wq + (int)k)], hi = stage[emit_sw(wq + (int)k + 1)];
      const u32 a[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      u32 b[5];
#pragma unroll
      for (int j = 0; j < 5; j++) b[j] = q == 0 ? a[j] : q == 1 ? a[j + 1] : q == 2 ? a[j + 2] : a[j + 3];
      *reinterpret_cast<uint4*>(dst + b0) = make_uint4(__funnelshift_r(b[0], b[1], bs), __funnelshift_r(b[1], b[2], bs),
                                                       __funnelshift_r(b[2], b[3], bs), __funnelshift_r(b[3], b[4], bs));
    } else {
      for (u32 x = max(b0, fo); x < min(b0 + 16, end); x++) dst[x] = (u8)stage_byte(stage, (u32)(delta + (int)x));
    }
  }
}
// A tile with runs of four or more: every raw byte of the thread computes its output position and writes its literal
// (+ count byte).
__device__ void emit_general(const u8* __restrict__ in, const BlkInfo& bi, u64 tstart, u64 Pt, const TileView& v, u8* __restrict__ Tb) {
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
// Emits the span's part [X0, X1) of the block and folds the CRC of those raw bytes (all of them, also run bytes that
// emit nothing and bytes past the block's output length) into acc, in the layout k_crc_final reads with unit RLE_TILE.
// 40 registers (no spills), 21 KiB of shared memory: six CTAs per SM
__global__ void __launch_bounds__(RT_THREADS, 6)
k_rle_emit(const u8* __restrict__ in, u64 N, const u32* __restrict__ carry, const u64* __restrict__ prefix, const u8* __restrict__ plain,
           const BlkInfo* __restrict__ blocks, u32 first, const uint2* __restrict__ map, u8* __restrict__ T, u32* __restrict__ acc) {
  __shared__ __align__(16) uint4 stage[EMIT_STAGE_WORDS];
  __shared__ u32 tab[4][256];
  __shared__ TileScratch sc;
  __shared__ u32 red[RT_THREADS / 32 + 1];
  const u32 tid = threadIdx.x;
  crc_load_tables(tab);
  const uint2 m = map[blockIdx.x];
  const BlkInfo bi = blocks[first + m.x];
  const u64 t0 = bi.s / RLE_TILE + (u64)m.y * EMIT_TILES;
  const u32 ntl = (u32)min((u64)EMIT_TILES, (bi.e - 1) / RLE_TILE - t0 + 1);
  const u64 sstart = t0 * RLE_TILE;
  const u64 X0 = max(bi.s, sstart), X1 = min(bi.e, sstart + (u64)ntl * RLE_TILE);
  u8* Tb = T + ((size_t)m.x << SEG_SHIFT);
  u32 pmask = 0;
#pragma unroll
  for (u32 i = 0; i < EMIT_TILES; i++)
    if (i < ntl && plain[t0 + i]) pmask |= 1u << i;
  // 1. stage the raw bytes; tiles with long runs are emitted here, from their TileView
  uint4 q[EMIT_TILES];
#pragma unroll
  for (u32 i = 0; i < EMIT_TILES; i++)
    if ((pmask >> i) & 1) q[i] = load16(in, N, sstart + i * RLE_TILE + 16 * tid);
#pragma unroll
  for (u32 i = 0; i < EMIT_TILES; i++)
    if ((pmask >> i) & 1) stage[emit_sw((int)(i * RT_THREADS + tid))] = q[i];
  for (u32 i = 0; i < ntl; i++) {
    if ((pmask >> i) & 1) continue;
    const u64 t = t0 + i, tstart = t * RLE_TILE;
    TileView v;
    tile_view(in, N, tstart, carry[t], sc, v);
    emit_general(in, bi, tstart, prefix[t], v, Tb);
    u32 a[4] = {0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < RT_PER; j++) a[j >> 2] |= (u32)v.by[j] << (8 * (j & 3));
    stage[emit_sw((int)(i * RT_THREADS + tid))] = make_uint4(a[0], a[1], a[2], a[3]);
  }
  __syncthreads();
  // 2. runs of plain tiles: every raw byte emits itself (w = 1) whatever the phase, so the run's part of the block is a
  // byte copy to output position (x - x0) + o0 (o0 by the same formulas as emit_general, with w = 1 everywhere)
  for (u32 i = 0; i < ntl;) {
    if (!((pmask >> i) & 1)) { i++; continue; }
    u32 j = i + 1;
    while (j < ntl && ((pmask >> j) & 1)) j++;
    const u64 tstart = sstart + (u64)i * RLE_TILE;
    const u64 x0 = max(X0, tstart), x1 = min(X1, sstart + (u64)j * RLE_TILE);
    const u64 o0 = x0 < bi.b ? (x0 - bi.s) : (u64)bi.ofs + (prefix[t0 + i] + (x0 - tstart) - bi.Wb);
    if (o0 < bi.n) emit_copy(stage, (u32)(x0 - sstart), o0, (u32)min(x1 - x0, (u64)bi.n - o0), Tb);
    i = j;
  }
  // 3. CRC: thread tid takes the span bytes of [64 tid, 64 tid + 64) that lie in [rx0, rx1).  Bytes before rx0 count as leading zeros;
  // the segment that holds rx1 - 1 (segment L) stops exactly at rx1, so its remainder needs no shift.
  const u32 rx0 = (u32)(X0 - sstart), rx1 = (u32)(X1 - sstart);
  const u32 seg0 = tid * EMIT_SEG;
  u32 R = 0;
  if (seg0 < rx1 && seg0 + EMIT_SEG > rx0) {
#pragma unroll
    for (u32 j4 = 0; j4 < EMIT_SEG / 16; j4++) {
      const uint4 s4 = stage[emit_sw((int)(tid * (EMIT_SEG / 16) + j4))];
      const u32 a[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
      for (u32 w = 0; w < 4; w++) {
        const u32 pos = seg0 + 16 * j4 + 4 * w;
        u32 x = a[w];
        if (pos < rx0) x = rx0 - pos >= 4 ? 0u : x & (0xffffffffu << (8 * (rx0 - pos)));
        if (pos + 4 <= rx1) R = crc_step4(R, x, tab);
        else
          for (u32 b = pos; b < rx1; b++) R = crc_step1(R, x >> (8 * (b - pos)), tab);
      }
    }
  }
  // segment i < L is followed by r + 64 (L - 1 - i) bytes of the span, r = rx1 - 64 L in 1..64
  const u32 L = (rx1 - 1) / EMIT_SEG, r = rx1 - L * EMIT_SEG;
  u32 c = tid < L ? gf_mulmod(R, g_crc.pow_seg[L - 1 - tid]) : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(FULL_MASK, c, o);
  if (lane_id() == 0) red[tid >> 5] = c;
  if (tid == L) red[RT_THREADS / 32] = R;
  __syncthreads();
  if (tid == 0) {
    u32 S = 0;
#pragma unroll
    for (int w = 0; w < RT_THREADS / 32; w++) S ^= red[w];
    u32 tot = gf_mulmod(S, g_crc.pow_byte[r]) ^ red[RT_THREADS / 32];
    if (X1 == bi.e) {
      atomicXor(&acc[2 * m.x + 1], tot);
    } else {
      // X1 is a tile edge k tiles before the last tile edge at or before e
      const u64 k = bi.e / RLE_TILE - X1 / RLE_TILE;
      if (k) tot = gf_mulmod(tot, g_crc.pow_tile[k]);
      atomicXor(&acc[2 * m.x], tot);
    }
  }
}
__global__ void k_emit_map(const u32* __restrict__ sbase, uint2* __restrict__ map) {
  const u32 k = blockIdx.x, b = sbase[k], n = sbase[k + 1] - b;
  for (u32 j = threadIdx.x; j < n; j += blockDim.x) map[b + j] = make_uint2(k, j);
}

// ---- CRC of byte ranges (decoder, b2_crc32) ---------------------------------------------------
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
  __shared__ u32 tab[4][256];
  crc_load_tables(tab);
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
      crc = crc_step4(crc, q.x, tab);
      crc = crc_step4(crc, q.y, tab);
      crc = crc_step4(crc, q.z, tab);
      crc = crc_step4(crc, q.w, tab);
    }
  } else {
    for (u32 i = 0; i < len; i++) crc = crc_step1(crc, p[i], tab);
  }
  if (pend == bi.e) {
    atomicXor(&acc[2 * lo + 1], crc);
  } else {
    const u64 k = (bi.e - pend) / CRC_PIECE;
    if (k) crc = gf_mulmod(crc, crc_xpow(k * CRC_PIECE));
    atomicXor(&acc[2 * lo], crc);
  }
}
// acc[2k] holds the parts of block k that end on a unit edge, shifted to the last edge at or before e' = e + mis;
// acc[2k+1] the part that ends the block
__global__ void k_crc_final(const BlkInfo* __restrict__ blocks, u32 first, u32 count, const u32* __restrict__ acc, u32 unit, u32 mis,
                            u32* __restrict__ crc_out) {
  u32 k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const BlkInfo bi = blocks[first + k];
  const u64 len = bi.e - bi.s;
  const u32 body = gf_mulmod(acc[2 * k], crc_xpow((bi.e + mis) % unit)) ^ acc[2 * k + 1];
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
  const u32 mis = (u32)((size_t)d_p & (CRC_PIECE - 1));
  const u64 pieces = crc_piece_count(0, n, mis);
  if (pieces) {
    k_crc_pieces<<<(unsigned)((pieces + 255) / 256), 256, 0, c.stream>>>(d_p, db, 0, 1, pb, pieces, acc);
    KLAUNCH(c); KCHECK();
  }
  k_crc_final<<<1, 32, 0, c.stream>>>(db, 0, 1, acc, CRC_PIECE, mis, out);
  KLAUNCH(c); KCHECK();
  u32 h = 0;
  c.to_host(&h, out, 4);
  c.sync();
  return h;
}

// ---- host drivers ---------------------------------------------------------------------------
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

void rle1_scan_tiles(Ctx& c, const u8* d_in, size_t n, Rle1Plan& plan, u64 st0, u64 W0, u64* summary) {
  crc_setup();
  StageScope s(c, ST_RLE1);
  if (n == 0) return;
  const u64 ntiles = (n + RLE_TILE - 1) / RLE_TILE;
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
    k_rle_scan_groups<RsCombine><<<1, RS_THREADS, 0, c.stream>>>(gagg, ng, gstart, st0, dagg);
    KLAUNCH(c); KCHECK();
    k_rle_scan_g3<<<ng, RG_THREADS, 0, c.stream>>>(sums, ntiles, n, gstart, plan.tile_carry, plan.tile_prefix, gsum);
    KLAUNCH(c); KCHECK();
    k_rle_scan_groups<Add64><<<1, RS_THREADS, 0, c.stream>>>(gsum, ng, gbase, W0, nullptr);
    KLAUNCH(c); KCHECK();
    k_rle_scan_g5<<<ng, RG_THREADS, 0, c.stream>>>(ntiles, gbase, ng, plan.tile_prefix);
    KLAUNCH(c); KCHECK();
  }
  if (summary) {
    k_share_lead<<<1, 32, 0, c.stream>>>(sums, ntiles, dagg.p + 1);
    KLAUNCH(c); KCHECK();
    c.to_host(summary, dagg, 16);
  }
  c.to_host(&plan.w_total, plan.tile_prefix.p + ntiles, 8);
  c.sync();
}

// The blocks a single-CTA walk wrote to plan.blocks, and their count (*dnb), into plan.h_blocks and plan.nblocks.
static void fetch_blocks(Ctx& c, Rle1Plan& plan, const u32* dnb) {
  u32 nb = 0;
  c.to_host(&nb, dnb, 4);
  c.sync();
  plan.nblocks = nb;
  plan.h_blocks.resize(nb);
  if (nb) c.to_host(plan.h_blocks.data(), plan.blocks, sizeof(BlkInfo) * nb);
  c.sync();
}
// exact: every block of the buffer.  Otherwise blocks [first, first+count) of the whole input, walked from the
// speculative boundary W = first * BS (see k_rle_blocks); plan.first_index records the global index of h_blocks[0].
static void cut_blocks(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan, bool exact, size_t first, size_t count) {
  StageScope s(c, ST_RLE1);
  if (n == 0) return;
  const u32 BS = rle1_block_size(level);
  const u64 ntiles = (n + RLE_TILE - 1) / RLE_TILE;
  u32 maxblocks = (u32)(n / ((u64)BS * 4 / 5) + 2);
  u64 u_start = 0;
  if (!exact) {
    maxblocks = (u32)std::min<size_t>(maxblocks, count);
    u_start = (u64)first * BS;
    plan.first_index = first;
    if (maxblocks == 0) return;
  }
  plan.blocks.alloc(c, maxblocks);
  // many blocks: walk P segments in parallel first (see k_rle_blocks)
  const u32 total = (u32)plan.total_guess(level);
  const u32 rfirst = exact ? 0u : (u32)first, rcount = exact ? total : maxblocks;
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
  fetch_blocks(c, plan, dnb);
}
void rle1_cut_range(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan, size_t first, size_t count) {
  cut_blocks(c, d_in, n, level, plan, false, first, count);
}
// libbz2 flavor: every block of the buffer, walked by one CTA (see k_rle_blocks_libbz2).  A block holds at least
// blockSize RLE1 bytes and RLE1 makes at most 5 of 4 raw bytes, so there are at most n / (4 BS / 5) + 1 blocks.
static void cut_blocks_libbz2(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan) {
  StageScope s(c, ST_RLE1);
  if (n == 0) return;
  const u32 BS = rle1_block_size(level);
  const u64 ntiles = (n + RLE_TILE - 1) / RLE_TILE;
  const u32 maxblocks = (u32)(n / ((u64)BS * 4 / 5) + 2);
  plan.blocks.alloc(c, maxblocks);
  c.stats.rle_walk_serial++;
  DBuf<u32> dnb(c, 1);
  k_rle_blocks_libbz2<<<1, RT_THREADS, 0, c.stream>>>(d_in, n, BS, plan.tile_carry, plan.tile_prefix, ntiles, plan.blocks, dnb, maxblocks);
  KLAUNCH(c); KCHECK();
  fetch_blocks(c, plan, dnb);
}
// libbz2 flavor over a share buffer: the piece-start bitmap (k_piece_probe) of a scanned plan; wbuf / wshare = W of the
// buffer's / share's end relative to the buffer's W base.
struct PieceMap {
  DBuf<u32> bits;
  u64 wbuf = 0, wshare = 0;
};
static void piece_map(Ctx& c, const u8* d_buf, size_t n, size_t share_len, const Rle1Plan& plan, u64 W0, PieceMap& pm) {
  StageScope s(c, ST_RLE1);
  pm.wbuf = plan.w_total - W0;
  pm.wshare = pm.wbuf;
  const u64 nwords = pm.wbuf / 32 + 2;
  pm.bits.alloc(c, nwords);
  CUDA_CHECK(cudaMemsetAsync(pm.bits, 0, 4 * nwords, c.stream));
  const u64 ntiles = (n + RLE_TILE - 1) / RLE_TILE;
  DBuf<u64> dws(c, 1);
  c.to_device(dws, &pm.wshare, 8);
  k_piece_probe<<<(unsigned)ntiles, RT_THREADS, 0, c.stream>>>(d_buf, n, plan.tile_carry, plan.tile_prefix, share_len, pm.bits, dws);
  KLAUNCH(c); KCHECK();
  c.to_host(&pm.wshare, dws, 8);
  c.sync();
}
// The tile scan and piece bitmap of the last b2_bzip2_share_cut_table.  The b2_bzip2_plan_share_flavor that follows on
// the same (buffer, length, run state, W base) walks its entry over them instead of scanning and probing the share again.
struct ShareProbe {
  Rle1Plan plan;
  PieceMap pm;
  const u8* ptr = nullptr;
  size_t n = 0;
  u64 st0 = 0, W0 = 0;
};
static std::optional<ShareProbe> g_probe;
void rle1_release_share_probe() { g_probe.reset(); }
static void share_probe(Ctx& c, const u8* d_buf, size_t n, u64 st0, u64 W0, size_t share_len, ShareProbe& p) {
  p.ptr = d_buf; p.n = n; p.st0 = st0; p.W0 = W0;
  rle1_scan_tiles(c, d_buf, n, p.plan, st0, W0);
  piece_map(c, d_buf, n, share_len, p.plan, W0, p.pm);
}
void rle1_share_cut_table(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t share_len, u64 dmax, u32* h_table) {
  g_probe.reset();
  const u32 M = rle1_block_size(level);
  if (n == 0) {  // nothing starts in an empty buffer: every entry passes through
    for (u64 d = 0; d <= dmax; d++) {
      const u64 k = W0 > d ? (W0 - d + M - 1) / M : 0;
      u32* row = h_table + 4 * d;
      row[0] = (u32)k; row[1] = 0; row[2] = (u32)d; row[3] = 0;
    }
    return;
  }
  ShareProbe p;
  share_probe(c, d_buf, n, st0, W0, share_len, p);
  StageScope s(c, ST_RLE1);
  DBuf<uint4> dt(c, dmax + 1);
  k_cut_table<<<(unsigned)((dmax + 128) / 128), 128, 0, c.stream>>>(p.pm.bits, p.pm.wbuf, p.pm.wshare, W0, M, dmax, dt);
  KLAUNCH(c); KCHECK();
  c.to_host(h_table, dt, 16 * (dmax + 1));
  c.sync();
  g_probe = std::move(p);
}
// The blocks [first, first + count) of the whole input whose first block starts at W = first * M + drift, inside the
// share buffer d_buf[0, n) entered with run state st0 and W base W0, in the form k_rle_blocks_libbz2 writes (b == s,
// ofs == 0).  The scan and bitmap of the table call before it are reused when they are of the same buffer and entry
// state.  Fewer blocks are cut when the entry is not a piece start or the buffer ends first (its last block then ends at
// the buffer's end).
void rle1_cut_share_libbz2(Ctx& c, const u8* d_buf, size_t n, int level, u64 st0, u64 W0, size_t first, u64 drift, size_t count,
                           Rle1Plan& plan) {
  std::optional<ShareProbe> p;
  if (g_probe && g_probe->ptr == d_buf && g_probe->n == n && g_probe->st0 == st0 && g_probe->W0 == W0) p = std::move(g_probe);
  g_probe.reset();
  const u32 M = rle1_block_size(level);
  const u64 S0 = (u64)first * M + drift;
  if (!p && (n == 0 || count == 0 || S0 < W0)) {  // nothing to cut: only W at the buffer's end is asked for
    rle1_scan_tiles(c, d_buf, n, plan, st0, W0);
  } else if (!p) {
    p.emplace();
    share_probe(c, d_buf, n, st0, W0, n, *p);
  }
  if (p) plan = std::move(p->plan);
  plan.first_index = first;
  plan.nblocks = 0;
  plan.h_blocks.clear();
  if (n == 0 || count == 0 || S0 < W0) return;
  const PieceMap& pm = p->pm;
  StageScope s(c, ST_RLE1);
  const u64 ntiles = (n + RLE_TILE - 1) / RLE_TILE;
  count = std::min<u64>(count, pm.wbuf / M + 1);  // a block holds at least M RLE1 bytes, except one that ends the buffer
  DBuf<u64> starts(c, count + 1), raw(c, count + 1), dn(c, 1);
  k_cut_chain<<<1, 1, 0, c.stream>>>(pm.bits, pm.wbuf, S0 - W0, M, count, starts, dn);
  KLAUNCH(c); KCHECK();
  u64 nb = 0;
  c.to_host(&nb, dn, 8);
  c.sync();
  if (nb == 0) return;
  k_w_to_raw<<<(unsigned)(nb + 1), RT_THREADS, 0, c.stream>>>(d_buf, n, plan.tile_carry, plan.tile_prefix, ntiles, starts, raw);
  KLAUNCH(c); KCHECK();
  std::vector<u64> hs(nb + 1), hr(nb + 1);
  c.to_host(hs.data(), starts, 8 * (nb + 1));
  c.to_host(hr.data(), raw, 8 * (nb + 1));
  c.sync();
  plan.h_blocks.resize(nb);
  for (u64 i = 0; i < nb; i++) {
    BlkInfo& bi = plan.h_blocks[i];
    bi.s = hr[i]; bi.e = hr[i + 1]; bi.b = bi.s; bi.Wb = W0 + hs[i]; bi.ofs = 0; bi.n = (u32)(hs[i + 1] - hs[i]);
  }
  plan.blocks.alloc(c, nb);
  c.to_device(plan.blocks, plan.h_blocks.data(), sizeof(BlkInfo) * nb);
  plan.nblocks = nb;
  c.sync();
}
void rle1_plan(Ctx& c, const u8* d_in, size_t n, int level, Rle1Plan& plan) {
  rle1_scan_tiles(c, d_in, n, plan);
  if (c.bz_flavor == B2_BZ2_LIBBZ2) cut_blocks_libbz2(c, d_in, n, level, plan);
  else cut_blocks(c, d_in, n, level, plan, true, 0, 0);
}
void rle1_materialize(Ctx& c, const u8* d_in, size_t n, const Rle1Plan& plan, size_t first, size_t count, u8* d_T, u32* d_n, u32* d_crc) {
  if (count == 0) return;
  crc_setup();
  std::vector<u32> sbase(count + 1);  // first emit CTA of every block
  std::vector<u32> hn(count);
  u64 ss = 0;
  for (size_t k = 0; k < count; k++) {
    const BlkInfo& bi = plan.h_blocks[first + k];
    const u64 ta = bi.s / RLE_TILE, tb = (bi.e - 1) / RLE_TILE;
    if (bi.e / RLE_TILE - ta >= CRC_TILE_POWS) throw B2Error{B2_ERR_CUDA, "internal error: RLE1 block longer than the CRC shift table"};
    sbase[k] = (u32)ss;
    ss += (tb - ta + EMIT_TILES) / EMIT_TILES;
    hn[k] = bi.n;
  }
  sbase[count] = (u32)ss;
  DBuf<u32> dsb(c, count + 1);
  DBuf<uint2> map(c, ss);
  DBuf<u32> acc(c, 2 * count);
  c.to_device(dsb, sbase.data(), 4 * (count + 1));
  c.to_device(d_n, hn.data(), 4 * count);
  CUDA_CHECK(cudaMemsetAsync(acc, 0, 8 * count, c.stream));
  k_emit_map<<<(unsigned)count, 128, 0, c.stream>>>(dsb, map);
  KLAUNCH(c); KCHECK();
  k_rle_emit<<<(unsigned)ss, RT_THREADS, 0, c.stream>>>(d_in, n, plan.tile_carry, plan.tile_prefix, plan.tile_plain, plan.blocks, (u32)first, map,
                                                       d_T, acc);
  KLAUNCH(c); KCHECK();
  k_crc_final<<<(unsigned)((count + 127) / 128), 128, 0, c.stream>>>(plan.blocks, (u32)first, (u32)count, acc, RLE_TILE, 0, d_crc);
  KLAUNCH(c); KCHECK();
}

// CRC32 of arbitrary byte ranges [s,e) of one device buffer (decoder: per-block CRC of the output).
// h_ranges/d_ranges: only .s and .e are used.
void crc_ranges(Ctx& c, const u8* d_data, const BlkInfo* d_ranges, const std::vector<BlkInfo>& h_ranges, u32* d_crc_out) {
  crc_setup();
  const size_t count = h_ranges.size();
  if (count == 0) return;
  const u32 mis = (u32)((size_t)d_data & (CRC_PIECE - 1));
  std::vector<u64> pbase(count + 1);
  u64 pp = 0;
  for (size_t k = 0; k < count; k++) {
    pbase[k] = pp;
    pp += crc_piece_count(h_ranges[k].s, h_ranges[k].e, mis);
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
  k_crc_final<<<(unsigned)((count + 127) / 128), 128, 0, c.stream>>>(d_ranges, 0, (u32)count, acc, CRC_PIECE, mis, d_crc_out);
  KLAUNCH(c); KCHECK();
  c.sync();
}
