// bwtc.cu -- compressjs' BWTC container (lib/BWTC.js:12-231) on the GPU.
//
// The serial model / range-coder code (bwtc_core.cuh) is checked on its host build against the oracle
// (tests/test_host_api.py::test_bwtc_core_matches_oracle).  The kernels and the orchestration below are checked against
// the oracle on whole streams (tests/test_gpu_zz_bwtc*.py) and on the designed corpus of tests/bwtc_cases.py, whose
// inputs reach every rescale, escape, carry, reciprocal correction and batch seam (tests/test_gpu_zz_bwtc_seams.py).
// The benchmark's `bwtc` leg measures BASELINE config 4 on a 64 MiB slice.
//
// Per block the container needs: sentinel BWT (lib/BWT.js:328-350), MTF over the used bytes, zero runs as
// RUNA/RUNB digits, an adaptive model (Fenwick tree, or the deferred-sum model below level 6) that turns every
// symbol into a (sy_f, lt_f, tot_f) triple, and ONE range coder that runs over the whole file.  The first three are
// the block-parallel kernels of the bzip2 path (bwt.cu in sentinel mode, mtf.cu: the symbol values are identical,
// bzip2 merely appends an end-of-block symbol).  The model is a serial chain per block (k_bwtc_model: one thread per
// block, blocks in parallel), the coder a serial chain per file (k_bwtc_code: one thread; its `range` recurrence
// needs an integer division per symbol and nothing shortens it).  Decode cannot even split model and coder:
// k_bwtc_decode is one thread that decodes a batch of blocks at a time, followed by one batched inverse sentinel BWT
// (decode.cu), so device memory is bounded by the batch.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "enc.h"
#include "bwtc_core.cuh"

void bwt_inverse_sentinel_batch(Ctx& c, const u8* d_L, const u32* h_n, const u32* h_pidx, u32 nb, u8* d_out);

struct BwtcState {
  bc_enc rc;
  u32 overflow;  // a block's triples did not fit its buffer
  u32 pad;
};

// The coder writes each batch into an output window of its own (k_bwtc_window), from the window's byte 0.  Its output is
// final as it is written: a carry lives in `buffer` and the `help` counter of bytes held back, never in a byte already
// out.  The start writes nothing (the first normalisation comes with the next symbol); the finish appends the trailer to
// the window of the last batch.
__global__ void k_bwtc_start(BwtcState* st, u8* out, u64 cap, u32 finalByte, u32 level) {
  if (threadIdx.x || blockIdx.x) return;
  bc_enc_start(&st->rc, out, cap, finalByte);                 // lib/BWTC.js:13-14
  bc_enc_code(&st->rc, bc_triple(1, level, 256));             // encoder.encodeByte(blockSize), :21
  st->overflow = 0;
}

// The zero-run coder writes its symbols in one byte each (NarrowSyms, enc.h); the models read u16 symbols.  One thread
// widens 16 symbols of a block; the masks of the symbols >= 256 are only read in the blocks that have one.
#define WD_THREADS 256
__global__ void __launch_bounds__(WD_THREADS)
k_bwtc_widen(const u8* __restrict__ lo, const unsigned long long* __restrict__ hi, const u32* __restrict__ any_hi, const u32* __restrict__ d_m,
             u32 tps, u16* __restrict__ sym) {
  const u32 b = blockIdx.x / tps;
  const u32 p0 = ((blockIdx.x % tps) * WD_THREADS + threadIdx.x) * 16;
  const u32 m = d_m[b];
  if (p0 >= m) return;
  const uint4 x = *reinterpret_cast<const uint4*>(lo + ((size_t)b << SEG_SHIFT) + p0);  // inside the 1 MiB slot
  u32 w[8] = {__byte_perm(x.x, 0, 0x4140), __byte_perm(x.x, 0, 0x4342), __byte_perm(x.y, 0, 0x4140), __byte_perm(x.y, 0, 0x4342),
              __byte_perm(x.z, 0, 0x4140), __byte_perm(x.z, 0, 0x4342), __byte_perm(x.w, 0, 0x4140), __byte_perm(x.w, 0, 0x4342)};
  if (any_hi[b]) {
    const unsigned long long* h = hi + (size_t)b * SEL_STRIDE;
#pragma unroll
    for (u32 j = 0; j < 16; j++) {
      const u32 p = p0 + j;
      if (p < m && ((h[p / HUFF_GROUP] >> (p % HUFF_GROUP)) & 1u)) w[j >> 1] |= 0x100u << (16 * (j & 1));
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(sym + ((size_t)b << SEG_SHIFT) + p0);   // symbols past m are never read
  dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
  dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// one thread per block (lane 0 of its warp): header + model -> triples
__global__ void __launch_bounds__(32)
k_bwtc_model(const u16* __restrict__ sym, const u32* __restrict__ d_m, const u32* __restrict__ d_n, const u32* __restrict__ d_pidx1,
             const u32* __restrict__ d_used, u32 blockSize, int fast, u64* __restrict__ triples, u32 tcap, u32* __restrict__ tcount) {
  if (threadIdx.x) return;
  const u32 b = blockIdx.x;
  bc_model model;
  bc_emit e;
  e.t = triples + (size_t)b * tcap; e.n = 0; e.cap = tcap;
  const u32 m = d_m[b];
  bc_block_triples(&e, &model, blockSize, d_n[b], d_pidx1[b], d_used + (size_t)b * 8, sym + ((size_t)b << SEG_SHIFT), m ? m - 1 : 0, fast);
  tcount[b] = e.n;
}

// Fenwick model (levels 6..9) with one WARP per block: the tree lives in shared memory, the nodes on the path from a
// leaf to the root sit in different lanes (lane l owns node (numSyms + symbol) >> l), so the cumulative frequency is one
// warp reduction over the left siblings and the update one add per lane; the rescale (every ~128 symbols,
// lib/FenwickModel.js:125-161) runs over the leaves in parallel and re-sums the tree level by level.
// Same triples as bc_fen_encode (bwtc_core.cuh), which the host tests check against the oracle.
struct FenWarp { u32 tree[2 * 260]; };
__device__ __forceinline__ void fenw_sum(u32* tree, u32 numSyms, u32 lane) {
  for (int k = 8; k >= 0; k--) {               // nodes [2^k, 2^(k+1)) only depend on deeper ones
    const u32 lo = 1u << k, hi = min(2u << k, numSyms);
    for (u32 i = lo + lane; i < hi; i += 32) tree[i] = tree[2 * i] + tree[2 * i + 1];
    __syncwarp();
  }
}
__device__ __forceinline__ void fenw_rescale(u32* tree, u32 numSyms, u32 lane) {
  u32 noEscape = 1;
  for (u32 i = lane; i + 1 < numSyms; i += 32) {
    u32 prob = tree[numSyms + i];
    if (prob & BC_ESC_MASK) { noEscape = 0; continue; }
    prob = (prob & BC_SCALE_MASK) >> 1;
    if (prob == 0) { prob = 1; noEscape = 0; }
    tree[numSyms + i] = prob;
  }
  noEscape = __all_sync(FULL_MASK, noEscape);
  if (lane == 0) {
    u32 prob = (tree[2 * numSyms - 1] & BC_SCALE_MASK) >> 1;
    if (noEscape) prob = 0; else if (prob == 0) prob = 1u << 16;
    tree[2 * numSyms - 1] = prob;
  }
  __syncwarp();
  fenw_sum(tree, numSyms, lane);
}
// one trip up the tree (bc_fen_step); every lane returns the triple
__device__ __forceinline__ u64 fenw_step(u32* tree, u32 numSyms, u32 symbol, u32 sy_leaf, int esc, u32 lane) {
  const u32 i = numSyms + symbol;
  u32 mask = BC_SYM_MASK, shift = 16, update = BC_F_PROB_INCR << 16;
  const u32 root = tree[1];
  if (esc) { mask = BC_ESC_MASK; update -= 1; shift = 0; }
  else if (symbol == numSyms - 1 && (root & BC_ESC_MASK) == 1) update = 0u - tree[i];  // the last escape
  const u32 node = lane < 31 ? (i >> lane) : 0u;
  const bool on_path = node > 1;
  u32 contrib = (on_path && (node & 1u)) ? tree[node - 1] : 0u;   // left sibling
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(FULL_MASK, contrib, o);
  __syncwarp();
  if (on_path) tree[node] += update;
  if (lane == 31) tree[1] = root + update;
  __syncwarp();
  const u64 tr = bc_triple((sy_leaf & mask) >> shift, (contrib & mask) >> shift, (root & mask) >> shift);
  if ((((root + update) & BC_SYM_MASK) >> 16) >= BC_F_PROB_MAX) fenw_rescale(tree, numSyms, lane);
  return tr;
}
__global__ void __launch_bounds__(32)
k_bwtc_model_fenwick(const u16* __restrict__ sym, const u32* __restrict__ d_m, const u32* __restrict__ d_n, const u32* __restrict__ d_pidx1,
                     const u32* __restrict__ d_used, u32 blockSize, u64* __restrict__ triples, u32 tcap, u32* __restrict__ tcount) {
  __shared__ FenWarp fw;
  __shared__ u32 s_hdr[2];
  const u32 b = blockIdx.x, lane = threadIdx.x;
  u64* out = triples + (size_t)b * tcap;
  const u32 m = d_m[b], nsym = m ? m - 1 : 0;
  if (lane == 0) {
    bc_emit e;
    e.t = out; e.n = 0; e.cap = tcap;
    s_hdr[1] = bc_block_header(&e, blockSize, d_n[b], d_pidx1[b], d_used + (size_t)b * 8);
    s_hdr[0] = e.n;
  }
  __syncwarp();
  u32 n_out = s_hdr[0];
  const u32 size = s_hdr[1] + 1, numSyms = size + 1;      // bc_fen_init(alphabetSize + 1)
  u32* tree = fw.tree;
  for (u32 i = lane; i < 2 * 260; i += 32) tree[i] = 0;
  __syncwarp();
  for (u32 i = lane; i < size; i += 32) tree[numSyms + i] = 1;
  if (lane == 0) tree[numSyms + size] = BC_F_PROB_INCR << 16;
  __syncwarp();
  fenw_sum(tree, numSyms, lane);
  const u16* sp = sym + ((size_t)b << SEG_SHIFT);
  for (u32 k0 = 0; k0 < nsym; k0 += 32) {
    const u32 mine = k0 + lane < nsym ? sp[k0 + lane] : 0u;
    const u32 cnt = min(32u, nsym - k0);
    for (u32 j = 0; j < cnt; j++) {
      const u32 symbol = __shfl_sync(FULL_MASK, mine, j);
      const u32 sy_leaf = tree[numSyms + symbol];
      u64 t0, t1 = 0;
      u32 produced = 1;
      if ((sy_leaf & BC_SYM_MASK) == 0) {
        const u32 escSym = numSyms - 1;
        t0 = fenw_step(tree, numSyms, escSym, tree[numSyms + escSym], 0, lane);
        t1 = fenw_step(tree, numSyms, symbol, sy_leaf, 1, lane);
        produced = 2;
      } else {
        t0 = fenw_step(tree, numSyms, symbol, sy_leaf, 0, lane);
      }
      if (lane == 0) {
        if (n_out < tcap) out[n_out] = t0;
        if (produced == 2 && n_out + 1 < tcap) out[n_out + 1] = t1;
      }
      n_out += produced;
    }
  }
  if (lane == 0) tcount[b] = n_out;
}

// One warp: the blocks of a batch through the file's range coder.  The recurrence on (low, range) is serial and runs in
// lane 0; what can be taken off its critical path is done by the whole warp, 32 symbols at a time: the coalesced load
// of the triples, their unpacking, and a reciprocal of every total so that the serial step replaces the integer
// division range / tot_f (RangeCoder.js:83) by a multiply-high and an exact correction.
__device__ __forceinline__ void bc_enc_code_fast(bc_enc* rc, u32 sy_f, u32 lt_f, u32 tot_f, u32 magic) {
  bc_enc_normalize(rc);
  u32 r = __umulhi(rc->range, magic);          // floor(range * floor((2^32 - 1) / tot) / 2^32) <= range / tot
  u32 rem = rc->range - r * tot_f;
  while (rem >= tot_f) { r++; rem -= tot_f; }  // at most one step: range <= 2^31 puts r within 1 of range / tot
  const u32 tmp = r * lt_f;
  rc->low += tmp;
  if (lt_f + sy_f < tot_f) rc->range = r * sy_f; else rc->range -= tmp;
}
__global__ void __launch_bounds__(32) k_bwtc_code(BwtcState* st, const u64* __restrict__ triples, const u32* __restrict__ tcount, u32 nblk, u32 tcap) {
  __shared__ uint4 s_t[2][32];   // (sy, lt, tot, reciprocal) of a batch of 32 symbols, double buffered
  const u32 lane = threadIdx.x;
  bc_enc rc = st->rc;
  u32 overflow = st->overflow;
  for (u32 b = 0; b < nblk && !overflow; b++) {
    const u32 n = tcount[b];
    if (n > tcap) { overflow = 1; break; }
    const u64* t = triples + (size_t)b * tcap;
    u64 nxt = lane < n ? t[lane] : 0ull;        // one batch ahead: the load latency hides behind the serial steps
    for (u32 k0 = 0, it = 0; k0 < n; k0 += 32, it++) {
      const u64 tr = nxt;
      if (k0 + 32 + lane < n) nxt = t[k0 + 32 + lane];
      const u32 tot = (u32)(tr >> 42);
      s_t[it & 1][lane] = make_uint4((u32)(tr & 0x1FFFFF), (u32)((tr >> 21) & 0x1FFFFF), tot, tot ? 0xFFFFFFFFu / tot : 0u);
      __syncwarp();
      if (lane == 0) {
        const u32 cnt = min(32u, n - k0);
        const uint4* q = s_t[it & 1];
        uint4 cur = q[0];
        for (u32 j = 0; j < cnt; j++) {
          const uint4 nx = q[(j + 1) & 31];     // fetched one step ahead of its use
          bc_enc_code_fast(&rc, cur.x, cur.y, cur.z, cur.w);
          cur = nx;
        }
      }
      // (no second barrier: the next batch goes to the other buffer, and lane 0 is past this one by the time the
      // buffer is written again two batches later -- all lanes wait for lane 0 at the next __syncwarp)
    }
  }
  if (lane == 0) {
    st->rc = rc;
    st->overflow = overflow;
  }
}

// the next batch's bytes go to `out`, from its byte 0 (a launch of its own: the coder's serial loop stays as it is)
__global__ void k_bwtc_window(BwtcState* st, u8* out, u64 cap) {
  if (threadIdx.x || blockIdx.x) return;
  st->rc.out = out; st->rc.cap = cap; st->rc.n = 0;
}

__global__ void k_bwtc_finish(BwtcState* st) {
  if (threadIdx.x || blockIdx.x) return;
  bc_enc_code(&st->rc, bc_triple(1, 2, 3));                   // "no more blocks", lib/BWTC.js:141
  bc_enc_finish(&st->rc);
}

// The coded size of n raw bytes as BWTC streams usually come out (random bytes grow by under 10 %): the size a result
// buffer or a staging buffer starts with.  Both grow when a stream needs more.
size_t bwtc_bound(size_t n) { return n + n / 8 + (n / 100000 + 2) * 1024 + 64; }

// The most bytes the coder can write for nb blocks of n raw bytes in all, whatever the data: the size of an output
// window, which cannot grow while the coder runs.  A raw byte makes at most one symbol (a zero run of length r makes
// under log2(r + 2) digits) and a symbol at most two triples, an escape and the symbol among the unseen ones.
// - Fenwick model (levels 6..9): a symbol is coded with sy_f >= 1 and tot_f < 0xFF00 (the tree is rescaled as soon as its
//   total reaches 0xFF00), under 16 bits; the literal of an escape with tot_f <= 257 unseen symbols, under 8.01 bits.
// - Deferred-sum model (levels 1..5): tot_f = 256 and sy_f >= 1, at most 8 bits, plus 8.01 bits for the literal.
// - Range coder: r = floor(range / tot_f) with range > 2^23 and tot_f < 2^16 loses at most log2(1 / (1 - 2^-7)) < 0.0113
//   bits per triple; its bytes out are the bits coded plus at most 8 bits of `range` over 8.
// So a raw byte costs under 3 bytes + 0.04 bits at levels 6..9 and 2 bytes + 0.04 bits at levels 1..5: n / 64 bytes
// cover the fractions.  A block's header (the length, the start index and the used-byte tree: under 900 bits) gets 1 KiB.
// Random bytes come to 1.096 n at level 9, and ranks built so that every symbol is coded just after its weight was
// halved to 1.141 n (tests/bwtc_cases.py): more than bwtc_bound gives.
static size_t bwtc_window_bound(size_t n, size_t nb, int fast) { return (fast ? 2 : 3) * n + n / 64 + nb * 1024 + 64; }

// BWTC.compressFile from a host source into a host sink: b2_bwtc_compress / _unsized (the caller's buffer, complete from
// the start, into the result buffer) and b2_bwtc_compress_stream (read and write callbacks).  file_size is the size field
// of the header (Util.js:118-124), or (u64)-1 (a single size byte 0x80) for a stream without a size.
//
// Blocks are fixed cuts of the raw input (level * 100 000 bytes, lib/BWTC.js:24-44), so the input is taken a batch of
// B blocks at a time, straight from `in` into the batch's slots: the device never holds more than one batch of input.
// The coder writes batch k into output window k & 1, sized for the batch's coded bytes plus the `help` bytes still held
// back when it starts.  Batch k's bytes go to the host and to `out` while batch k + 1 runs on the device, and the next
// batch's input is read while batch k runs.  Device memory: one batch of scratch and two windows, whatever the size of
// the input (include/b2bz.h gives the bound).
void bwtc_compress(Ctx& c, StreamIn& in, int level, u64 file_size, StreamOut& out) {
  if (level < 1 || level > 9) level = 9;                      // lib/BWTC.js:16-19
  const u32 blockSize = (u32)level * 100000u;
  const int fast = level <= 5;                                // :22
  u8 hdr[24];
  u32 finalByte = 0;
  const u32 hlen = bc_file_header(hdr, file_size, &finalByte);
  // The first batch sizes the buffers: an input that ends inside it gets only the blocks it has.
  u32 B = c.bwt_batch;
  size_t end = in.fill((size_t)B * blockSize);
  if (in.eof) B = (u32)std::min<size_t>(B, (end + blockSize - 1) / blockSize);
  const u32 tcap = 2 * (blockSize + 1) + 1024;                // every symbol can cost an escape and a literal
  DBuf<u8> T, U, sym_lo;
  DBuf<unsigned long long> sym_hi;
  DBuf<u32> sym_any_hi, dn, dpidx, dm, dfreq, dused, tcount;
  DBuf<u16> sym;
  DBuf<u64> triples;
  if (B) {
    T.alloc(c, (size_t)B << SEG_SHIFT); U.alloc(c, (size_t)B << SEG_SHIFT); sym_lo.alloc(c, (size_t)B << SEG_SHIFT);
    sym_hi.alloc(c, (size_t)B * SEL_STRIDE); sym_any_hi.alloc(c, B);
    CUDA_CHECK(cudaMemsetAsync(sym_hi, 0, (size_t)B * SEL_STRIDE * 8, c.stream));
    CUDA_CHECK(cudaMemsetAsync(sym_any_hi, 0, (size_t)B * 4, c.stream));
    sym.alloc(c, (size_t)B << SEG_SHIFT);
    dn.alloc(c, B); dpidx.alloc(c, B); dm.alloc(c, B); dfreq.alloc(c, (size_t)B * HUFF_MAXSYM); dused.alloc(c, (size_t)B * 8); tcount.alloc(c, B);
    triples.alloc(c, (size_t)B * tcap);
  }
  const NarrowSyms nsym{sym_lo, sym_hi, sym_any_hi};
  const size_t wcap = bwtc_window_bound((size_t)B * blockSize, B, fast);   // grows only if `help` holds more than its slack
  DBuf<u8> win[2];
  size_t cap[2] = {wcap, wcap};
  win[0].alloc(c, wcap);
  if (B) win[1].alloc(c, wcap);
  DBuf<BwtcState> st(c, 1);
  k_bwtc_start<<<1, 1, 0, c.stream>>>(st, win[0], wcap, finalByte, (u32)level);
  KLAUNCH(c); KCHECK();
  struct Ev {
    cudaEvent_t e = nullptr;
    cudaStream_t d2h;
    ~Ev() {   // no copy out of a window may outlive it, also when the call fails half way
      cudaStreamSynchronize(d2h);
      if (e) cudaEventDestroy(e);
    }
  } ev{nullptr, c.d2h_stream};
  CUDA_CHECK(cudaEventCreateWithFlags(&ev.e, cudaEventDisableTiming));
  // a result gets room for the whole stream at once (its input is complete: `end` is all of it)
  out.reserve(out.wr ? hlen : hlen + bwtc_bound(end));
  memcpy(out.next(), hdr, hlen);
  out.put(out.next(), hlen);
  BwtcState h;
  // the coder's state once the launch before `ev` has finished; its bytes (window w) start on their way to `out`
  auto fetch = [&](int w) -> size_t {
    CUDA_CHECK(cudaEventSynchronize(ev.e));
    CUDA_CHECK(cudaMemcpyAsync(&h, st, sizeof h, cudaMemcpyDeviceToHost, c.d2h_stream));
    CUDA_CHECK(cudaStreamSynchronize(c.d2h_stream));
    if (h.overflow) throw B2Error{B2_ERR_CUDA, "internal error: BWTC triple buffer overflow"};
    if (h.rc.n > h.rc.cap) throw B2Error{B2_ERR_CUDA, "internal error: BWTC output window overflow"};
    const size_t bytes = (size_t)h.rc.n;
    out.reserve(bytes, false, bwtc_bound((size_t)B * blockSize));   // a staging buffer of the usual size, more if needed
    CUDA_CHECK(cudaMemcpyAsync(out.next(), win[w], bytes, cudaMemcpyDeviceToHost, c.d2h_stream));
    return bytes;
  };
  std::vector<u32> hn(std::max(B, 1u));
  size_t pos = 0;       // raw bytes taken
  int w = 0;            // the window of the next batch
  bool held = false;    // the previous batch's bytes are still in window w ^ 1
  u64 help = 0;         // bytes the coder holds back when the next batch starts
  for (;;) {
    in.drop(pos);
    end = in.fill(pos + (size_t)B * blockSize);
    const size_t take = std::min(end, pos + (size_t)B * blockSize) - pos;   // < B blocks only at the end of the input
    if (!take) break;
    const u32 nb = (u32)((take + blockSize - 1) / blockSize);
    for (u32 b = 0; b < nb; b++) hn[b] = (u32)std::min<size_t>(blockSize, take - (size_t)b * blockSize);
    const u32 full = hn[nb - 1] == blockSize ? nb : nb - 1;   // only the last block of the input can be short
    if (full)
      CUDA_CHECK(cudaMemcpy2DAsync(T.p, SEG_SIZE, in.at(pos), blockSize, blockSize, full, cudaMemcpyHostToDevice, c.stream));
    if (full < nb)
      CUDA_CHECK(cudaMemcpyAsync(T.p + ((size_t)full << SEG_SHIFT), in.at(pos + (size_t)full * blockSize), hn[full], cudaMemcpyHostToDevice, c.stream));
    c.to_device(dn, hn.data(), 4 * nb);
    CUDA_CHECK(cudaMemsetAsync(dpidx, 0, 4 * nb, c.stream));
    {
      StageScope s(c, ST_BWT);
      bwt_forward_batch(c, T, U, dn, hn.data(), nb, dpidx, true, nullptr);   // U = sentinel BWT, dpidx = pidx + 1
    }
    {
      StageScope s(c, ST_MTF);
      mtf_rle2_batch(c, T, U, dn, hn.data(), nb, nsym, dm, dfreq, dused);
      u32 mmax = 0;   // m <= n + 1
      for (u32 b = 0; b < nb; b++) mmax = std::max(mmax, hn[b] + 1);
      const u32 tps = (mmax + WD_THREADS * 16 - 1) / (WD_THREADS * 16);
      k_bwtc_widen<<<nb * tps, WD_THREADS, 0, c.stream>>>(sym_lo, sym_hi, sym_any_hi, dm, tps, sym);
      KLAUNCH(c); KCHECK();
    }
    {
      StageScope s(c, ST_HUFF);   // statistics: the model takes the slot of the Huffman stage (ms_huff) ...
      if (fast) k_bwtc_model<<<nb, 32, 0, c.stream>>>(sym, dm, dn, dpidx, dused, blockSize, fast, triples, tcap, tcount);
      else k_bwtc_model_fenwick<<<nb, 32, 0, c.stream>>>(sym, dm, dn, dpidx, dused, blockSize, triples, tcap, tcount);
      KLAUNCH(c); KCHECK();
    }
    // the previous batch's coder has finished by now or soon: its bytes leave window w ^ 1, and its `help` sizes window w
    size_t prev = 0;
    if (held) {
      prev = fetch(w ^ 1);
      help = h.rc.help;
    }
    const size_t need = bwtc_window_bound(take, nb, fast) + (size_t)help + 16;   // the batch, the bytes held back, the trailer
    if (need > cap[w]) { win[w].alloc(c, need); cap[w] = need; }
    {
      StageScope s(c, ST_PACK);   // ... and the serial range coder the slot of the bit packer (ms_pack)
      k_bwtc_window<<<1, 1, 0, c.stream>>>(st, win[w], cap[w]);
      KLAUNCH(c); KCHECK();
      k_bwtc_code<<<1, 32, 0, c.stream>>>(st, triples, tcount, nb, tcap);
      KLAUNCH(c); KCHECK();
    }
    CUDA_CHECK(cudaEventRecord(ev.e, c.stream));
    if (held) out.put(out.next(), prev);   // while this batch runs
    held = true;
    w ^= 1;
    pos += take;
    c.stats.blocks += nb;
  }
  // the trailer goes behind the last batch's bytes (window w ^ 1), or into window 0 when there was no batch
  k_bwtc_finish<<<1, 1, 0, c.stream>>>(st);
  KLAUNCH(c); KCHECK();
  CUDA_CHECK(cudaEventRecord(ev.e, c.stream));
  const size_t last = fetch(held ? w ^ 1 : 0);
  out.put(out.next(), last);
  CUDA_CHECK(cudaStreamSynchronize(c.d2h_stream));   // a result is complete when the call returns
  c.stats.raw_bytes = pos;
  c.stats.comp_bytes = out.written;
}

// ---- decode ---------------------------------------------------------------------------------------------------
// The range decoder and the level are all that carries from one block to the next (the block models start afresh in
// bc_decode_block, the length model is stateless), so the decode stops after a batch of blocks and resumes from here.
// The coded stream reaches the device a window [a, a + wlen) at a time; rc.pos counts from the window of the last launch
// (st->a), and a launch over another window moves it.
#define BD_MORE 0      // more blocks may follow
#define BD_END 1       // "no more blocks" has been read
#define BD_NEED 2      // the next block reads past the window, which is not the end of the input: slide the window
#define BD_CORRUPT (-1)
#define BD_SIZE (-2)   // the blocks add up to more than the size field
#define BC_EOF 0xFFFFFFFFu
struct BwtcDecState {
  bc_dec rc;
  u64 a;            // absolute position of the window of the last launch
  u64 total;        // bytes in the blocks decoded so far
  u64 limit;        // the size field's size; ~0 when the stream has no size
  u32 level;
  u32 nblocks;      // blocks decoded so far
  u32 nb;           // blocks decoded by the last launch
  int status;       // BD_*
};

// the coder's first bytes: pos = the first byte behind the header, at the window's start
__global__ void k_bwtc_dec_start(BwtcDecState* st, const u8* __restrict__ win, u64 wlen, u64 a, u64 limit) {
  if (threadIdx.x || blockIdx.x) return;
  bc_dec_start(&st->rc, win, wlen, 0);                          // lib/BWTC.js:142-143
  st->level = bc_dec_cul(&st->rc, 256);                         // decoder.decodeByte(), :144
  bc_dec_update(&st->rc, 1, st->level, 256);
  st->a = a;
  st->total = 0; st->limit = limit;
  st->nblocks = 0; st->nb = 0;
  st->status = st->level >= 1 && st->level <= 9 ? BD_MORE : BD_CORRUPT;
}

// One thread: up to B more blocks down to their L columns (inverse MTF folded in), block b of the launch at slot b << 20.
// `final`: the input ends at the window's end, so a read past it is the reference's EOF.  Otherwise a step that reads past
// the window is undone (the decoder's state at the block's start is all that crosses a block) and the launch stops with
// BD_NEED.  maxblocks: the most blocks the stream may hold; when `need_at_max`, it is a lower bound taken from the input
// seen so far, and reaching it asks for more input instead of deciding.
__global__ void k_bwtc_decode(BwtcDecState* st, u32 B, const u8* __restrict__ win, u64 wlen, u64 a, int final, u64 maxblocks,
                              int need_at_max, u8* __restrict__ L, u32* __restrict__ lengths, u32* __restrict__ pidx1) {
  if (threadIdx.x || blockIdx.x) return;
  st->nb = 0;
  if (st->status != BD_MORE && st->status != BD_NEED) return;
  bc_dec rc = st->rc;
  rc.pos = st->a + rc.pos - a;   // a <= the next byte to read: the host never slides past it
  rc.in = win; rc.n = wlen;
  const u32 level = st->level;
  const bool unsized = st->limit == ~0ull;
  u64 total = st->total;
  bc_model model;
  u32 nb = 0;
  int status = BD_MORE;
  while (nb < B) {
    const bc_dec keep = rc;
    u32 len = 0, p1 = 0;
    int r;
    if (st->nblocks + nb >= maxblocks) {
      if (need_at_max) { status = BD_NEED; break; }
      r = bc_dec_cul(&rc, 3) == 2 ? 1 : -5;                     // only "no more blocks" may follow
    } else {
      r = bc_decode_block(&rc, &model, level * 100000u, level <= 5, L + ((size_t)nb << SEG_SHIFT), &len, &p1);
    }
    if (rc.buffer == BC_EOF) {   // the step has read past the window
      if (!final) { rc = keep; status = BD_NEED; break; }
      // Without a size, the end of the input is the only bound.  A whole stream is never read past its end (the
      // coder's trailer is longer than the decoder's look-ahead), so a decoder that has read past it is decoding a cut
      // stream: an error, where the reference has no check and decodes on.
      if (unsized) { status = BD_CORRUPT; break; }
    }
    if (r) { status = r == 1 ? BD_END : BD_CORRUPT; break; }
    if (total + len > st->limit) { status = BD_SIZE; break; }
    total += len;
    lengths[nb] = len; pidx1[nb] = p1;
    nb++;
  }
  st->rc = rc;
  st->a = a;
  st->total = total;
  st->nblocks += nb;
  st->nb = nb;
  st->status = status;
}

// blocks per decode batch ($B2_BWTC_DEC_BATCH: test hook, small batches exercise the batch seams on small inputs)
static u32 bwtc_dec_batch(const Ctx& c) {
  if (const char* e = getenv("B2_BWTC_DEC_BATCH")) { const int v = atoi(e); if (v >= 1) return (u32)v; }
  return c.bwt_batch;
}

// lib/Util.js:211-220 readUnsignedNumber after the magic.  Returns the size field (0 = unknown size, else size + 1) and
// sets *pos behind it: its last byte is the range coder's first.
static u64 bwtc_parse_header(const u8* in, size_t n, size_t* pos) {
  if (n < 5 || memcmp(in, "bwtc", 4)) throw B2Error{B2_ERR_BAD_MAGIC, "Bad magic"};   // lib/Util.js:151-153
  size_t p = 4;
  u64 fs = 0;
  for (;;) {
    // nine 7-bit groups hold any size below 2^63; a longer number cannot be the size of a real file and would overflow
    if (p >= n || p > 4 + 9) throw B2Error{B2_ERR_DATA_ERROR, "truncated or oversized BWTC header"};
    const u32 ch = in[p++];
    if (ch & 0x80) { fs += ch & 0x7F; break; }
    fs = (fs + ch) * 128;
  }
  if (fs != 0 && fs - 1 > ((u64)1 << 40)) throw B2Error{B2_ERR_DATA_ERROR, "Data error: implausible BWTC size field"};
  *pos = p;
  return fs;
}

// BWTC.decompressFile from a host source: b2_bwtc_decompress (the caller's buffer into the result) and
// b2_bwtc_decompress_stream (read and write callbacks).  The coded stream goes to the device a window of W bytes at a
// time (dec_window()); a launch that stops with BD_NEED slides the window to the first byte the next block needs, and a
// window that would start where the last one did is twice as long.  The decoded bytes go to `out` a batch at a time.
// Device memory: one window and one batch of blocks, whatever the size of the file (include/b2bz.h gives the bound).
void bwtc_decompress(Ctx& c, StreamIn& in, StreamOut& out) {
  size_t pos = 0;
  const u64 fs = bwtc_parse_header(in.at(0), in.fill(4 + 10), &pos);   // the longest header it accepts; before any device work
  const bool unsized = fs == 0;
  const u64 limit = unsized ? ~0ull : fs - 1;
  // The header is not trusted: the level is inside the coded stream, so the size field bounds the blocks for the
  // smallest block size, and a block costs at least a few coded bytes, so n compressed bytes cannot hold more than n / 2
  // blocks.  n is known once the input has ended; before, the bytes seen so far give a lower bound.
  const u64 size_blocks = unsized ? ~0ull : limit / 100000u + 2;
  size_t W = dec_window();
  size_t a = pos, wlen = 0;     // the window
  bool final = false;
  u64 maxblocks = 0;
  int need_at_max = 0;
  DBuf<u8> dwin;
  size_t dcap = 0;
  auto load = [&]() {
    in.drop(a);
    const size_t e = in.fill(a + W + 1);   // one byte more than the window: a window is the last one exactly when the input ends in it
    final = in.eof && e <= a + W;
    wlen = std::min(W, e - a);
    const u64 from_n = (u64)e / 2 + 2;
    maxblocks = std::min(size_blocks, from_n);
    need_at_max = !final && from_n < size_blocks;
    if (wlen > dcap) { dwin.alloc(c, wlen); dcap = wlen; }
    if (wlen) CUDA_CHECK(cudaMemcpyAsync(dwin.p, in.at(a), wlen, cudaMemcpyHostToDevice, c.stream));
  };
  load();
  const u32 B = (u32)std::min<u64>(bwtc_dec_batch(c), maxblocks);
  DBuf<u8> L(c, (size_t)B << SEG_SHIFT), dout(c, (size_t)B * 900000u);
  DBuf<u32> lengths(c, B), pidx1(c, B);
  DBuf<BwtcDecState> st(c, 1);
  k_bwtc_dec_start<<<1, 1, 0, c.stream>>>(st, dwin, wlen, a, limit);
  KLAUNCH(c); KCHECK();
  std::vector<u32> hl(B), hp(B);
  // a result with a known size gets all of its buffer now, up to what maxblocks blocks can hold (more would fail the size
  // check); a staging buffer holds one batch
  if (!unsized && !out.wr) out.reserve((size_t)std::min<u64>(limit, maxblocks * 900000u), true);
  for (;;) {
    {
      StageScope s(c, ST_HDEC);
      k_bwtc_decode<<<1, 1, 0, c.stream>>>(st, B, dwin, wlen, a, final, maxblocks, need_at_max, L, lengths, pidx1);
      KLAUNCH(c); KCHECK();
    }
    BwtcDecState h;
    c.to_host(&h, st, sizeof h);
    c.to_host(hl.data(), lengths, 4 * B);
    c.to_host(hp.data(), pidx1, 4 * B);
    c.sync();   // also ends the previous batch's copy to the host
    // the blocks decoded in full go out first, also in front of an error (lib/BWTC.js:228 writes each block as it ends)
    u64 bytes = 0;
    for (u32 b = 0; b < h.nb; b++) bytes += hl[b];
    if (h.nb) {
      out.reserve((size_t)bytes, false, (size_t)B * 900000u);   // a result grows only without a size field
      {
        StageScope s(c, ST_IBWT);   // BWT.unbwtransform of every block of the batch, lib/BWTC.js:224
        bwt_inverse_sentinel_batch(c, L, hl.data(), hp.data(), h.nb, dout);
      }
      CUDA_CHECK(cudaMemcpyAsync(out.next(), dout, bytes, cudaMemcpyDeviceToHost, c.stream));
      out.put(out.next(), (size_t)bytes);
      c.stats.blocks += h.nb;
    }
    if (h.status == BD_CORRUPT) throw B2Error{B2_ERR_DATA_ERROR, "Data error: BWTC stream is corrupt"};
    if (h.status == BD_SIZE) throw B2Error{B2_ERR_DATA_ERROR, "outputsize does not match decoded input"};   // lib/Util.js:69-71
    if (h.status == BD_END) break;
    if (h.status == BD_NEED) {
      const size_t next = (size_t)(h.a + h.rc.pos);   // the next block's first byte still to read
      if (next == a) W *= 2;                           // not one block fits: a longer window
      a = next;
      load();
    }
  }
  c.sync();
  if (!unsized && out.written != limit) throw B2Error{B2_ERR_DATA_ERROR, "outputsize does not match decoded input"};
}
