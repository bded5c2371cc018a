// api.cu -- the C ABI declared in include/b2bz.h.  Thin: argument checks, H2D/D2H staging,
// error translation.  All compute is in the CUDA stages (rle1.cu, bwt.cu, mtf.cu, huff.cu,
// decode.cu).  There is no CPU fallback anywhere: without a CUDA device every call fails.
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include "enc.h"

static std::mutex g_mu;
static Ctx* g_ctx = nullptr;
static thread_local std::string g_err;
// Set while a stream call runs one of its callbacks on this thread.  That thread holds g_mu, so a library call from the
// callback would wait for itself: it fails at once instead.
static thread_local bool t_in_callback = false;
static const char* const IN_CALLBACK = "called from inside a stream callback";
struct InCallback {
  std::string err;  // the call's own error state, which the callback's library calls may overwrite
  InCallback() : err(g_err) { t_in_callback = true; }
  ~InCallback() { t_in_callback = false; g_err = err; }
};
static std::map<void*, size_t> g_pinned_live;                  // pointers handed to the caller
static std::multimap<size_t, void*> g_pinned_free;             // cached pinned buffers by capacity

void Ctx::collect() {
  float acc[ST_COUNT];
  for (int i = 0; i < ST_COUNT; i++) acc[i] = 0.f;
  for (auto& t : ev_tags) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev_pool[t.second].a, ev_pool[t.second].b) == cudaSuccess) acc[t.first] += ms;
  }
  stats.ms_total = acc[ST_TOTAL]; stats.ms_h2d = acc[ST_H2D]; stats.ms_d2h = acc[ST_D2H];
  stats.ms_rle1 = acc[ST_RLE1]; stats.ms_bwt = acc[ST_BWT]; stats.ms_mtf = acc[ST_MTF];
  stats.ms_huff = acc[ST_HUFF]; stats.ms_pack = acc[ST_PACK]; stats.ms_scan = acc[ST_SCAN];
  stats.ms_hdec = acc[ST_HDEC]; stats.ms_unmtf = acc[ST_UNMTF]; stats.ms_ibwt = acc[ST_IBWT];
  stats.ms_unrle = acc[ST_UNRLE]; stats.ms_radix = acc[ST_RADIX];
  stats.ms_msd_scatter = acc[ST_MSD_SCATTER]; stats.ms_msd_bucket = acc[ST_MSD_BUCKET];
  // overlapped copies of the pipelined host path: span from the first to the last copy on their stream
  for (int w = 0; w < 2; w++) {
    float ms = 0.f;
    if (copy_used[w] && cudaEventElapsedTime(&ms, copy_ev[w][0], copy_ev[w][1]) == cudaSuccess) (w ? stats.ms_d2h : stats.ms_h2d) += ms;
  }
  uint64_t high = 0;
  if (pool && cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &high) == cudaSuccess) stats.dev_peak_bytes = high;
  else cudaGetLastError();
}

// ---- small control transfers through mapped pinned memory ----------------------------------
// During the pipelined host encode the copy engines are busy with 64 MiB uploads and per-batch downloads; an
// 8-byte cudaMemcpyAsync would wait behind them for milliseconds.  A tiny kernel moves control data through a
// mapped pinned staging area instead (SM loads/stores over PCIe, no copy engine).
__global__ void k_stage_copy(void* dst, const void* src, size_t bytes) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  if ((((size_t)dst | (size_t)src | bytes) & 3) == 0) {
    u32* d = (u32*)dst; const u32* s = (const u32*)src;
    for (size_t i = i0; i < bytes / 4; i += step) d[i] = s[i];
  } else {
    u8* d = (u8*)dst; const u8* s = (const u8*)src;
    for (size_t i = i0; i < bytes; i += step) d[i] = s[i];
  }
}
size_t Ctx::stage_take(size_t bytes) {
  if (!stage_h) {
    CUDA_CHECK(cudaHostAlloc((void**)&stage_h, stage_cap, cudaHostAllocMapped));
    CUDA_CHECK(cudaHostGetDevicePointer((void**)&stage_d, stage_h, 0));
  }
  const size_t need = (bytes + 15) & ~(size_t)15;
  if (stage_used + need > stage_cap) sync();
  const size_t off = stage_used;
  stage_used += need;
  return off;
}
void Ctx::to_device(void* ddst, const void* hsrc, size_t bytes) {
  if (!bytes) return;
  if (bytes > stage_cap / 2) { CUDA_CHECK(cudaMemcpyAsync(ddst, hsrc, bytes, cudaMemcpyHostToDevice, stream)); CUDA_CHECK(cudaStreamSynchronize(stream)); return; }
  const size_t off = stage_take(bytes);
  memcpy(stage_h + off, hsrc, bytes);
  k_stage_copy<<<(unsigned)std::min<size_t>((bytes / 4 + 255) / 256 + 1, 64), 256, 0, stream>>>(ddst, stage_d + off, bytes);
  CUDA_CHECK(cudaGetLastError());
}
void Ctx::to_host(void* hdst, const void* dsrc, size_t bytes) {
  if (!bytes) return;
  if (bytes > stage_cap / 2) { CUDA_CHECK(cudaMemcpyAsync(hdst, dsrc, bytes, cudaMemcpyDeviceToHost, stream)); return; }
  const size_t off = stage_take(bytes);
  k_stage_copy<<<(unsigned)std::min<size_t>((bytes / 4 + 255) / 256 + 1, 64), 256, 0, stream>>>(stage_d + off, dsrc, bytes);
  CUDA_CHECK(cudaGetLastError());
  fetches.push_back({hdst, off, bytes});
}
void Ctx::sync() {
  CUDA_CHECK(cudaStreamSynchronize(stream));
  for (auto& f : fetches) memcpy(f.dst, stage_h + f.off, f.bytes);
  fetches.clear();
  stage_used = 0;
}

static int pick_device() {
  const char* e = getenv("B2_DEVICE");
  if (e && *e) return atoi(e);
  e = getenv("LOCAL_RANK");
  if (e && *e) {
    int cnt = 0;
    if (cudaGetDeviceCount(&cnt) == cudaSuccess && cnt > 0) return atoi(e) % cnt;
  }
  return 0;
}

static Ctx& ctx_locked() {
  if (!g_ctx) {
    int dev = pick_device();
    int cnt = 0;
    cudaError_t e = cudaGetDeviceCount(&cnt);
    if (e != cudaSuccess || cnt == 0)
      throw B2Error{B2_ERR_CUDA, std::string("no CUDA device available (libb2bz has no CPU fallback): ") + cudaGetErrorString(e)};
    if (dev >= cnt) throw B2Error{B2_ERR_CUDA, "requested CUDA device does not exist"};
    CUDA_CHECK(cudaSetDevice(dev));
    Ctx* c = new Ctx();
    c->device = dev;
    memset(&c->stats, 0, sizeof c->stats);
    CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&c->h2d_stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&c->d2h_stream, cudaStreamNonBlocking));
    for (int w = 0; w < 2; w++) for (int k = 0; k < 2; k++) CUDA_CHECK(cudaEventCreate(&c->copy_ev[w][k]));
    cudaMemPool_t pool;
    CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, dev));
    uint64_t thr = UINT64_MAX;
    CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    c->pool = pool;
    int sms = 0;
    CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    c->bwt_batch = 2u * (u32)sms;
    const char* b = getenv("B2_BWT_BATCH");
    if (b && atoi(b) > 0) c->bwt_batch = (u32)atoi(b);
    const char* msd = getenv("B2_BWT_MSD");
    if (msd && *msd) c->bwt_msd = atoi(msd) != 0;
    const char* w8 = getenv("B2_BWT_PREFIX8");
    if (w8 && *w8) { c->bwt_wide_forced = true; c->bwt_wide = atoi(w8) != 0; }
    g_ctx = c;
  } else {
    CUDA_CHECK(cudaSetDevice(g_ctx->device));
  }
  return *g_ctx;
}

static void* pinned_alloc(size_t bytes) {
  if (bytes == 0) bytes = 1;
  auto it = g_pinned_free.lower_bound(bytes);
  if (it != g_pinned_free.end() && it->first <= bytes * 2 + 4096) {
    void* p = it->second; size_t cap = it->first;
    g_pinned_free.erase(it);
    g_pinned_live[p] = cap;
    return p;
  }
  void* p = nullptr;
  size_t cap = (bytes + 4095) & ~(size_t)4095;
  CUDA_CHECK(cudaHostAlloc(&p, cap, cudaHostAllocDefault));
  g_pinned_live[p] = cap;
  return p;
}

// give a live pinned buffer back to the cache (caller holds g_mu)
static void pinned_release(void* p) {
  auto it = g_pinned_live.find(p);
  if (it == g_pinned_live.end()) return;
  size_t cap = it->second;
  g_pinned_live.erase(it);
  size_t cached = 0;
  for (auto& kv : g_pinned_free) cached += kv.first;
  if (cached + cap > ((size_t)8 << 30)) cudaFreeHost(p);
  else g_pinned_free.insert({cap, p});
}

template <typename F>
static int guarded(F f) {
  if (t_in_callback) { g_err = IN_CALLBACK; return B2_ERR_BAD_ARG; }
  std::lock_guard<std::mutex> lk(g_mu);
  try {
    g_err.clear();
    return f();
  } catch (const B2Error& e) {
    g_err = e.msg;
    if (g_ctx && e.code == B2_ERR_CUDA) { cudaStreamSynchronize(g_ctx->stream); cudaGetLastError(); }
    return e.code;
  } catch (const std::exception& e) {
    g_err = e.what();
    return B2_ERR_CUDA;
  }
}

extern "C" {

int b2_init(int device) {
  return guarded([&]() {
    if (g_ctx && g_ctx->device != device) throw B2Error{B2_ERR_BAD_ARG, "b2_init: context already bound to another device"};
    if (!g_ctx) {
      char buf[16]; snprintf(buf, sizeof buf, "%d", device);
      setenv("B2_DEVICE", buf, 1);
    }
    ctx_locked();
    return 0;
  });
}

void b2_shutdown(void) {
  if (t_in_callback) { g_err = IN_CALLBACK; return; }
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_ctx) return;
  cudaSetDevice(g_ctx->device);
  // state kept across calls holds device buffers of this context: free it while the context is alive
  bzip2_release_plan();
  dec_shard_release();
  cudaStreamSynchronize(g_ctx->stream);
  for (auto& kv : g_pinned_free) cudaFreeHost(kv.second);
  g_pinned_free.clear();
  for (auto& e : g_ctx->ev_pool) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
  if (g_ctx->stage_h) cudaFreeHost(g_ctx->stage_h);
  cudaStreamDestroy(g_ctx->stream);
  cudaStreamDestroy(g_ctx->h2d_stream);
  cudaStreamDestroy(g_ctx->d2h_stream);
  for (int w = 0; w < 2; w++) for (int k = 0; k < 2; k++) cudaEventDestroy(g_ctx->copy_ev[w][k]);
  delete g_ctx;
  g_ctx = nullptr;
}

const char* b2_last_error(void) { return g_err.c_str(); }

void b2_free(void* p) {
  if (!p) return;
  if (t_in_callback) { g_err = IN_CALLBACK; return; }
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_pinned_live.find(p) == g_pinned_live.end()) { free(p); return; }
  pinned_release(p);
}

void b2_get_stats(b2_stats* s) {
  if (t_in_callback) { g_err = IN_CALLBACK; memset(s, 0, sizeof *s); return; }
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_ctx) *s = g_ctx->stats; else memset(s, 0, sizeof *s);
}

size_t b2_last_trace(b2_block_trace* out, size_t cap) {
  if (t_in_callback) { g_err = IN_CALLBACK; return 0; }
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_ctx) return 0;
  size_t n = g_ctx->trace.size();
  if (out) for (size_t i = 0; i < n && i < cap; i++) out[i] = g_ctx->trace[i];
  return n;
}

// ---- BWT ---------------------------------------------------------------------------------
int b2_bwt_cyclic_batch(const uint8_t* T, uint8_t* U, const uint64_t* offs, const int32_t* lens, int32_t* pidx, size_t nblocks) {
  return guarded([&]() {
    Ctx& c = ctx_locked();
    c.reset_call();
    for (size_t k = 0; k < nblocks; k++)
      if (lens[k] < 0 || lens[k] > 900000) throw B2Error{B2_ERR_BAD_ARG, "block length out of range (0..900000)"};
    {
      StageScope tot(c, ST_TOTAL);
      for (size_t k0 = 0; k0 < nblocks; k0 += c.bwt_batch) {
        const u32 nb = (u32)std::min<size_t>(c.bwt_batch, nblocks - k0);
        DBuf<u8> dT(c, (size_t)nb << SEG_SHIFT), dU(c, (size_t)nb << SEG_SHIFT);
        DBuf<u32> dn(c, nb), dp(c, nb);
        std::vector<u32> hn(nb);
        for (u32 b = 0; b < nb; b++) {
          hn[b] = (u32)lens[k0 + b];
          if (hn[b]) CUDA_CHECK(cudaMemcpyAsync(dT.p + ((size_t)b << SEG_SHIFT), T + offs[k0 + b], hn[b], cudaMemcpyHostToDevice, c.stream));
        }
        CUDA_CHECK(cudaMemcpyAsync(dn, hn.data(), nb * 4, cudaMemcpyHostToDevice, c.stream));
        CUDA_CHECK(cudaMemsetAsync(dp, 0, nb * 4, c.stream));
        {
          StageScope s(c, ST_BWT);
          bwt_forward_batch(c, dT, dU, dn, hn.data(), nb, dp);
        }
        std::vector<u32> hp(nb);
        CUDA_CHECK(cudaMemcpyAsync(hp.data(), dp, nb * 4, cudaMemcpyDeviceToHost, c.stream));
        for (u32 b = 0; b < nb; b++)
          if (hn[b]) CUDA_CHECK(cudaMemcpyAsync(U + offs[k0 + b], dU.p + ((size_t)b << SEG_SHIFT), hn[b], cudaMemcpyDeviceToHost, c.stream));
        c.sync();
        for (u32 b = 0; b < nb; b++) pidx[k0 + b] = (int32_t)hp[b];
        c.stats.blocks += nb;
      }
    }
    c.sync();
    c.collect();
    return 0;
  });
}

int32_t b2_bwt_cyclic(const uint8_t* T, uint8_t* U, int32_t n) {
  if (n <= 1) {  // lib/BWT.js:376-379
    if (n == 1) U[0] = T[0];
    return 0;
  }
  uint64_t off = 0;
  int32_t pidx = 0;
  int rc = b2_bwt_cyclic_batch(T, U, &off, &n, &pidx, 1);
  return rc < 0 ? rc : pidx;
}

// suffix array / sentinel BWT of one string (<= 2^20 - 2 bytes, the slot size of the block pipeline)
static int sentinel_sort(const uint8_t* T, int32_t n, int32_t* SA, uint8_t* U, int32_t* pidx1) {
  return guarded([&]() {
    if (n < 2 || (uint32_t)n > SEG_SIZE - 2) throw B2Error{B2_ERR_BAD_ARG, "length out of range (2..1048574)"};
    Ctx& c = ctx_locked();
    c.reset_call();
    {
      StageScope tot(c, ST_TOTAL);
      DBuf<u8> dT(c, SEG_SIZE), dU(c, SEG_SIZE);
      DBuf<u32> dn(c, 1), dp(c, 1), dsa(c, SEG_SIZE);
      u32 hn = (u32)n, hp = 0;
      CUDA_CHECK(cudaMemcpyAsync(dT.p, T, n, cudaMemcpyHostToDevice, c.stream));
      c.to_device(dn, &hn, 4);
      CUDA_CHECK(cudaMemsetAsync(dp, 0, 4, c.stream));
      bwt_forward_batch(c, dT, U ? dU.p : nullptr, dn, &hn, 1, dp, true, SA ? dsa.p : nullptr);
      c.to_host(&hp, dp, 4);
      if (SA) CUDA_CHECK(cudaMemcpyAsync(SA, dsa.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c.stream));
      if (U) CUDA_CHECK(cudaMemcpyAsync(U, dU.p, n, cudaMemcpyDeviceToHost, c.stream));
      c.sync();
      if (pidx1) *pidx1 = (int32_t)hp;
    }
    c.sync();
    c.collect();
    return 0;
  });
}
int b2_suffixsort(const uint8_t* T, int32_t* SA, int32_t n) {
  if (n <= 1) {  // lib/BWT.js:307-310
    if (n == 1) SA[0] = 0;
    return 0;
  }
  return sentinel_sort(T, n, SA, nullptr, nullptr);
}
int32_t b2_bwt_sentinel(const uint8_t* T, uint8_t* U, int32_t n) {
  if (n <= 1) {  // lib/BWT.js:332-335
    if (n == 1) U[0] = T[0];
    return n < 0 ? 0 : n;
  }
  int32_t p = 0;
  int rc = sentinel_sort(T, n, nullptr, U, &p);
  return rc < 0 ? rc : p;
}
int b2_bwt_inverse(const uint8_t* L, uint8_t* out, int32_t n, int32_t pidx) {
  if (n <= 0) return 0;
  if (n == 1) { out[0] = L[0]; return 0; }
  return guarded([&]() {
    if ((uint32_t)n > SEG_SIZE - 2) throw B2Error{B2_ERR_BAD_ARG, "length out of range (0..1048574)"};
    if (pidx < 0 || pidx > n) throw B2Error{B2_ERR_BAD_ARG, "primary index out of range"};
    Ctx& c = ctx_locked();
    c.reset_call();
    {
      StageScope tot(c, ST_TOTAL);
      DBuf<u8> dL(c, SEG_SIZE), dO(c, n);
      CUDA_CHECK(cudaMemcpyAsync(dL.p, L, n, cudaMemcpyHostToDevice, c.stream));
      const u32 hn = (u32)n, hp = (u32)pidx;
      bwt_inverse_sentinel_batch(c, dL, &hn, &hp, 1, dO);
      CUDA_CHECK(cudaMemcpyAsync(out, dO.p, n, cudaMemcpyDeviceToHost, c.stream));
    }
    c.sync();
    c.collect();
    return 0;
  });
}

}  // extern "C"

// ---- BWTC container (see bwtc.cu) ----------------------------------------------------------
// Every BWTC call is one of the two drivers of bwtc.cu between a source and a sink.
template <typename F>
static void bwtc_call(Ctx& c, F run) {
  try {
    StageScope tot(c, ST_TOTAL);
    run();
  } catch (...) {
    cudaStreamSynchronize(c.stream);  // nothing of this call may still be running when the next one starts
    throw;
  }
  c.sync();
  c.collect();
}
// file_size: the header's size field, n or (u64)-1 for a stream without a size (lib/Util.js:118-124)
static int bwtc_compress_buffer(const uint8_t* in, size_t n, int level, u64 file_size, uint8_t** out, size_t* out_n) {
  return guarded([&]() {
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn src(in, n);
    StreamOut dst(c.d2h_stream);
    bwtc_call(c, [&]() { bwtc_compress(c, src, level, file_size, dst); });
    *out_n = dst.written; *out = dst.take();
    return 0;
  });
}

extern "C" {

int b2_bwtc_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n) {
  return bwtc_compress_buffer(in, n, level, n, out, out_n);
}
int b2_bwtc_compress_unsized(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n) {
  return bwtc_compress_buffer(in, n, level, ~(u64)0, out, out_n);
}
int b2_bwtc_compress_stream(b2_read_fn rd, b2_write_fn wr, void* user, int level, int64_t size) {
  return guarded([&]() {
    if (!rd || !wr) throw B2Error{B2_ERR_BAD_ARG, "null callback"};
    if (size < -1) throw B2Error{B2_ERR_BAD_ARG, "size must be >= 0, or -1 for a stream without a size"};
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn src(rd, user, c.h2d_stream);   // the uploads are from pageable memory: nothing is ever queued out of its buffer
    StreamOut dst(wr, user, c.d2h_stream);
    bwtc_call(c, [&]() { bwtc_compress(c, src, level, size < 0 ? ~(u64)0 : (u64)size, dst); });
    return 0;
  });
}
int b2_bwtc_decompress(const uint8_t* in, size_t n, uint8_t** out, size_t* out_n) {
  return guarded([&]() {
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn src(in, n);
    StreamOut dst(c.stream);
    bwtc_call(c, [&]() { bwtc_decompress(c, src, dst); });   // on an error the result is dropped with dst
    c.stats.raw_bytes = dst.written; c.stats.comp_bytes = n;
    *out_n = dst.written; *out = dst.take();
    return 0;
  });
}
int b2_bwtc_decompress_stream(b2_read_fn rd, b2_write_fn wr, void* user) {
  return guarded([&]() {
    if (!rd || !wr) throw B2Error{B2_ERR_BAD_ARG, "null callback"};
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn src(rd, user, c.stream);
    StreamOut dst(wr, user, c.stream);
    bwtc_call(c, [&]() { bwtc_decompress(c, src, dst); });
    c.stats.raw_bytes = dst.written; c.stats.comp_bytes = src.base + src.have;
    return 0;
  });
}

uint32_t b2_crc32_bzip2(const uint8_t* p, size_t n) {
  if (t_in_callback) { g_err = IN_CALLBACK; return (uint32_t)B2_ERR_BAD_ARG; }
  uint32_t crc = 0;
  int rc = guarded([&]() {
    Ctx& c = ctx_locked();
    c.reset_call();
    DBuf<u8> d(c, n ? n : 1);
    if (n) CUDA_CHECK(cudaMemcpyAsync(d, p, n, cudaMemcpyHostToDevice, c.stream));
    crc = crc32_device(c, d, n);
    return 0;
  });
  (void)rc;
  return crc;
}

// ---- bzip2 -------------------------------------------------------------------------------
size_t b2_bzip2_bound(size_t n) {
  // worst case per block: Huffman codes up to 20 bits for <= n+1 symbols would be 2.5x, but the
  // flat 2nd table bounds every 50-group at 50*ceil(log2(258)) = 450 bits = 9 bits/symbol;
  // RLE1 can expand the block stream by 5/4.  Use a comfortable 1.5x + per-block headers.
  size_t blocks = n / 99981 + 2;
  return n + n / 2 + blocks * 4096 + 64;
}

}  // extern "C"

// Inputs above the streaming window pass through the device in windows (bounded device memory: files larger than HBM);
// $B2_STREAM_WINDOW sets the window in bytes (default 8 GiB, at least 64 MiB -- a test hook allows less).
static size_t stream_window() {
  size_t win = (size_t)8 << 30;
  if (const char* e = getenv("B2_STREAM_WINDOW")) { const long long v = atoll(e); if (v >= (1 << 20)) win = (size_t)v; }
  return win;
}
size_t dec_window() {
  if (const char* e = getenv("B2_DEC_WINDOW")) { const long long v = atoll(e); if (v >= (64 << 10)) return (size_t)v; }
  return (size_t)4 << 30;
}

// ---- the host-side input and output of the host entry points ----
StreamIn::~StreamIn() {
  if (rd && buf) { cudaStreamSynchronize(busy); free(buf); }
}
size_t StreamIn::fill(size_t end) {
  while (base + have < end && !eof) {
    if (have == cap) {
      // double (from 64 KiB), but never past what is asked for: memory follows the data that has arrived.  Pageable:
      // pinning every size a growing buffer passes through costs more than the driver's staged copies out of it
      const size_t ncap = std::max<size_t>((size_t)64 << 10, std::min(2 * cap, end - base));
      CUDA_CHECK(cudaStreamSynchronize(busy));
      u8* nb = (u8*)realloc(buf, ncap);
      if (!nb) throw B2Error{B2_ERR_CUDA, "out of host memory"};
      buf = nb; cap = ncap;
    }
    int64_t got;
    {
      InCallback in;
      got = rd(user, buf + have, cap - have);
    }
    if (got < 0) throw B2Error{B2_ERR_STREAM, "the read callback aborted the stream"};
    if ((uint64_t)got > cap - have) throw B2Error{B2_ERR_BAD_ARG, "the read callback returned more bytes than it was asked for"};
    if (got == 0) eof = true;
    have += (size_t)got;
  }
  return base + have;
}
void StreamIn::drop(size_t pos) {
  const size_t k = std::min(pos > base ? pos - base : 0, have);
  if (!k) return;
  base += k; have -= k;
  if (!rd) { buf += k; cap -= k; return; }  // the caller's buffer: its bytes stay where they are
  CUDA_CHECK(cudaStreamSynchronize(busy));
  memmove(buf, buf + k, have);
}
// the buffers come from (and go back to) the pinned buffers b2_free recycles: a second call reuses them
StreamOut::~StreamOut() {
  if (buf) { cudaStreamSynchronize(busy); pinned_release(buf); }
}
void StreamOut::reserve(size_t bytes, bool last, size_t limit) {
  const size_t kept = wr ? 0 : (size_t)written;
  if (kept + bytes <= cap) return;
  const size_t ncap = last ? kept + bytes : std::max(kept + bytes, std::min(2 * cap, wr ? limit : SIZE_MAX));
  u8* nb = (u8*)pinned_alloc(ncap);
  if (kept) { CUDA_CHECK(cudaStreamSynchronize(busy)); memcpy(nb, buf, kept); }
  if (buf) pinned_release(buf);
  buf = nb; cap = ncap;
}
void StreamOut::put(const u8* p, size_t n) {
  if (!n) return;
  if (wr) {
    CUDA_CHECK(cudaStreamSynchronize(busy));
    int r;
    {
      InCallback in;
      r = wr(user, p, n);
    }
    if (r != 0) throw B2Error{B2_ERR_STREAM, "the write callback aborted the stream"};
  }
  written += n;
}
u8* StreamOut::take() {
  u8* p = buf ? buf : (u8*)pinned_alloc(0);
  buf = nullptr; cap = 0;
  return p;
}

// b2_bzip2_compress and b2_bzip2_compress_stream.  The first window sizes the buffers: an input that ends inside it is
// one window of exactly its size.
static int compress_host(Ctx& c, StreamIn& in, StreamOut& out, int level, bool pinned_in) {
  size_t produced = 0;
  try {
    StageScope tot(c, ST_TOTAL);
    size_t win = stream_window();
    const size_t first = in.fill(win + 1);
    const bool whole = in.eof && first <= win;
    if (whole) win = first;
    const size_t dcap = whole ? b2_bzip2_bound(first) : b2_bzip2_bound(win) + 64;
    // a staging sink holds one window's output, a result the whole stream (its input is complete: `first` is all of it)
    out.reserve(out.wr ? dcap : b2_bzip2_bound(first), true);
    DBuf<u8> din(c, win ? win : 1), dout(c, dcap);
    c.sync();  // the buffers are used from the copy streams as well
    bzip2_compress_host(c, in, level, din, win, dout, dcap, out, &produced, pinned_in);
  } catch (...) {
    cudaStreamSynchronize(c.stream);  // nothing of this call may still be running when the next one starts
    throw;
  }
  c.sync();
  c.collect();
  c.stats.raw_bytes = in.base + in.have; c.stats.comp_bytes = produced;
  return 0;
}

// Every decode from a host input: b2_bzip2_decompress_partial and the calls built on it, and b2_bzip2_decompress_stream.
// run(&produced) is one of the host-input drivers of decode.cu.  On a decode error (-2/-5/-7) the code is returned, not
// thrown, and the output / the rows hold what the reference has written by the time it throws; any other error throws.
template <class Run>
static int decode_host(Ctx& c, StreamIn& in, Run run) {
  size_t produced = 0;
  int rc = 0;
  try {
    StageScope tot(c, ST_TOTAL);
    try {
      run(&produced);
    } catch (const B2Error& e) {
      if (e.code != B2_ERR_NOT_BZIP_DATA && e.code != B2_ERR_UNEXPECTED_INPUT_EOF && e.code != B2_ERR_DATA_ERROR &&
          e.code != B2_ERR_OBSOLETE_INPUT)
        throw;
      g_err = e.msg;
      rc = e.code;
    }
    c.sync();
  } catch (...) {
    cudaStreamSynchronize(c.stream);
    throw;
  }
  c.sync();
  c.collect();
  c.stats.raw_bytes = produced; c.stats.comp_bytes = in.base + in.have;
  return rc;
}

// The host-buffer decodes: decode_host over the caller's buffer, run(c, src, dst, &produced), with the result dst in *out
// when out is given.  The input stays on the host; the decoder uploads it a window at a time.
template <class Run>
static int decode_common(const uint8_t* in, size_t n, Run run, uint8_t** out, size_t* out_n) {
  Ctx& c = ctx_locked();
  c.reset_call();
  StreamIn src(in, n);
  StreamOut dst(c.stream);
  const int rc = decode_host(c, src, [&](size_t* produced) { run(c, src, dst, produced); });
  if (out) { *out_n = dst.written; *out = dst.take(); }
  return rc;
}

// b2_bzip2_recover and b2_bzip2_recover_stream: the recovery from `in` to `out`, its rows in *rows / *count
static int recover_host(Ctx& c, StreamIn& in, StreamOut& out, int mode, b2_recovered_block** rows, size_t* count) {
  std::vector<b2_recovered_block> r;
  try {
    StageScope tot(c, ST_TOTAL);
    bzip2_recover(c, in, mode == B2_RECOVER_BZ2, out, r);
  } catch (...) {
    cudaStreamSynchronize(c.stream);
    throw;
  }
  c.sync();
  c.collect();
  c.stats.raw_bytes = out.written; c.stats.comp_bytes = in.base + in.have;
  b2_recovered_block* p = (b2_recovered_block*)malloc(sizeof(b2_recovered_block) * (r.size() + 1));
  if (!p) throw B2Error{B2_ERR_CUDA, "out of host memory"};
  if (!r.empty()) memcpy(p, r.data(), sizeof(b2_recovered_block) * r.size());
  *rows = p; *count = r.size();
  return 0;
}
static void check_recover(int mode, b2_recovered_block** rows, size_t* count) {
  if (mode != B2_RECOVER_BYTES && mode != B2_RECOVER_BZ2) throw B2Error{B2_ERR_BAD_ARG, "unknown recovery mode"};
  if (!rows || !count) throw B2Error{B2_ERR_BAD_ARG, "null output argument"};
}

extern "C" {

int b2_bzip2_recover(const uint8_t* in, size_t n, int mode, uint8_t** out, size_t* out_n, b2_recovered_block** rows, size_t* count) {
  return guarded([&]() {
    check_recover(mode, rows, count);
    if (!out || !out_n || (n && !in)) throw B2Error{B2_ERR_BAD_ARG, "null output argument or input"};
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn src(in, n);
    StreamOut dst(c.stream);
    recover_host(c, src, dst, mode, rows, count);
    *out_n = dst.written; *out = dst.take();
    return 0;
  });
}

int b2_bzip2_recover_stream(b2_read_fn rd, b2_write_fn wr, void* user, int mode, b2_recovered_block** rows, size_t* count) {
  return guarded([&]() {
    if (!rd || !wr) throw B2Error{B2_ERR_BAD_ARG, "null callback"};
    check_recover(mode, rows, count);
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn src(rd, user, c.stream);
    StreamOut dst(wr, user, c.stream);
    return recover_host(c, src, dst, mode, rows, count);
  });
}

// the encoder flavor of a compress call: checked with the other arguments, before anything is read
static void check_flavor(int flavor) {
  if (flavor != B2_BZ2_COMPRESSJS && flavor != B2_BZ2_LIBBZ2) throw B2Error{B2_ERR_BAD_ARG, "unknown bzip2 flavor"};
}

int b2_bzip2_compress_stream(b2_read_fn rd, b2_write_fn wr, void* user, int level) {
  return b2_bzip2_compress_stream_flavor(rd, wr, user, level, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_compress_stream_flavor(b2_read_fn rd, b2_write_fn wr, void* user, int level, int flavor) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    if (!rd || !wr) throw B2Error{B2_ERR_BAD_ARG, "null callback"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = flavor;
    StreamIn in(rd, user, c.h2d_stream);
    StreamOut out(wr, user, c.d2h_stream);
    return compress_host(c, in, out, level, false);
  });
}

int b2_bzip2_decompress_stream(b2_read_fn rd, b2_write_fn wr, void* user, int multistream) {
  return b2_bzip2_decompress_stream_flavor(rd, wr, user, multistream, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_decompress_stream_flavor(b2_read_fn rd, b2_write_fn wr, void* user, int multistream, int flavor) {
  return guarded([&]() {
    if (!rd || !wr) throw B2Error{B2_ERR_BAD_ARG, "null callback"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    StreamIn in(rd, user, c.stream);
    StreamOut out(wr, user, c.stream);
    return decode_host(c, in, [&](size_t* produced) { bzip2_decompress_host(c, in, multistream, flavor, out, produced); });
  });
}

int b2_bzip2_compress_dev(const void* d_in, size_t n, int level, void* d_out, size_t out_cap, size_t* out_n) {
  return b2_bzip2_compress_dev_flavor(d_in, n, level, d_out, out_cap, out_n, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_compress_dev_flavor(const void* d_in, size_t n, int level, void* d_out, size_t out_cap, size_t* out_n, int flavor) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = flavor;
    {
      StageScope tot(c, ST_TOTAL);
      bzip2_compress_dev(c, (const u8*)d_in, n, level, (u8*)d_out, out_cap, out_n);
    }
    c.sync();
    c.collect();
    c.stats.raw_bytes = n; c.stats.comp_bytes = *out_n;
    return 0;
  });
}

int b2_bzip2_compress(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n) {
  return b2_bzip2_compress_flavor(in, n, level, out, out_n, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_compress_flavor(const uint8_t* in, size_t n, int level, uint8_t** out, size_t* out_n, int flavor) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = flavor;
    cudaPointerAttributes pa;
    const bool pinned_in = n && cudaPointerGetAttributes(&pa, in) == cudaSuccess && pa.type == cudaMemoryTypeHost;
    cudaGetLastError();
    StreamIn src(in, n);
    StreamOut dst(c.d2h_stream);
    compress_host(c, src, dst, level, pinned_in);
    *out_n = dst.written; *out = dst.take();
    return 0;
  });
}

int b2_bzip2_plan(const void* d_in, size_t n, int level, size_t* total_blocks) {
  return b2_bzip2_plan_flavor(d_in, n, level, total_blocks, B2_BZ2_COMPRESSJS);
}

int b2_dec_shard_open(const void* d_in, size_t n, int rank, int world, uint64_t* info) {
  return b2_dec_shard_open_flavor(d_in, n, rank, world, info, B2_BZ2_COMPRESSJS);
}
int b2_dec_shard_open_flavor(const void* d_in, size_t n, int rank, int world, uint64_t* info, int flavor) {
  return guarded([&]() {
    check_flavor(flavor);
    if (world < 1 || rank < 0 || rank >= world) throw B2Error{B2_ERR_BAD_ARG, "bad rank/world"};
    Ctx& c = ctx_locked();
    c.reset_call();
    {
      StageScope tot(c, ST_TOTAL);
      dec_shard_open(c, (const u8*)d_in, n, rank, world, flavor, info);
    }
    c.sync();
    c.collect();
    return 0;
  });
}
int b2_dec_shard_export(uint64_t* buf) {
  return guarded([&]() { dec_shard_export(buf); return 0; });
}
int b2_dec_shard_finish(const uint64_t* all, int multistream, void* d_out, size_t out_cap, uint64_t* res) {
  return guarded([&]() {
    ctx_locked();
    dec_shard_finish(all, multistream, (u8*)d_out, out_cap, res);
    return 0;
  });
}

int b2_dec_share_open(const void* d_buf, size_t hold, uint64_t g0, size_t share_len, size_t total, uint64_t* info) {
  return b2_dec_share_open_flavor(d_buf, hold, g0, share_len, total, info, B2_BZ2_COMPRESSJS);
}
int b2_dec_share_open_flavor(const void* d_buf, size_t hold, uint64_t g0, size_t share_len, size_t total, uint64_t* info, int flavor) {
  return guarded([&]() {
    check_flavor(flavor);
    if (share_len > hold || g0 > total || hold > total - g0) throw B2Error{B2_ERR_BAD_ARG, "the buffer is not a share of the stream"};
    if (g0 + hold < total && hold - share_len < B2_SHARE_HALO_MIN) throw B2Error{B2_ERR_BAD_ARG, "halo shorter than 14 bytes"};
    Ctx& c = ctx_locked();
    c.reset_call();
    {
      StageScope tot(c, ST_TOTAL);
      dec_share_open(c, (const u8*)d_buf, hold, g0, share_len, total, flavor, info);
    }
    c.sync();
    c.collect();
    return 0;
  });
}
int b2_dec_share_export(uint64_t* buf) {
  return guarded([&]() { dec_share_export(buf); return 0; });
}
int b2_dec_share_finish(const uint64_t* all, size_t count, int multistream, void* d_out, size_t out_cap, uint64_t* res) {
  return guarded([&]() {
    ctx_locked();
    dec_share_finish(all, count, multistream, (u8*)d_out, out_cap, res);
    return 0;
  });
}

int b2_bitshift_dev(const void* d_src, uint64_t nbits, int phase, void* d_dst) {
  return guarded([&]() {
    if (phase < 0 || phase > 7 || (((size_t)d_src | (size_t)d_dst) & 3)) throw B2Error{B2_ERR_BAD_ARG, "bad phase or unaligned buffers"};
    Ctx& c = ctx_locked();
    bitshift_device(c, d_src, nbits, phase, d_dst);
    return 0;
  });
}

int b2_bzip2_plan_spec(const void* d_in, size_t n, int level, int rank, int world, uint64_t* info) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    if (world < 1 || rank < 0 || rank >= world) throw B2Error{B2_ERR_BAD_ARG, "bad rank/world"};
    Ctx& c = ctx_locked();
    c.reset_call();
    bzip2_plan_spec(c, (const u8*)d_in, n, level, rank, world, info);
    c.sync();
    return 0;
  });
}

int b2_bzip2_share_summary(const void* d_share, size_t n, uint64_t* summary) {
  return guarded([&]() {
    Ctx& c = ctx_locked();
    c.reset_call();
    bzip2_share_summary(c, (const u8*)d_share, n, summary);
    c.sync();
    return 0;
  });
}

int b2_bzip2_plan_share(const void* d_buf, size_t n, int level, uint64_t state_in, uint64_t w_in, size_t first, size_t count, uint64_t* info) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    Ctx& c = ctx_locked();
    c.reset_call();
    bzip2_plan_share(c, (const u8*)d_buf, n, level, state_in, w_in, first, count, info);
    c.sync();
    return 0;
  });
}

int b2_bzip2_plan_flavor(const void* d_in, size_t n, int level, size_t* total_blocks, int flavor) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = flavor;
    const size_t nb = bzip2_plan(c, (const u8*)d_in, n, level);
    if (total_blocks) *total_blocks = nb;
    c.sync();
    return 0;
  });
}

int b2_bzip2_share_cut_table(const void* d_buf, size_t n, int level, uint64_t state_in, uint64_t w_in, size_t share_len, uint64_t dmax,
                             uint32_t* table) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    if (share_len > n || !table || dmax >= ((u64)1 << 31)) throw B2Error{B2_ERR_BAD_ARG, "bad share length, drift bound or table"};
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = B2_BZ2_LIBBZ2;
    bzip2_share_cut_table(c, (const u8*)d_buf, n, level, state_in, w_in, share_len, dmax, table);
    c.sync();
    return 0;
  });
}

int b2_bzip2_plan_share_flavor(const void* d_buf, size_t n, int level, uint64_t state_in, uint64_t w_in, size_t first, size_t count,
                               uint64_t drift, int flavor, uint64_t* info) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = flavor;
    bzip2_plan_share_flavor(c, (const u8*)d_buf, n, level, state_in, w_in, first, count, drift, info);
    c.sync();
    return 0;
  });
}

int b2_bzip2_encode_range_dev(const void* d_in, size_t n, int level, size_t first, size_t count, int bit_phase, void* d_out,
                              size_t out_cap, uint64_t* out_bits, uint32_t* block_crcs) {
  return b2_bzip2_encode_range_dev_flavor(d_in, n, level, first, count, bit_phase, d_out, out_cap, out_bits, block_crcs, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_encode_range_dev_flavor(const void* d_in, size_t n, int level, size_t first, size_t count, int bit_phase, void* d_out,
                                     size_t out_cap, uint64_t* out_bits, uint32_t* block_crcs, int flavor) {
  return guarded([&]() {
    if (level < 1 || level > 9) throw B2Error{B2_ERR_BAD_LEVEL, "Invalid block size multiplier"};
    if (bit_phase < 0 || bit_phase > 7) throw B2Error{B2_ERR_BAD_ARG, "bit_phase must be 0..7"};
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    c.bz_flavor = flavor;
    {
      StageScope tot(c, ST_TOTAL);
      bzip2_encode_range(c, (const u8*)d_in, n, level, first, count, bit_phase, (u8*)d_out, out_cap, out_bits, block_crcs);
    }
    c.sync();
    c.collect();
    return 0;
  });
}

int b2_bzip2_decompress_partial(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n) {
  return b2_bzip2_decompress_partial_flavor(in, n, multistream, out, out_n, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_decompress_partial_flavor(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n, int flavor) {
  return guarded([&]() {
    check_flavor(flavor);
    return decode_common(in, n, [&](Ctx& c, StreamIn& s, StreamOut& d, size_t* p) { bzip2_decompress_host(c, s, multistream, flavor, d, p); },
                         out, out_n);
  });
}

int b2_bzip2_decompress_blocks(const uint8_t* in, size_t n, const uint64_t* bitpos, size_t count, uint8_t** out, size_t* out_n,
                               uint64_t** ends, size_t* done) {
  return guarded([&]() {
    if (count && !bitpos) throw B2Error{B2_ERR_BAD_ARG, "bitpos is null"};
    if (!out || !out_n || !ends || !done) throw B2Error{B2_ERR_BAD_ARG, "null output argument"};
    struct HostBuf { void* p; ~HostBuf() { free(p); } } ep{malloc(sizeof(uint64_t) * (count + 1))};
    if (!ep.p) throw B2Error{B2_ERR_CUDA, "out of host memory"};
    const std::vector<u64> pos(bitpos, bitpos + count);
    DecRows rows;
    int rc = 0;
    uint8_t* o = nullptr; size_t on = 0;
    if (count) rc = decode_common(in, n, [&](Ctx& c, StreamIn& s, StreamOut& d, size_t* p) { bzip2_decompress_list(c, s, pos, d, rows, p); }, &o, &on);
    else if (!(o = (uint8_t*)malloc(1))) throw B2Error{B2_ERR_CUDA, "out of host memory"};  // no position: nothing is read, not even the header
    for (size_t i = 0; i < rows.ends.size(); i++) ((uint64_t*)ep.p)[i] = rows.ends[i];
    *out = o; *out_n = on; *ends = (uint64_t*)ep.p; *done = rows.ends.size();
    ep.p = nullptr;
    return rc;
  });
}

// one-element position lists
int b2_bzip2_decompress_block_partial(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n) {
  uint64_t* ends = nullptr; size_t done = 0;
  const int rc = b2_bzip2_decompress_blocks(in, n, &bitpos, 1, out, out_n, &ends, &done);
  b2_free(ends);
  return rc;
}

int b2_bzip2_table_partial(const uint8_t* in, size_t n, int multistream, uint64_t** bitpos, uint32_t** sizes, size_t* count) {
  return guarded([&]() {
    DecRows rows;
    const int rc = decode_common(in, n, [&](Ctx& c, StreamIn& s, StreamOut&, size_t* p) { bzip2_table(c, s, multistream, rows, p); }, nullptr, nullptr);
    *count = rows.pos.size();
    *bitpos = (uint64_t*)malloc(sizeof(uint64_t) * (rows.pos.size() + 1));
    *sizes = (uint32_t*)malloc(sizeof(uint32_t) * (rows.pos.size() + 1));
    for (size_t i = 0; i < rows.pos.size(); i++) { (*bitpos)[i] = rows.pos[i]; (*sizes)[i] = rows.len[i]; }
    return rc;
  });
}

// The all-or-nothing entry points: the partial call, with what it returned on an error released here.
static int drop_on_error(int rc, uint8_t* p, size_t pn, uint8_t** out, size_t* out_n) {
  if (rc || !out) { b2_free(p); return rc; }
  *out = p; *out_n = pn;
  return 0;
}

int b2_bzip2_decompress(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n) {
  return b2_bzip2_decompress_flavor(in, n, multistream, out, out_n, B2_BZ2_COMPRESSJS);
}

int b2_bzip2_decompress_flavor(const uint8_t* in, size_t n, int multistream, uint8_t** out, size_t* out_n, int flavor) {
  uint8_t* p = nullptr; size_t pn = 0;
  const int rc = b2_bzip2_decompress_partial_flavor(in, n, multistream, &p, &pn, flavor);
  return drop_on_error(rc, p, pn, out, out_n);
}

int b2_bzip2_decompress_block(const uint8_t* in, size_t n, uint64_t bitpos, uint8_t** out, size_t* out_n) {
  uint8_t* p = nullptr; size_t pn = 0;
  const int rc = b2_bzip2_decompress_block_partial(in, n, bitpos, &p, &pn);
  return drop_on_error(rc, p, pn, out, out_n);
}

int b2_bzip2_table(const uint8_t* in, size_t n, int multistream, uint64_t** bitpos, uint32_t** sizes, size_t* count) {
  uint64_t* bp = nullptr; uint32_t* sz = nullptr; size_t cnt = 0;
  const int rc = b2_bzip2_table_partial(in, n, multistream, &bp, &sz, &cnt);
  if (rc) { b2_free(bp); b2_free(sz); return rc; }
  *bitpos = bp; *sizes = sz; *count = cnt;
  return 0;
}

int b2_bzip2_decompress_dev(const void* d_in, size_t n, int multistream, void* d_out, size_t out_cap, size_t* out_n) {
  return b2_bzip2_decompress_dev_flavor(d_in, n, multistream, d_out, out_cap, out_n, B2_BZ2_COMPRESSJS);
}
int b2_bzip2_decompress_dev_flavor(const void* d_in, size_t n, int multistream, void* d_out, size_t out_cap, size_t* out_n, int flavor) {
  return guarded([&]() {
    check_flavor(flavor);
    Ctx& c = ctx_locked();
    c.reset_call();
    {
      StageScope tot(c, ST_TOTAL);
      if (d_out) bzip2_decompress_dev(c, (const u8*)d_in, n, multistream, flavor, (u8*)d_out, out_cap, out_n);
      else bzip2_decompress_size(c, (const u8*)d_in, n, multistream, flavor, out_n);
    }
    c.sync();
    c.collect();
    c.stats.raw_bytes = *out_n; c.stats.comp_bytes = n;
    return 0;
  });
}

}  // extern "C"
