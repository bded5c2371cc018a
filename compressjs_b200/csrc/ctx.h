// ctx.h -- per-process library context: device, stream, stream-ordered allocations, timers.
#pragma once
#include <vector>
#include <utility>
#include <mutex>
#include "common.cuh"
#include "../../include/b2bz.h"

struct EventPair {
  cudaEvent_t a, b;
};

struct Ctx {
  int device = -1;
  cudaStream_t stream = nullptr;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;  // host-buffer entry points: copies overlapped with the encode
  cudaEvent_t copy_ev[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};
  bool copy_used[2] = {false, false};
  b2_stats stats;
  std::vector<EventPair> ev_pool;   // reusable events
  size_t ev_used = 0;
  std::vector<std::pair<int, size_t>> ev_tags;  // (stage id, pool index) recorded in the current call
  std::vector<b2_block_trace> trace;
  u32 bwt_batch = 264;  // bzip2 blocks processed together in one batch: 2 CTAs per SM for the per-block kernels (set from the SM count)
  int bz_flavor = B2_BZ2_COMPRESSJS;  // bzip2 encoder flavor of the current call (block cut and Huffman table search)
  bool timing = true;
  bool bwt_msd = true;  // MSD + shared-memory bucket sort for sparse-tie batches (bwt_msd.cu); B2_BWT_MSD=0 disables it
  bool bwt_wide = false, bwt_wide_forced = false, bwt_mode_known = false;  // 8-byte initial sort for text-like batches (see bwt.cu)

  void* dalloc(size_t bytes) {
    void* p = nullptr;
    if (bytes == 0) bytes = 16;
    CUDA_CHECK(cudaMallocAsync(&p, bytes, stream));
    return p;
  }
  void dfree(void* p) {
    if (p) cudaFreeAsync(p, stream);
  }
  // Make the stream-ordered pool hold at least `bytes` of physical memory (one big allocation, freed at once; the
  // pool's release threshold keeps it).  Batches of different sizes then never have to grow the pool mid-call.
  size_t warmed = 0;
  void prewarm(size_t bytes) {
    if (bytes <= warmed) return;
    void* p = nullptr;
    if (cudaMallocAsync(&p, bytes, stream) == cudaSuccess) { cudaFreeAsync(p, stream); warmed = bytes; }
    else cudaGetLastError();  // not fatal: the stages allocate what they need anyway
  }
  template <typename T>
  T* dalloc_t(size_t count) { return (T*)dalloc(count * sizeof(T)); }

  // stage timing with CUDA events on the library stream
  size_t begin(int stage) {
    if (!timing) return 0;
    if (ev_used >= ev_pool.size()) {
      EventPair e;
      CUDA_CHECK(cudaEventCreate(&e.a));
      CUDA_CHECK(cudaEventCreate(&e.b));
      ev_pool.push_back(e);
    }
    size_t i = ev_used++;
    ev_tags.push_back({stage, i});
    CUDA_CHECK(cudaEventRecord(ev_pool[i].a, stream));
    return i;
  }
  void end(size_t i) {
    if (!timing) return;
    CUDA_CHECK(cudaEventRecord(ev_pool[i].b, stream));
  }
  // first / last copy of a call on a copy stream (which: 0 = host to device, 1 = device to host)
  void copy_begin(cudaStream_t s, int which) { CUDA_CHECK(cudaEventRecord(copy_ev[which][0], s)); copy_used[which] = true; }
  void copy_end(cudaStream_t s, int which) { CUDA_CHECK(cudaEventRecord(copy_ev[which][1], s)); }
  cudaMemPool_t pool = nullptr;  // the device's default pool: every dalloc comes from it (b2_stats.dev_peak_bytes)
  void reset_call() {
    if (pool) {
      uint64_t zero = 0;  // the high-water mark restarts from what is in use now
      CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &zero));
    }
    copy_used[0] = copy_used[1] = false;
    fetches.clear();  // a call that failed half way may have left some behind
    stage_used = 0;
    ev_used = 0;
    ev_tags.clear();
    bwt_mode_known = false;
    bz_flavor = B2_BZ2_COMPRESSJS;
    memset(&stats, 0, sizeof stats);
  }
  void collect();  // after the final sync: fold event pairs into stats

  // small control transfers that bypass the copy engines (see api.cu); to_host results are valid after sync()
  u8* stage_h = nullptr; u8* stage_d = nullptr;
  size_t stage_cap = (size_t)8 << 20, stage_used = 0;
  struct Fetch { void* dst; size_t off, bytes; };
  std::vector<Fetch> fetches;
  size_t stage_take(size_t bytes);
  void to_device(void* ddst, const void* hsrc, size_t bytes);
  void to_host(void* hdst, const void* dsrc, size_t bytes);
  void sync();
};

enum Stage {
  ST_TOTAL = 0, ST_H2D, ST_D2H, ST_RLE1, ST_BWT, ST_MTF, ST_HUFF, ST_PACK,
  ST_SCAN, ST_HDEC, ST_UNMTF, ST_IBWT, ST_UNRLE, ST_RADIX, ST_MSD_SCATTER, ST_MSD_BUCKET, ST_COUNT
};

struct StageScope {
  Ctx& c; size_t i;
  StageScope(Ctx& c_, int stage) : c(c_), i(c_.begin(stage)) {}
  ~StageScope() { try { c.end(i); } catch (...) {} }
};

// RAII device buffer (stream-ordered)
template <typename T>
struct DBuf {
  Ctx* c = nullptr; T* p = nullptr; size_t n = 0;
  DBuf() {}
  DBuf(Ctx& c_, size_t count) : c(&c_), p(c_.dalloc_t<T>(count)), n(count) {}
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  DBuf(DBuf&& o) : c(o.c), p(o.p), n(o.n) { o.p = nullptr; }
  DBuf& operator=(DBuf&& o) { release(); c = o.c; p = o.p; n = o.n; o.p = nullptr; return *this; }
  void alloc(Ctx& c_, size_t count) { release(); c = &c_; p = c_.dalloc_t<T>(count); n = count; }
  void release() { if (p && c) c->dfree(p); p = nullptr; }
  ~DBuf() { release(); }
  operator T*() const { return p; }
};

#define KLAUNCH(ctx) ((ctx).stats.kernel_launches++)
#define KCHECK() CUDA_CHECK(cudaGetLastError())
