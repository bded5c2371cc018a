// common.cuh -- shared device helpers for the b2bz kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdexcept>
#include <string>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

struct B2Error {
  int code;
  std::string msg;
};

#define CUDA_CHECK(x)                                                                              \
  do {                                                                                             \
    cudaError_t e_ = (x);                                                                          \
    if (e_ != cudaSuccess) {                                                                       \
      char b_[512];                                                                                \
      snprintf(b_, sizeof b_, "CUDA error %s at %s:%d (%s)", cudaGetErrorString(e_), __FILE__, __LINE__, #x); \
      throw B2Error{-200, b_};                                                                     \
    }                                                                                              \
  } while (0)

// Blocks of a batch live at a fixed stride of 2^20 positions (max bzip2 block = 900000 < 2^20):
// global slot g = (block << SEG_SHIFT) | local position.
#define SEG_SHIFT 20
#define SEG_SIZE (1u << SEG_SHIFT)
#define SEG_MASK (SEG_SIZE - 1u)

#define FULL_MASK 0xffffffffu

__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ u32 lanemask_lt() {
  u32 m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// ---- warp / block scans --------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_incl_add(T v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    T t = __shfl_up_sync(FULL_MASK, v, o);
    if (lane_id() >= (u32)o) v += t;
  }
  return v;
}
template <typename T>
__device__ __forceinline__ T warp_incl_max(T v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    T t = __shfl_up_sync(FULL_MASK, v, o);
    if (lane_id() >= (u32)o) v = v > t ? v : t;
  }
  return v;
}
template <typename T>
__device__ __forceinline__ T warp_reduce_add(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}
template <typename T>
__device__ __forceinline__ T warp_reduce_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    T t = __shfl_xor_sync(FULL_MASK, v, o);
    v = v > t ? v : t;
  }
  return v;
}

// Block-wide exclusive add scan of one value per thread.  `ws` needs (THREADS/32 + 1) entries.
// Returns the exclusive prefix; *total receives the block total (valid for all threads).
template <int THREADS, typename T>
__device__ __forceinline__ T block_excl_add(T v, T* ws, T* total) {
  T inc = warp_incl_add(v);
  const int w = threadIdx.x >> 5;
  if (lane_id() == 31) ws[w] = inc;
  __syncthreads();
  if (w == 0) {
    T x = (lane_id() < THREADS / 32) ? ws[lane_id()] : T(0);
    T xi = warp_incl_add(x);
    if (lane_id() < THREADS / 32) ws[lane_id()] = xi - x;
    if (lane_id() == THREADS / 32 - 1) ws[THREADS / 32] = xi;
  }
  __syncthreads();
  T r = ws[w] + inc - v;
  *total = ws[THREADS / 32];
  __syncthreads();
  return r;
}
// Block-wide inclusive max scan of one value per thread.  `ws` needs (THREADS/32 + 1) entries.
template <int THREADS, typename T>
__device__ __forceinline__ T block_incl_max(T v, T* ws, T* total) {
  T inc = warp_incl_max(v);
  const int w = threadIdx.x >> 5;
  if (lane_id() == 31) ws[w] = inc;
  __syncthreads();
  if (w == 0) {
    T x = (lane_id() < THREADS / 32) ? ws[lane_id()] : T(0);
    T xi = warp_incl_max(x);
    T xe = __shfl_up_sync(FULL_MASK, xi, 1);
    if (lane_id() == 0) xe = T(0);
    if (lane_id() < THREADS / 32) ws[lane_id()] = xe;
    if (lane_id() == THREADS / 32 - 1) ws[THREADS / 32] = xi;
  }
  __syncthreads();
  T c = ws[w];
  T r = inc > c ? inc : c;
  *total = ws[THREADS / 32];
  __syncthreads();
  return r;
}

// ---- decoupled look-back across tiles (single-pass chained scan) ----------------------
// One 64-bit status word per tile: bits 63..62 = flag, bits 31..0 = value.  Flag and value
// travel in one word, so no fence is needed between them.
#define LB_EMPTY 0ull
#define LB_AGG (1ull << 62)
#define LB_PREFIX (2ull << 62)
#define LB_FLAGS (3ull << 62)

struct OpAdd {
  __device__ __forceinline__ u32 operator()(u32 a, u32 b) const { return a + b; }
  static __device__ __forceinline__ u32 identity() { return 0; }
};
struct OpMax {
  __device__ __forceinline__ u32 operator()(u32 a, u32 b) const { return a > b ? a : b; }
  static __device__ __forceinline__ u32 identity() { return 0; }
};

__device__ __forceinline__ u64 ld_volatile_u64(const u64* p) {
  u64 v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_volatile_u64(u64* p, u64 v) {
  asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ u32 ld_volatile_u32(const u32* p) {
  u32 v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_volatile_u32(u32* p, u32 v) {
  asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Called by ONE FULL WARP.  Publishes this tile's aggregate, walks back over predecessor
// tiles and returns the exclusive prefix (valid in every lane); then publishes the inclusive
// prefix.  Tiles must have been handed out in increasing order (atomic ticket) so that all
// predecessors are running or done.
template <class Op>
__device__ __forceinline__ u32 lookback_warp(u64* status, u32 tile, u32 aggregate, Op op) {
  const u32 lane = lane_id();
  if (tile == 0) {
    if (lane == 0) st_volatile_u64(&status[0], LB_PREFIX | (u64)aggregate);
    return Op::identity();
  }
  if (lane == 0) st_volatile_u64(&status[tile], LB_AGG | (u64)aggregate);
  u32 excl = Op::identity();
  int base = (int)tile - 1;  // lane l looks at tile base - l
  while (true) {
    int t = base - (int)lane;
    u64 w = LB_PREFIX;  // tiles before 0 behave like an identity prefix
    if (t >= 0) {
      do {
        w = ld_volatile_u64(&status[t]);
      } while ((w & LB_FLAGS) == LB_EMPTY);
    }
    u32 has_prefix = __ballot_sync(FULL_MASK, (w & LB_FLAGS) == LB_PREFIX);
    u32 val = (t >= 0) ? (u32)w : Op::identity();
    // lanes up to and including the first PREFIX lane contribute
    u32 first = has_prefix ? (u32)(__ffs(has_prefix) - 1) : 32u;
    u32 contrib = (lane <= first) ? val : Op::identity();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) contrib = op(contrib, __shfl_xor_sync(FULL_MASK, contrib, o));
    excl = op(excl, contrib);
    if (has_prefix) break;
    base -= 32;
  }
  if (lane == 0) st_volatile_u64(&status[tile], LB_PREFIX | (u64)op(excl, aggregate));
  return excl;
}
