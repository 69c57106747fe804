// Shared helpers of libdgr_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "dgr_b200.h"

void dgr_set_error(const char* fmt, ...);
void dgr_note_launches(int n);   // bookkeeping for dgr_launch_count()

#define DGR_CUDA_CHECK(expr)                                                            \
  do {                                                                                  \
    cudaError_t e__ = (expr);                                                           \
    if (e__ != cudaSuccess) {                                                           \
      dgr_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
      return DGR_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

#define DGR_LAUNCH_CHECK() DGR_CUDA_CHECK(cudaGetLastError())

// Opt a kernel in to `bytes` of dynamic shared memory.  The attribute is per FUNCTION, not per launch, and only
// ever raised here (monotone maximum per call site, under a mutex): two host threads - two pairs in flight -
// that set launch-specific sizes without this would race (thread A sets 100 KB, thread B sets 60 KB, A's launch
// then fails with "invalid argument").  cudaFuncSetAttribute is a driver call that takes the context lock, so
// it is skipped once the attribute is large enough.
#include <mutex>
#define DGR_ENSURE_SMEM(func, bytes)                                                                 \
  do {                                                                                               \
    static std::atomic<int> cur_smem_{0};                                                            \
    static std::mutex smem_mu_;                                                                      \
    if ((int)(bytes) > cur_smem_.load(std::memory_order_acquire)) {                                  \
      std::lock_guard<std::mutex> lock_(smem_mu_);                                                   \
      if ((int)(bytes) > cur_smem_.load(std::memory_order_relaxed)) {                                \
        DGR_CUDA_CHECK(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
        cur_smem_.store((int)(bytes), std::memory_order_release);                                    \
      }                                                                                              \
    }                                                                                                \
  } while (0)

#define DGR_ARG_CHECK(cond, msg)                                      \
  do {                                                                \
    if (!(cond)) {                                                    \
      dgr_set_error("%s:%d: bad argument: %s", __FILE__, __LINE__, msg); \
      return DGR_ERR_ARG;                                             \
    }                                                                 \
  } while (0)

static inline unsigned dgr_blocks(int64_t n, int per_block) {
  int64_t b = (n + per_block - 1) / per_block;
  return (unsigned)(b < 1 ? 1 : b);
}

// ---------------------------------------------------------------------------------------
// coordinate keys and the open-addressing table
// ---------------------------------------------------------------------------------------
#define DGR_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

__device__ __forceinline__ uint64_t dgr_pack_key(const int32_t* __restrict__ row,
                                                 const dgr_keyspec_t& s) {
  uint64_t k = 0;
#pragma unroll
  for (int i = 0; i < DGR_MAX_COLS; ++i)
    if (i < s.ncols) k += (uint64_t)(uint32_t)(row[i] - s.lo[i]) << s.shift[i];
  return k;
}

__device__ __forceinline__ uint64_t dgr_mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// Claim (or find) the slot of `key`; linear probing.
__device__ __forceinline__ uint32_t dgr_hash_insert(uint64_t* keys, uint64_t mask, uint64_t key) {
  uint64_t s = dgr_mix64(key) & mask;
  while (true) {
    unsigned long long prev =
        atomicCAS(reinterpret_cast<unsigned long long*>(keys + s), DGR_EMPTY_KEY, key);
    if (prev == DGR_EMPTY_KEY || prev == key) return (uint32_t)s;
    s = (s + 1) & mask;
  }
}

__device__ __forceinline__ int32_t dgr_hash_lookup(const uint64_t* __restrict__ keys,
                                                   const int32_t* __restrict__ vals, uint64_t mask,
                                                   uint64_t key) {
  // ld.global.cg (L2, coherent): random 8-byte probes gain nothing from L1, and a table is written by the
  // kernels launched just before its readers - no reliance on the non-coherent path being flushed in between
  uint64_t s = dgr_mix64(key) & mask;
  while (true) {
    uint64_t k = __ldcg(reinterpret_cast<const unsigned long long*>(keys) + s);
    if (k == key) return __ldcg(vals + s);
    if (k == DGR_EMPTY_KEY) return -1;
    s = (s + 1) & mask;
  }
}

// ---------------------------------------------------------------------------------------
// block-wide exclusive scan of one int per thread (blockDim.x == 256)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int dgr_block_exclusive_scan_256(int v, int* total) {
  __shared__ int warp_sums[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    int s = warp_sums[w];
    if (w < warp) base += s;
    tot += s;
  }
  __syncthreads();
  if (total) *total = tot;
  return base + inc - v;
}
