// Shared helpers of libdgr_b200 (sm_90a only).
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "dgr_b200.h"

void dgr_set_error(const char* fmt, ...);
void dgr_note_launches(int n);   // bookkeeping for dgr_launch_count()

// knn.cu: dgr_knn_top1's fp32 brute force, one thread per f0 row; packed[i] = (sqrt(d2 + 1e-7) bits << 32) | row
// (lowest row on a tie).  One launch, skipped when live != nullptr and *live == 0.
void dgr_knn_top1_packed(const float* f0, int n0, const float* f1, int n1, int c, uint64_t* packed,
                         const int32_t* live, cudaStream_t st);

// posegraph.cu: open3d's 6x6 information matrix [[tr(Q) I - Q, [S]x], [[S]x^T, n I]] from per-CTA partials
// part[b][10] = (n, sum q, sum q q^T (xx, xy, xz, yy, yz, zz)), b < n_blocks, added in a fixed order; out[37] = the
// matrix row-major, then n.  One launch (not counted: its callers count it).
void dgr_info_final(const double* part, int n_blocks, double* out, cudaStream_t st);

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

#define DGR_TRY(expr)                 \
  do {                                \
    int32_t rc__ = (expr);            \
    if (rc__ != DGR_OK) return rc__;  \
  } while (0)

static inline unsigned dgr_blocks(int64_t n, int per_block) {
  int64_t b = (n + per_block - 1) / per_block;
  return (unsigned)(b < 1 ? 1 : b);
}

// ---------------------------------------------------------------------------------------
// coordinate keys and the open-addressing table
// ---------------------------------------------------------------------------------------
#define DGR_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

// Row count of a kernel that takes (n_max, n_dev): the device count when given, else the host bound
__device__ __forceinline__ int dgr_dev_count(const int32_t* n_dev, int64_t n_max) {
  return n_dev != nullptr ? *n_dev : (int)n_max;
}

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

// Draw number `draw` of the counter-hash stream of `seed`: uniform in [0, n).  RANSAC hypothesis h takes draws
// 4h .. 4h + 3, an FGR tuple trial k draws 3k .. 3k + 2; oracle/ransac.py restates it (sample_indices).
__device__ __forceinline__ uint32_t dgr_counter_pick(uint64_t seed, uint64_t draw, uint32_t n) {
  const uint64_t z = dgr_mix64(seed + (draw + 1) * 0x9E3779B97F4A7C15ull);
  return (uint32_t)(((z >> 32) * (uint64_t)n) >> 32);
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

// Row in cell c (0 <= c < side^3, x fastest) of the block of side = 2 reach + 1 cells centred on cell c3, batch
// column `batch`, or -1 when that cell is empty or outside the key spec's range
__device__ __forceinline__ int32_t dgr_probe_cell(int c, int side, int reach, const int c3[3], int32_t batch,
                                                  const dgr_keyspec_t& s, const uint64_t* __restrict__ keys,
                                                  const int32_t* __restrict__ vals, uint64_t mask) {
  const int dx = c % side - reach, dy = (c / side) % side - reach, dz = c / (side * side) - reach;
  const int32_t row[4] = {batch, c3[0] + dx, c3[1] + dy, c3[2] + dz};
  bool inside = true;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const long long d = (long long)row[q] - s.lo[q];
    inside = inside && d >= 0 && d < (1ll << s.bits[q]);
  }
  if (!inside) return -1;
  return dgr_hash_lookup(keys, vals, mask, dgr_pack_key(row, s));
}

// Nearest target row strictly within sqrt(best) of the point p, through a voxel hash holding at most one
// target point per cell of size `cell` (the cells within `reach` = ceil(radius / cell) of p's cell on every
// side are the candidates).  8 lanes share one query point: an aligned group of 8 lanes of the warp, lane
// `sub` probing cells sub, sub + 8, ... (a thread per point walking all (2 reach + 1)^3 cells serially waits
// on that many dependent L2 round trips).  The group's best (smaller d2, then lower row) is reduced with
// shuffles, so the answer does not depend on the probe order and every lane of the group leaves with it.
// Whole warps must call it; lanes with have == false probe nothing.  best: in = radius^2, out = its d2;
// best_j: -1 when nothing is within the radius.
__device__ __forceinline__ void dgr_voxel_nearest8(const double p[3], bool have, int sub, const float* __restrict__ tgt,
                                                   const dgr_keyspec_t& s, const uint64_t* __restrict__ keys,
                                                   const int32_t* __restrict__ vals, uint64_t mask, int32_t batch,
                                                   double cell, int reach, double& best, int& best_j) {
  const int side = 2 * reach + 1, n_cells = side * side * side;
  int c3[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c3[a] = (int)floor(p[a] / cell);
  best_j = -1;
  for (int c = sub; c < n_cells && have; c += 8) {
    const int32_t j = dgr_probe_cell(c, side, reach, c3, batch, s, keys, vals, mask);
    if (j < 0) continue;
    const double ex = p[0] - tgt[3 * (int64_t)j], ey = p[1] - tgt[3 * (int64_t)j + 1],
                 ez = p[2] - tgt[3 * (int64_t)j + 2];
    const double d2 = ex * ex + ey * ey + ez * ez;
    if (d2 < best || (d2 == best && (best_j < 0 || j < best_j))) {
      best = d2;
      best_j = j;
    }
  }
#pragma unroll
  for (int d = 1; d < 8; d <<= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, d);
    const int oj = __shfl_xor_sync(0xffffffffu, best_j, d);
    if (oj >= 0 && (best_j < 0 || ob < best || (ob == best && oj < best_j))) {
      best = ob;
      best_j = oj;
    }
  }
}

// What every search of a voxel hash requires of its arguments, checked on the host: a power-of-two table capacity,
// a positive finite cell, a positive radius, and reach = ceil(radius / cell) <= max_reach (false for NaN and an
// infinite radius; an infinite cell would give reach 0)
inline int32_t dgr_check_hash_search(int64_t cap, double cell, double radius, int max_reach) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(cell > 0 && cell < INFINITY && radius > 0, "cell and radius must be positive, the cell finite");
  if (!(ceil(radius / cell) <= (double)max_reach)) {
    dgr_set_error("%s:%d: bad argument: search radius above %d cells is not supported", __FILE__, __LINE__, max_reach);
    return DGR_ERR_ARG;
  }
  return DGR_OK;
}

// The float32 coordinate a search may read for a coordinate x stored under cell k of size `cell`: every search finds
// a row's cell as floor(double(x32) / cell), so (float)x is moved toward cell k one ulp at a time while that cell
// differs (a float64 x needs 1 step, an x keyed by a float32 division at most 2).  A coordinate already in its cell
// keeps its (float)x bits.  dgr_float32_in_cells (coords.cu) and the pair compaction (coordplan.cu) write rows with it.
__device__ __forceinline__ float dgr_float32_in_cell(double x, int32_t k, double cell) {
  float x32 = __double2float_rn(x);
#pragma unroll
  for (int s = 0; s < DGR_CELL_NUDGE_STEPS; ++s) {
    const double c = floor(__ddiv_rn((double)x32, cell));
    if (c == (double)k) break;
    x32 = nextafterf(x32, c < (double)k ? INFINITY : -INFINITY);
  }
  return x32;
}

// ---------------------------------------------------------------------------------------
// Radius neighbours of a point in its own cloud's voxel hash (one point per cell): open3d's hybrid search, restated
// in oracle/normals.py (neighbours).  Row j is in the radius of point i when d2 = |p_j - p_i|^2 < radius^2, and the
// rows are ranked by (d2, row).  Normals and colour gradients (icp.cu) and FPFH (fpfh.cu) search with these.
// ---------------------------------------------------------------------------------------
// offset e = p_j - p_i and d2 = |e|^2 evaluated as numpy does ((ex ex + ey ey) + ez ez, no contraction), so that the
// strict radius test and the (d2, row) order agree with the oracle bit for bit
__device__ __forceinline__ double dgr_offset_d2(const float* __restrict__ xyz, int32_t j, const double p[3],
                                                double e[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) e[a] = __dsub_rn((double)__ldg(xyz + 3 * (int64_t)j + a), p[a]);
  return __dadd_rn(__dadd_rn(__dmul_rn(e[0], e[0]), __dmul_rn(e[1], e[1])), __dmul_rn(e[2], e[2]));
}

// (d2, row) of a before b
__device__ __forceinline__ bool dgr_key_less(double da, int32_t ja, double db, int32_t jb) {
  return da < db || (da == db && ja < jb);
}

// Cell c of the probe block (numbered as in dgr_probe_cell) can hold a point within the radius: sum max(|d| - 1, 0)^2
// <= gap_limit = (radius / cell)^2 (1 + 1e-6), the margin covering the rounding of p / cell.  A dead cell cannot hold
// a point strictly inside the radius, so skipping it changes no neighbour list.
__host__ __device__ __forceinline__ bool dgr_cell_live(int c, int side, int reach, double gap_limit) {
  const int dx = c % side - reach, dy = (c / side) % side - reach, dz = c / (side * side) - reach;
  const int gx = dx < 0 ? -dx - 1 : dx - 1, gy = dy < 0 ? -dy - 1 : dy - 1, gz = dz < 0 ? -dz - 1 : dz - 1;
  const int s = (gx > 0 ? gx * gx : 0) + (gy > 0 ? gy * gy : 0) + (gz > 0 ? gz * gz : 0);
  return (double)s <= gap_limit;
}

inline double dgr_gap_limit(double radius, double cell) { return radius * radius * (1.0 + 1e-6) / (cell * cell); }

// The live cells of the probe block: with one point per cell, the most keys dgr_gather_in_radius appends
inline int dgr_live_cells(int reach, double gap_limit) {
  const int side = 2 * reach + 1, n_cells = side * side * side;
  int live = 0;
  for (int c = 0; c < n_cells; ++c) live += dgr_cell_live(c, side, reach, gap_limit);
  return live;
}

// The in-radius keys (d2, row) of point p, appended to kd / kj in cell order (ballot + prefix popcount), dead cells
// not probed.  A whole warp calls it for one point; it returns the key count in every lane, with the keys visible
// to the whole warp.  kd / kj have room for dgr_live_cells(reach, gap_limit) keys.
__device__ __forceinline__ int dgr_gather_in_radius(const float* __restrict__ xyz, const double p[3], double cell,
                                                    int reach, double r2, double gap_limit, int32_t batch,
                                                    const dgr_keyspec_t& s, const uint64_t* __restrict__ keys,
                                                    const int32_t* __restrict__ vals, uint64_t mask, double* kd,
                                                    int32_t* kj) {
  const int side = 2 * reach + 1, n_cells = side * side * side;
  const int lane = threadIdx.x & 31;
  int c3[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c3[a] = (int)floor(p[a] / cell);
  int cnt = 0;
  for (int c0 = 0; c0 < n_cells; c0 += 32) {
    const int c = c0 + lane;
    int32_t j = -1;
    double d2 = 0.0;
    if (c < n_cells && dgr_cell_live(c, side, reach, gap_limit)) {
      j = dgr_probe_cell(c, side, reach, c3, batch, s, keys, vals, mask);
      if (j >= 0) {
        double e[3];
        d2 = dgr_offset_d2(xyz, j, p, e);
        if (!(d2 < r2)) j = -1;
      }
    }
    const unsigned ball = __ballot_sync(0xffffffffu, j >= 0);
    if (j >= 0) {
      const int pos = cnt + __popc(ball & ((1u << lane) - 1u));
      kd[pos] = d2;
      kj[pos] = j;
    }
    cnt += __popc(ball);
  }
  __syncwarp();
  return cnt;
}

// Rank of the key (d2, j) among the cnt keys of kd / kj: how many come before it (keys are distinct: rows are).
// The loop walks pointers: indexed as kd[l], the unrolled loop recomputed the warp's slice base every few keys.
__device__ __forceinline__ int dgr_key_rank(const double* kd, const int32_t* kj, int cnt, double d2, int32_t j) {
  int rank = 0;
  for (const double* end = kd + cnt; kd < end; ++kd, ++kj) rank += dgr_key_less(*kd, *kj, d2, j);
  return rank;
}

// ---------------------------------------------------------------------------------------
// exclusive scan of `nb` ints in place with one block; returns the total (valid in every thread)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int dgr_block_scan_inplace(int32_t* cnt, int64_t nb) {
  __shared__ int carry_s;
  __shared__ int wsum[32];
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = 0; base < nb; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int v = (i < nb) ? cnt[i] : 0;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += t;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    int wbase = 0, tot = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      const int sm = wsum[w];
      if (w < warp) wbase += sm;
      tot += sm;
    }
    const int carry = carry_s;
    if (i < nb) cnt[i] = carry + wbase + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + tot;
    __syncthreads();
  }
  return carry_s;
}

// ---------------------------------------------------------------------------------------
// block-wide exclusive scan of one int per thread (blockDim.x == BS).  The warp totals stay in shared memory until
// the caller's next __syncthreads, so two calls need one between them.
// ---------------------------------------------------------------------------------------
template <int BS>
__device__ __forceinline__ int dgr_block_exclusive_scan(int v, int* total) {
  __shared__ int warp_sums[BS / 32];
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
  for (int w = 0; w < BS / 32; ++w) {
    int s = warp_sums[w];
    if (w < warp) base += s;
    tot += s;
  }
  if (total) *total = tot;
  return base + inc - v;
}

// ---------------------------------------------------------------------------------------
// coords.cu: the count scan and the ordered selection shared by the unique-coordinate pass, FGR and the RANSAC
// ---------------------------------------------------------------------------------------
// exclusive scan in place of the per-block counts cnt[0, nb) with one block; cnt[nb] = the total
void dgr_scan_counts(int32_t* cnt, int64_t nb, cudaStream_t st);
// The first `cap` flagged rows of flag[0, n), in row order: sel[rank] = h0 + row, one 256-row block per count of
// blk (scanned by dgr_scan_counts).  live (optional): the launch does nothing when *live == 0.
void dgr_select_first(const int32_t* flag, const int32_t* blk, int64_t n, int64_t cap, int64_t h0, int32_t* sel,
                      const int32_t* live, cudaStream_t st);

// ---------------------------------------------------------------------------------------
// Fixed-order fp64 sums.  Each value's lanes are added by xor butterfly (16, 8, 4, 2, 1), then the BS / 32 warp
// partials from warp 0 upward starting at +0.0 (so a sum of -0.0 terms is +0.0); the oracles restate this order.
// ---------------------------------------------------------------------------------------
// Sum N per-thread values over a block of BS threads.  Thread k < N returns the sum of value k, every other thread
// +0.0.  part: shared [BS / 32][>= N], rewritten by the next call only after a __syncthreads.  Whole blocks call it.
template <int BS, int N, int W>
__device__ __forceinline__ double dgr_block_sum(const double (&v)[N], double (*part)[W]) {
  static_assert(N <= W, "partial rows too narrow");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double x = v[k];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);
    if (lane == 0) part[warp][k] = x;
  }
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x < N)
    for (int w = 0; w < BS / 32; ++w) s += part[w][threadIdx.x];
  return s;
}

// Shared memory of dgr_allreduce for up to W values, BS threads and clusters of up to CS CTAs; embedded as the first
// member of a kernel's shared struct.
template <int W, int BS, int CS>
struct DgrReduceShared {
  double slots[2][CS][W];                               // per-CTA sums, double-buffered by the caller's parity
  double part[BS / 32][W];
  double tot[W];
};

// Sum N per-thread values over the CTA (CS == 1) or its cluster of CS CTAs: dgr_block_sum, then the CTA sums in rank
// order through distributed shared memory.  Every CTA ends with the same sh.tot[0, N); parity alternates the slots
// so that consecutive calls need one cluster barrier each.
template <int CS, int N, int W, int BS, int CSMAX>
__device__ __forceinline__ void dgr_allreduce(DgrReduceShared<W, BS, CSMAX>& sh, const double (&v)[N], int& parity) {
  static_assert(CS <= CSMAX, "cluster larger than the slots");
  double s = dgr_block_sum<BS>(v, sh.part);
  if constexpr (CS == 1) {
    if (threadIdx.x < N) sh.tot[threadIdx.x] = s;
  } else {
    cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
    const unsigned rank = cluster.block_rank();
    if (threadIdx.x < N)
      for (unsigned r = 0; r < CS; ++r) cluster.map_shared_rank(&sh, r)->slots[parity][rank][threadIdx.x] = s;
    cluster.sync();
    if (threadIdx.x < N) {
      s = 0.0;
      for (int r = 0; r < CS; ++r) s += sh.slots[parity][r][threadIdx.x];
      sh.tot[threadIdx.x] = s;
    }
  }
  __syncthreads();
  parity ^= 1;
}

// ---------------------------------------------------------------------------------------
// Workspace carving: regions of 8-byte words handed out in order.  With a null base it only counts the words, so one
// layout function gives both the size a dgr_*_ws_elems reports and the regions.
// ---------------------------------------------------------------------------------------
struct DgrCarver {
  uint64_t* base;
  int64_t words = 0;
  explicit DgrCarver(void* b) : base(static_cast<uint64_t*>(b)) {}
  // n elements of T, rounded up to whole words
  template <class T>
  T* take(int64_t n) {
    T* p = base != nullptr ? reinterpret_cast<T*>(base + words) : nullptr;
    words += (n * (int64_t)sizeof(T) + 7) / 8;
    return p;
  }
};
