// Integer coordinate work of the sparse-tensor engine: voxelisation, coordinate hash,
// first-occurrence dedup, strided maps and kernel maps.  All of it is HBM/L2-bound
// integer work: coalesced row-major loads, 64-bit packed keys so one probe is one
// 8-byte access, open-addressing tables sized to a load factor <= 0.5 that stay
// L2-resident (a 76k-voxel cloud is a 2 MB table).
//
// Replaces the MinkowskiEngine pieces reached from core/deep_global_registration.py:152-167
// (sparse_quantize, batched_coordinates, SparseTensor coordinate map) and the kernel-map
// builder behind model/residual_block.py:31-80.
#include <limits.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kScanElems = 2048;   // elements per block in the flag scans (256 threads x 8)

// ---------------------------------------------------------------------------------------
// voxelisation
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void quantize_kernel(const T* __restrict__ xyz, int64_t n, T voxel, int32_t batch,
                                int32_t* __restrict__ coords) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  // true IEEE division in the input dtype, then floor (numpy: np.floor(xyz / voxel))
  T x = xyz[3 * r + 0] / voxel, y = xyz[3 * r + 1] / voxel, z = xyz[3 * r + 2] / voxel;
  int4 c;
  c.x = batch;
  c.y = (int32_t)floor(x);
  c.z = (int32_t)floor(y);
  c.w = (int32_t)floor(z);
  reinterpret_cast<int4*>(coords)[r] = c;
}

__global__ void minmax_init_kernel(int32_t* minmax, int ncols) {
  int i = threadIdx.x;
  if (i < ncols) {
    minmax[i] = INT_MAX;
    minmax[ncols + i] = INT_MIN;
  }
}

__global__ void minmax_kernel(const int32_t* __restrict__ coords, int64_t n, int ncols,
                              int32_t* minmax) {
  int lo[DGR_MAX_COLS], hi[DGR_MAX_COLS];
#pragma unroll
  for (int c = 0; c < DGR_MAX_COLS; ++c) {
    lo[c] = INT_MAX;
    hi[c] = INT_MIN;
  }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n;
       r += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
    for (int c = 0; c < DGR_MAX_COLS; ++c)
      if (c < ncols) {
        int v = coords[r * ncols + c];
        lo[c] = min(lo[c], v);
        hi[c] = max(hi[c], v);
      }
  }
#pragma unroll
  for (int c = 0; c < DGR_MAX_COLS; ++c) {
    if (c >= ncols) break;
    int l = lo[c], h = hi[c];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      l = min(l, __shfl_xor_sync(0xffffffffu, l, d));
      h = max(h, __shfl_xor_sync(0xffffffffu, h, d));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin(minmax + c, l);
      atomicMax(minmax + ncols + c, h);
    }
  }
}

__global__ void keyspec_kernel(const int32_t* __restrict__ minmax, int ncols, int margin,
                               dgr_keyspec_t* spec) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  dgr_keyspec_t s;
  s.ncols = ncols;
  s.overflow = 0;
  int shift = 0;
  for (int c = 0; c < DGR_MAX_COLS; ++c) {
    s.lo[c] = 0;
    s.shift[c] = 0;
    s.bits[c] = 0;
    if (c >= ncols) continue;
    long long lo = minmax[c], hi = minmax[ncols + c];
    if (lo > hi) lo = hi = 0;   // empty input
    if (c > 0) {
      lo -= margin;
      hi += margin;
    }
    unsigned long long extent = (unsigned long long)(hi - lo + 1);
    int bits = 1;
    while ((1ull << bits) < extent) ++bits;
    s.lo[c] = (int32_t)lo;
    s.bits[c] = bits;
    s.shift[c] = shift;
    shift += bits;
    if (lo < INT_MIN || hi > INT_MAX) s.overflow = 1;
  }
  if (shift > 63) s.overflow = 1;
  *spec = s;
}

// ---------------------------------------------------------------------------------------
// hash table
// ---------------------------------------------------------------------------------------
__global__ void hash_clear_kernel(uint64_t* keys, int32_t* vals, int64_t cap) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cap) {
    keys[i] = DGR_EMPTY_KEY;
    vals[i] = INT_MAX;
  }
}

// insert every row; the table value converges to the smallest row index per key
__global__ void insert_min_kernel(const int32_t* __restrict__ coords, int64_t n, int ncols,
                                  const dgr_keyspec_t* __restrict__ spec_p, uint64_t* keys,
                                  int32_t* vals, uint64_t mask, int32_t* __restrict__ slot) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const dgr_keyspec_t s = *spec_p;
  uint32_t sl = dgr_hash_insert(keys, mask, dgr_pack_key(coords + r * ncols, s));
  atomicMin(vals + sl, (int32_t)r);
  slot[r] = (int32_t)sl;
}

__global__ void winner_flag_kernel(const int32_t* __restrict__ slot, const int32_t* __restrict__ vals,
                                   int64_t n, int32_t* __restrict__ flag) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) flag[r] = (vals[slot[r]] == (int32_t)r) ? 1 : 0;
}

// per-block population count of flag > 0 (flag array) or entry >= 0 (neighbour table)
template <bool kNonNegative>
__global__ void block_count_kernel(const int32_t* __restrict__ v, int64_t n, int32_t* block_cnt) {
  // grid: (blocks per segment, segments); segment = blockIdx.y, each of length n
  const int64_t base = (int64_t)blockIdx.y * n;
  const int64_t start = (int64_t)blockIdx.x * kScanElems;
  int c = 0;
#pragma unroll
  for (int e = 0; e < kScanElems / kThreads; ++e) {
    int64_t i = start + e * kThreads + threadIdx.x;
    if (i < n) {
      int x = v[base + i];
      c += kNonNegative ? (x >= 0) : (x > 0);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  __shared__ int ws[kThreads / 32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += ws[w];
    block_cnt[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = t;
  }
}

// single-block exclusive scan in place over nb entries; entry nb receives the total.
__global__ void scan_blocks_kernel(int32_t* cnt, int64_t nb, int32_t* kofs = nullptr, int K = 0, int bpk = 0,
                                   const dgr_keyspec_t* spec = nullptr) {
  __shared__ int carry_s;
  __shared__ int wsum[32];
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = 0; base < nb; base += blockDim.x) {
    int64_t i = base + threadIdx.x;
    int v = (i < nb) ? cnt[i] : 0;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += t;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    int wbase = 0, tot = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      int s = wsum[w];
      if (w < warp) wbase += s;
      tot += s;
    }
    int carry = carry_s;
    if (i < nb) cnt[i] = carry + wbase + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) cnt[nb] = carry_s;
  if (kofs != nullptr) {   // bucket offsets of a kernel map (+ the key-overflow flag), same launch
    __syncthreads();
    for (int k = threadIdx.x; k <= K + 1; k += blockDim.x)
      kofs[k] = (k <= K) ? cnt[(int64_t)k * bpk] : (spec != nullptr ? spec->overflow : 0);
  }
}

// rank winners: sel[rank] = row, table value <- rank
__global__ void unique_scatter_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ slot,
                                      int64_t n, const int32_t* __restrict__ block_ofs,
                                      int32_t* __restrict__ sel, int32_t* vals) {
  const int64_t start = (int64_t)blockIdx.x * kScanElems + (int64_t)threadIdx.x * 8;
  int f[8], c = 0;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    int64_t i = start + e;
    f[e] = (i < n) ? flag[i] : 0;
    c += f[e];
  }
  int pos = block_ofs[blockIdx.x] + dgr_block_exclusive_scan_256(c, nullptr);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (f[e]) {
      int64_t i = start + e;
      sel[pos] = (int32_t)i;
      vals[slot[i]] = pos;
      ++pos;
    }
  }
}

__global__ void inverse_kernel(const int32_t* __restrict__ slot, const int32_t* __restrict__ vals,
                               int64_t n, int32_t* __restrict__ inverse) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) inverse[r] = vals[slot[r]];
}

__global__ void copy_total_kernel(const int32_t* src, const dgr_keyspec_t* spec, int32_t* dst) {
  dst[0] = *src;
  dst[1] = spec->overflow;   // one host read returns the count and the key-overflow flag
}

__global__ void hash_find_kernel(const int32_t* __restrict__ coords, int64_t n, int ncols,
                                 const dgr_keyspec_t* __restrict__ spec_p,
                                 const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                 uint64_t mask, int32_t* __restrict__ rows) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const dgr_keyspec_t s = *spec_p;
  // rows outside the packed range cannot be present
  bool inside = true;
  for (int c = 0; c < s.ncols; ++c) {
    long long d = (long long)coords[r * ncols + c] - s.lo[c];
    inside = inside && d >= 0 && d < (1ll << s.bits[c]);
  }
  rows[r] = inside ? dgr_hash_lookup(keys, vals, mask, dgr_pack_key(coords + r * ncols, s)) : -1;
}

__global__ void gather_rows_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ idx,
                                   int64_t n, int ncols, int32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * ncols) return;
  int64_t r = i / ncols;
  int c = (int)(i - r * ncols);
  out[i] = src[(int64_t)idx[r] * ncols + c];
}

__global__ void stride_coords_kernel(const int32_t* __restrict__ in, int64_t n, int ncols, int stride,
                                     int32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * ncols) return;
  int c = (int)(i % ncols);
  int v = in[i];
  if (c > 0) {
    int q = v / stride;
    if ((v % stride != 0) && (v < 0)) --q;   // floor toward -inf
    v = q * stride;
  }
  out[i] = v;
}

// ---------------------------------------------------------------------------------------
// kernel maps
// ---------------------------------------------------------------------------------------
constexpr int kKappaChunk = 32;

// One-hash Bloom filter over the keys of a table (16 bits per slot of capacity): 6-D kernel
// maps miss on 99.7 % of their probes; the filter is small enough (cap * 2 bytes) to live in
// L1, so most misses never travel to L2.
__device__ __forceinline__ uint64_t bloom_bit(uint64_t key, uint64_t bit_mask) {
  return (dgr_mix64(key ^ 0x9e3779b97f4a7c15ull) >> 17) & bit_mask;
}

__global__ void bloom_build_kernel(const uint64_t* __restrict__ keys, int64_t cap, uint32_t* bloom,
                                   uint64_t bit_mask) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  const uint64_t k = keys[i];
  if (k == DGR_EMPTY_KEY) return;
  const uint64_t b = bloom_bit(k, bit_mask);
  atomicOr(bloom + (b >> 5), 1u << (b & 31));
}

__global__ void kernel_map_table_kernel(const int32_t* __restrict__ out_coords, int64_t n_out, int ncols,
                                        const dgr_keyspec_t* __restrict__ spec_p,
                                        const uint64_t* __restrict__ keys,
                                        const int32_t* __restrict__ vals, uint64_t mask,
                                        const uint32_t* __restrict__ bloom, uint64_t bit_mask,
                                        const int32_t* __restrict__ offsets, int K,
                                        int32_t* __restrict__ nbr, int32_t* block_cnt, int bpk) {
  __shared__ long long delta[kKappaChunk];
  const dgr_keyspec_t s = *spec_p;
  const int k0 = blockIdx.y * kKappaChunk;
  const int kn = min(kKappaChunk, K - k0);
  if (threadIdx.x < kn) {
    long long d = 0;
    const int32_t* o = offsets + (int64_t)(k0 + threadIdx.x) * (ncols - 1);
    for (int a = 0; a < ncols - 1; ++a) d += (long long)o[a] * (1ll << s.shift[a + 1]);
    delta[threadIdx.x] = d;
  }
  __syncthreads();
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = j < n_out;
  const uint64_t key = live ? dgr_pack_key(out_coords + j * ncols, s) : 0;
  int32_t* dst = nbr + (int64_t)k0 * n_out + j;
  const int cnt_col = (int)(((int64_t)blockIdx.x * blockDim.x) / kScanElems);   // 2048-row counting block
  for (int kk = 0; kk < kn; kk += 4) {
    // four independent probes in flight: filter words first, table only on a filter hit
    uint64_t q[4];
    bool maybe[4];
    int32_t found[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      q[u] = key + (uint64_t)delta[min(kk + u, kn - 1)];
      if (bloom != nullptr) {
        const uint64_t b = bloom_bit(q[u], bit_mask);
        maybe[u] = (__ldg(bloom + (b >> 5)) >> (b & 31)) & 1u;
      } else {
        maybe[u] = true;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      found[u] = (live && kk + u < kn && maybe[u]) ? dgr_hash_lookup(keys, vals, mask, q[u]) : -1;
      if (live && kk + u < kn) dst[(int64_t)(kk + u) * n_out] = found[u];
    }
    if (block_cnt != nullptr) {     // fused population count: saves a full pass over the table
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = __syncthreads_count(found[u] >= 0);
        if (threadIdx.x == 0 && kk + u < kn && c > 0)
          atomicAdd(block_cnt + (int64_t)(k0 + kk + u) * bpk + cnt_col, c);
      }
    }
  }
}

__global__ void kernel_map_fill_kernel(const int32_t* __restrict__ nbr, int64_t n_out,
                                       const int32_t* __restrict__ block_ofs,
                                       int32_t* __restrict__ in_idx, int32_t* __restrict__ out_idx) {
  const int64_t base = (int64_t)blockIdx.y * n_out;
  const int64_t start = (int64_t)blockIdx.x * kScanElems + (int64_t)threadIdx.x * 8;
  int v[8], c = 0;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    int64_t j = start + e;
    v[e] = (j < n_out) ? nbr[base + j] : -1;
    c += (v[e] >= 0);
  }
  int pos = block_ofs[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] +
            dgr_block_exclusive_scan_256(c, nullptr);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (v[e] >= 0) {
      in_idx[pos] = v[e];
      out_idx[pos] = (int32_t)(start + e);
      ++pos;
    }
  }
}

// gridDim.x == 2: block 0 writes the plain list, block 1 the paired one (both work lists of a map in one launch)
__global__ void tiles_kernel(const int32_t* __restrict__ kofs, int K, int tile_rows, int n_tiles, int pair,
                             int32_t* __restrict__ tile_k, int32_t* __restrict__ tile_start, int n_tiles_b = 0,
                             int32_t* __restrict__ tile_k_b = nullptr, int32_t* __restrict__ tile_start_b = nullptr) {
  if (blockIdx.x == 1) {
    pair = 1;
    n_tiles = n_tiles_b;
    tile_k = tile_k_b;
    tile_start = tile_start_b;
  }
  extern __shared__ int tofs[];   // K + 1 exclusive tile offsets
  __shared__ int wsum[32];
  __shared__ int carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < K; base += blockDim.x) {   // block-wide scan, 1024 buckets per round
    const int k = base + threadIdx.x;
    int v = k < K ? (kofs[k + 1] - kofs[k] + tile_rows - 1) / tile_rows : 0;
    if (pair) v = (v + 1) & ~1;     // CTA pairs: an even number of tiles per offset (last one may be empty)
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, inc, d);
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
    if (k < K) tofs[k] = carry + wbase + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) tofs[K] = carry_s;
  __syncthreads();
  for (int t = threadIdx.x; t < n_tiles; t += blockDim.x) {
    int lo = 0, hi = K;   // largest k with tofs[k] <= t (non-empty: tofs[k + 1] > t)
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (tofs[mid] <= t) lo = mid; else hi = mid;
    }
    tile_k[t] = lo;
    tile_start[t] = kofs[lo] + (t - tofs[lo]) * tile_rows;
  }
}

}  // namespace

// =========================================================================================
// C ABI
// =========================================================================================
extern "C" {

int64_t dgr_kmap_ws_elems(int32_t K, int64_t n_out);

int32_t dgr_coords_minmax(const int32_t* coords, int64_t n, int32_t ncols, int32_t* minmax,
                          void* stream) {
  DGR_ARG_CHECK(ncols >= 1 && ncols <= DGR_MAX_COLS, "ncols out of range");
  cudaStream_t st = (cudaStream_t)stream;
  minmax_init_kernel<<<1, 32, 0, st>>>(minmax, ncols);
  if (n > 0) {
    unsigned blocks = dgr_blocks(n, kThreads * 4);
    if (blocks > 1056) blocks = 1056;   // 132 SMs x 8
    minmax_kernel<<<blocks, kThreads, 0, st>>>(coords, n, ncols, minmax);
  }
  dgr_note_launches(n > 0 ? 2 : 1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_quantize_points(const void* xyz, int32_t is_f64, int64_t n, double voxel, int32_t batch,
                            int32_t* coords, int32_t* minmax, void* stream) {
  DGR_ARG_CHECK(voxel > 0, "voxel size must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  if (n > 0) {
    if (is_f64)
      quantize_kernel<double><<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(
          (const double*)xyz, n, voxel, batch, coords);
    else
      quantize_kernel<float><<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(
          (const float*)xyz, n, (float)voxel, batch, coords);
    dgr_note_launches(1);
    DGR_LAUNCH_CHECK();
  }
  return dgr_coords_minmax(coords, n, 4, minmax, stream);
}

int32_t dgr_keyspec_build(const int32_t* minmax, int32_t ncols, int32_t margin, dgr_keyspec_t* spec,
                          void* stream) {
  DGR_ARG_CHECK(ncols >= 1 && ncols <= DGR_MAX_COLS, "ncols out of range");
  keyspec_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(minmax, ncols, margin, spec);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_hash_clear(uint64_t* keys, int32_t* vals, int64_t cap, void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  hash_clear_kernel<<<dgr_blocks(cap, kThreads), kThreads, 0, (cudaStream_t)stream>>>(keys, vals, cap);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int64_t dgr_scan_ws_elems(int64_t n) { return (n + kScanElems - 1) / kScanElems + 2; }

int32_t dgr_unique_first(const int32_t* coords, int64_t n, int32_t ncols, const dgr_keyspec_t* spec,
                         uint64_t* keys, int32_t* vals, int64_t cap, int32_t* sel, int32_t* inverse,
                         int32_t* n_unique, int32_t* slot_ws, int32_t* rank_ws, int32_t* scan_ws,
                         void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(cap >= 2 * n || n == 0, "capacity must be at least 2n");
  DGR_ARG_CHECK(n < (int64_t)INT_MAX, "too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const uint64_t mask = (uint64_t)cap - 1;
  if (n == 0) {
    DGR_CUDA_CHECK(cudaMemsetAsync(n_unique, 0, 2 * sizeof(int32_t), st));
    return DGR_OK;
  }
  const unsigned nb = dgr_blocks(n, kScanElems);
  insert_min_kernel<<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(coords, n, ncols, spec, keys, vals,
                                                                   mask, slot_ws);
  winner_flag_kernel<<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(slot_ws, vals, n, rank_ws);
  block_count_kernel<false><<<dim3(nb, 1), kThreads, 0, st>>>(rank_ws, n, scan_ws);
  scan_blocks_kernel<<<1, 1024, 0, st>>>(scan_ws, nb);
  unique_scatter_kernel<<<nb, kThreads, 0, st>>>(rank_ws, slot_ws, n, scan_ws, sel, vals);
  inverse_kernel<<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(slot_ws, vals, n, inverse);
  copy_total_kernel<<<1, 1, 0, st>>>(scan_ws + nb, spec, n_unique);
  dgr_note_launches(7);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_hash_find(const int32_t* coords, int64_t n, int32_t ncols, const dgr_keyspec_t* spec,
                      const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t* rows_out,
                      void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  if (n == 0) return DGR_OK;
  hash_find_kernel<<<dgr_blocks(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      coords, n, ncols, spec, keys, vals, (uint64_t)cap - 1, rows_out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_gather_rows_i32(const int32_t* src, const int32_t* idx, int64_t n, int32_t ncols,
                            int32_t* out, void* stream) {
  if (n == 0) return DGR_OK;
  gather_rows_kernel<<<dgr_blocks(n * ncols, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      src, idx, n, ncols, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_stride_coords(const int32_t* coords, int64_t n, int32_t ncols, int32_t out_stride,
                          int32_t* out, void* stream) {
  DGR_ARG_CHECK(out_stride >= 1, "stride must be positive");
  if (n == 0) return DGR_OK;
  stride_coords_kernel<<<dgr_blocks(n * ncols, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      coords, n, ncols, out_stride, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_bloom_build(const uint64_t* keys, int64_t cap, uint32_t* bloom, int64_t bloom_bits, void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(bloom_bits >= 32 && (bloom_bits & (bloom_bits - 1)) == 0, "bloom_bits must be a power of two");
  cudaStream_t st = (cudaStream_t)stream;
  DGR_CUDA_CHECK(cudaMemsetAsync(bloom, 0, bloom_bits / 8, st));
  bloom_build_kernel<<<dgr_blocks(cap, kThreads), kThreads, 0, st>>>(keys, cap, bloom, (uint64_t)bloom_bits - 1);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_kernel_map_table(const int32_t* out_coords, int64_t n_out, int32_t ncols,
                             const dgr_keyspec_t* spec, const uint64_t* in_keys,
                             const int32_t* in_vals, int64_t in_cap, const uint32_t* bloom,
                             int64_t bloom_bits, const int32_t* offsets, int32_t K, int32_t* nbr,
                             int32_t* block_cnt, void* stream) {
  DGR_ARG_CHECK(bloom == nullptr || (bloom_bits >= 32 && (bloom_bits & (bloom_bits - 1)) == 0),
                "bloom_bits must be a power of two");
  DGR_ARG_CHECK(in_cap > 0 && (in_cap & (in_cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(K >= 1, "K must be positive");
  if (block_cnt != nullptr)
    DGR_CUDA_CHECK(cudaMemsetAsync(block_cnt, 0, (size_t)dgr_kmap_ws_elems(K, n_out) * sizeof(int32_t),
                                   (cudaStream_t)stream));
  if (n_out == 0) return DGR_OK;
  dim3 grid(dgr_blocks(n_out, kThreads), (K + kKappaChunk - 1) / kKappaChunk);
  kernel_map_table_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(
      out_coords, n_out, ncols, spec, in_keys, in_vals, (uint64_t)in_cap - 1, bloom,
      bloom != nullptr ? (uint64_t)bloom_bits - 1 : 0, offsets, K, nbr, block_cnt,
      (int)dgr_blocks(n_out, kScanElems));
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int64_t dgr_kmap_ws_elems(int32_t K, int64_t n_out) {
  int64_t bpk = (n_out + kScanElems - 1) / kScanElems;
  if (bpk < 1) bpk = 1;
  return (int64_t)K * bpk + 2;
}

int32_t dgr_kernel_map_count(const int32_t* nbr, int32_t K, int64_t n_out, int32_t* block_ws,
                             int32_t counts_ready, int32_t* kofs, const dgr_keyspec_t* spec, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned bpk = dgr_blocks(n_out, kScanElems);
  DGR_ARG_CHECK(K <= 65535, "K too large");
  if (!counts_ready) block_count_kernel<true><<<dim3(bpk, K), kThreads, 0, st>>>(nbr, n_out, block_ws);
  scan_blocks_kernel<<<1, 1024, 0, st>>>(block_ws, (int64_t)K * bpk, kofs, K, (int)bpk, spec);
  dgr_note_launches(counts_ready ? 1 : 2);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_kernel_map_fill(const int32_t* nbr, int32_t K, int64_t n_out, const int32_t* block_ws,
                            int32_t* in_idx, int32_t* out_idx, void* stream) {
  const unsigned bpk = dgr_blocks(n_out, kScanElems);
  kernel_map_fill_kernel<<<dim3(bpk, K), kThreads, 0, (cudaStream_t)stream>>>(nbr, n_out, block_ws,
                                                                            in_idx, out_idx);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// Both work lists of a kernel map (plain, and with an even tile count per offset) in one launch.
int32_t dgr_kernel_map_tiles2(const int32_t* kofs, int32_t K, int32_t tile_rows, int32_t n_tiles, int32_t n_tiles_paired,
                              int32_t* tile_k, int32_t* tile_start, int32_t* ptile_k, int32_t* ptile_start, void* stream) {
  DGR_ARG_CHECK(tile_rows >= 1, "tile_rows must be positive");
  if (n_tiles == 0 && n_tiles_paired == 0) return DGR_OK;
  tiles_kernel<<<2, 1024, (K + 1) * sizeof(int), (cudaStream_t)stream>>>(kofs, K, tile_rows, n_tiles, 0, tile_k, tile_start,
                                                                        n_tiles_paired, ptile_k, ptile_start);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_kernel_map_tiles(const int32_t* kofs, int32_t K, int32_t tile_rows, int32_t n_tiles, int32_t pair,
                             int32_t* tile_k, int32_t* tile_start, void* stream) {
  DGR_ARG_CHECK(tile_rows >= 1, "tile_rows must be positive");
  if (n_tiles == 0) return DGR_OK;
  tiles_kernel<<<1, 1024, (K + 1) * sizeof(int), (cudaStream_t)stream>>>(kofs, K, tile_rows, n_tiles, pair,
                                                                        tile_k, tile_start);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
