// Integer coordinate work of the sparse-tensor engine: voxelisation, coordinate hash,
// first-occurrence dedup.  All of it is HBM/L2-bound integer work: coalesced row-major
// loads, 64-bit packed keys so one probe is one 8-byte access, open-addressing tables
// sized to a load factor <= 0.5 that stay L2-resident (a 76k-voxel cloud is a 2 MB table).
// Strided maps and kernel maps are built in coordplan.cu.
//
// Replaces the MinkowskiEngine pieces reached from core/deep_global_registration.py:152-167
// (sparse_quantize, batched_coordinates, SparseTensor coordinate map).
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

// per-2048-row block count of flag > 0
__global__ void block_count_kernel(const int32_t* __restrict__ flag, int64_t n, int32_t* block_cnt) {
  const int64_t start = (int64_t)blockIdx.x * kScanElems;
  int c = 0;
#pragma unroll
  for (int e = 0; e < kScanElems / kThreads; ++e) {
    int64_t i = start + e * kThreads + threadIdx.x;
    if (i < n) c += flag[i] > 0;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  __shared__ int ws[kThreads / 32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += ws[w];
    block_cnt[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(1024) scan_counts_kernel(int32_t* cnt, int64_t nb) {
  const int total = dgr_block_scan_inplace(cnt, nb);
  if (threadIdx.x == 0) cnt[nb] = total;
}

__global__ void __launch_bounds__(256)
select_first_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ blk, int64_t n, int64_t cap,
                    int64_t h0, int32_t* __restrict__ sel, const int32_t* __restrict__ live) {
  if (live != nullptr && *live == 0) return;            // uniform per launch
  const int base = blk[blockIdx.x];
  if (base >= cap) return;                              // uniform per block
  const int64_t h = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int f = h < n ? flag[h] : 0;
  const int pos = base + dgr_block_exclusive_scan<256>(f, nullptr);
  if (f && pos < cap) sel[pos] = (int32_t)(h0 + h);
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
  int pos = block_ofs[blockIdx.x] + dgr_block_exclusive_scan<kThreads>(c, nullptr);
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

}  // namespace

void dgr_scan_counts(int32_t* cnt, int64_t nb, cudaStream_t st) { scan_counts_kernel<<<1, 1024, 0, st>>>(cnt, nb); }

void dgr_select_first(const int32_t* flag, const int32_t* blk, int64_t n, int64_t cap, int64_t h0, int32_t* sel,
                      const int32_t* live, cudaStream_t st) {
  select_first_kernel<<<dgr_blocks(n, 256), 256, 0, st>>>(flag, blk, n, cap, h0, sel, live);
}

// =========================================================================================
// C ABI
// =========================================================================================
extern "C" {

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
  block_count_kernel<<<nb, kThreads, 0, st>>>(rank_ws, n, scan_ws);
  dgr_scan_counts(scan_ws, nb, st);
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

}  // extern "C"
