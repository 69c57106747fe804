// Integer coordinate work of the sparse-tensor engine: voxelisation, coordinate hash and the
// first-occurrence pass behind unique rows, tables of distinct rows and coarse (strided) maps.
// All of it is HBM/L2-bound integer work: coalesced row-major loads, 64-bit packed keys so one
// probe is one 8-byte access, open-addressing tables sized to a load factor <= 0.5 that stay
// L2-resident (a 76k-voxel cloud is a 2 MB table).  Kernel maps are built in coordplan.cu.
//
// Replaces the MinkowskiEngine pieces reached from core/deep_global_registration.py:152-167
// (sparse_quantize, batched_coordinates, SparseTensor coordinate map).
#include <limits.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kScanElems = 2048;   // rows per block of the winner counts (256 threads x 8)
constexpr int kMaxLevels = 4;      // strides per first-occurrence pass

// ---------------------------------------------------------------------------------------
// voxelisation
// ---------------------------------------------------------------------------------------
// The cell of quotient q.  A float-to-int conversion of NaN is no cell at all, so a non-finite q (NaN or infinite
// input, or a division that overflows) goes to INT_MIN explicitly: below INT_MIN + the key margin, where
// keyspec_kernel sets the overflow flag and the cloud is refused, whichever point of its voxel comes first.  A finite
// q out of range saturates and is refused the same way.
template <typename T>
__device__ __forceinline__ int32_t cell_of(T q) {
  return isfinite(q) ? (int32_t)floor(q) : INT_MIN;
}

template <typename T>
__global__ void quantize_kernel(const T* __restrict__ xyz, int64_t n, T voxel, int32_t batch,
                                int32_t* __restrict__ coords) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  // true IEEE division in the input dtype, then floor (numpy: np.floor(xyz / voxel))
  T x = xyz[3 * r + 0] / voxel, y = xyz[3 * r + 1] / voxel, z = xyz[3 * r + 2] / voxel;
  int4 c;
  c.x = batch;
  c.y = cell_of(x);
  c.z = cell_of(y);
  c.w = cell_of(z);
  reinterpret_cast<int4*>(coords)[r] = c;
}

template <typename T>
__global__ void float32_in_cells_kernel(const T* __restrict__ xyz, int64_t n, const int32_t* __restrict__ cells,
                                        int64_t cells_stride, double cell, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * n) return;
  const int64_t r = i / 3;
  out[i] = dgr_float32_in_cell((double)xyz[i], cells[r * cells_stride + (i - 3 * r)], cell);
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
// first-occurrence pass: clear, insert, flag + count, scan, scatter (+ inverse)
// Keeps the first row of every distinct key and ranks the kept rows in row order, for up to
// kMaxLevels strides of the same rows at once (levels on blockIdx.y).  Level l keys a row
// floored to stride[l] on the spatial columns.  Row counts follow coordplan.cu: n_max bounds
// buffers and grids, n_dev (NULL: n_max) holds the actual count.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int floor_to(int v, int stride) {
  int q = v / stride;
  if ((v % stride != 0) && (v < 0)) --q;
  return q * stride;
}

// key of a row floored to `stride` on the spatial columns (column 0 = batch is kept); dgr_pack_key at stride 1
__device__ __forceinline__ uint64_t pack_key_strided(const int32_t* __restrict__ row, const dgr_keyspec_t& s,
                                                     int stride) {
  uint64_t k = 0;
#pragma unroll
  for (int i = 0; i < DGR_MAX_COLS; ++i)
    if (i < s.ncols) {
      const int v = (i == 0 || stride == 1) ? row[i] : floor_to(row[i], stride);
      k += (uint64_t)(uint32_t)(v - s.lo[i]) << s.shift[i];
    }
  return k;
}

struct Levels {
  int stride[kMaxLevels];
  uint64_t* keys[kMaxLevels];
  int32_t* vals[kMaxLevels];
  int32_t* slot[kMaxLevels];     // row -> table slot, ~slot once the row is known not to be first (NULL: not kept)
  int32_t* scan[kMaxLevels];     // winners per kScanElems-row block, then their exclusive scan
  int32_t* sel[kMaxLevels];      // optional: sel[rank] = row
  int32_t* coords[kMaxLevels];   // optional: coords[rank] = the floored row
};

__global__ void table_clear_kernel(uint64_t* keys, int32_t* vals, int64_t total) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) {
    keys[i] = DGR_EMPTY_KEY;
    vals[i] = INT_MAX;
  }
}

// insert every row; the table value converges to the smallest row of each key
__global__ void insert_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ n_dev, int64_t n_max,
                              int ncols, const dgr_keyspec_t* __restrict__ spec_p, uint64_t mask, Levels a) {
  const int n = dgr_dev_count(n_dev, n_max);
  const int l = blockIdx.y;
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const dgr_keyspec_t s = *spec_p;
  const uint32_t sl = dgr_hash_insert(a.keys[l], mask, pack_key_strided(rows + r * ncols, s, a.stride[l]));
  atomicMin(a.vals[l] + sl, (int32_t)r);
  if (a.slot[l] != nullptr) a.slot[l][r] = (int32_t)sl;
}

// winners (the first row of every key) keep slot >= 0, losers get ~slot; per-block winner counts go to scan[l]
__global__ void flag_kernel(const int32_t* __restrict__ n_dev, int64_t n_max, Levels a) {
  const int n = dgr_dev_count(n_dev, n_max);
  const int l = blockIdx.y;
  const int64_t start = (int64_t)blockIdx.x * kScanElems;
  int c = 0;
#pragma unroll
  for (int e = 0; e < kScanElems / kThreads; ++e) {
    const int64_t r = start + e * kThreads + threadIdx.x;
    if (r < n) {
      const int sl = a.slot[l][r];
      const bool win = a.vals[l][sl] == (int32_t)r;
      if (!win) a.slot[l][r] = ~sl;
      c += win;
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
    a.scan[l][blockIdx.x] = t;
  }
}

// Exclusive scan in place of the nb counts of level blockIdx.y (cnt + blockIdx.y * level_stride) with one block;
// the total goes to cnt[nb] and, when `total` is set, to total[blockIdx.y].  Blocks past a device row count hold
// zero counts, so scanning the nb of n_max gives the offsets and total of the actual rows.
__global__ void __launch_bounds__(1024) scan_counts_kernel(int32_t* cnt, int64_t nb, int64_t level_stride,
                                                           int32_t* total) {
  cnt += blockIdx.y * level_stride;
  const int t = dgr_block_scan_inplace(cnt, nb);
  if (threadIdx.x == 0) {
    cnt[nb] = t;
    if (total != nullptr) total[blockIdx.y] = t;
  }
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

// rank the winners in row order: table value <- rank, sel[rank] = row, coords[rank] = the floored row
__global__ void scatter_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ n_dev, int64_t n_max,
                               int ncols, Levels a) {
  const int n = dgr_dev_count(n_dev, n_max);
  const int l = blockIdx.y;
  const int64_t start = (int64_t)blockIdx.x * kScanElems + (int64_t)threadIdx.x * 8;
  if ((int64_t)blockIdx.x * kScanElems >= n) return;      // uniform per block
  int sl[8], c = 0;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int64_t r = start + e;
    sl[e] = (r < n) ? a.slot[l][r] : -1;
    c += (sl[e] >= 0);
  }
  int pos = a.scan[l][blockIdx.x] + dgr_block_exclusive_scan<kThreads>(c, nullptr);
  const int stride = a.stride[l];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (sl[e] >= 0) {
      const int64_t r = start + e;
      if (a.sel[l] != nullptr) a.sel[l][pos] = (int32_t)r;
      if (a.coords[l] != nullptr) {
        int32_t* dst = a.coords[l] + (int64_t)pos * ncols;
        dst[0] = rows[r * ncols];
        for (int col = 1; col < ncols; ++col) dst[col] = floor_to(rows[r * ncols + col], stride);
      }
      a.vals[l][sl[e]] = pos;
      ++pos;
    }
  }
}

// inverse[r] = rank of the first row of r's key; the key-overflow flag goes beside the count in n_unique, so one host
// read returns both
__global__ void inverse_kernel(const int32_t* __restrict__ slot, const int32_t* __restrict__ vals, int64_t n,
                               const dgr_keyspec_t* __restrict__ spec, int32_t* __restrict__ inverse,
                               int32_t* __restrict__ n_unique) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) n_unique[1] = spec->overflow;
  if (r < n) {
    const int sl = slot[r];
    inverse[r] = vals[sl >= 0 ? sl : ~sl];
  }
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

// The first-occurrence pass over rows [n_max, ncols] at n_levels strides, after the tables were cleared: level l's
// table (keys / vals + l * cap) ends up mapping each floored key to the rank of its first row, n_out[l] holds the
// number of keys, and sel + l * nmx / coords + l * nmx * ncols (each optional) the first rows by rank, with
// nmx = max(n_max, 1).  slot_ws: n_levels * nmx ints; scan_ws: n_levels * dgr_scan_ws_elems(nmx) ints.  Four launches.
void first_occurrence(const int32_t* rows, int64_t n_max, const int32_t* n_dev, int ncols, const dgr_keyspec_t* spec,
                      int n_levels, const int32_t* strides, uint64_t* keys, int32_t* vals, int64_t cap, int32_t* sel,
                      int32_t* coords, int32_t* n_out, int32_t* slot_ws, int32_t* scan_ws, cudaStream_t st) {
  const int64_t nmx = n_max > 0 ? n_max : 1, scan_elems = dgr_scan_ws_elems(nmx);
  Levels a{};
  for (int l = 0; l < n_levels; ++l) {
    a.stride[l] = strides[l];
    a.keys[l] = keys + l * cap;
    a.vals[l] = vals + l * cap;
    a.slot[l] = slot_ws + l * nmx;
    a.scan[l] = scan_ws + l * scan_elems;
    a.sel[l] = sel != nullptr ? sel + l * nmx : nullptr;
    a.coords[l] = coords != nullptr ? coords + l * nmx * ncols : nullptr;
  }
  const unsigned nb = dgr_blocks(nmx, kScanElems);
  insert_kernel<<<dim3(dgr_blocks(nmx, kThreads), n_levels), kThreads, 0, st>>>(rows, n_dev, n_max, ncols, spec,
                                                                               (uint64_t)cap - 1, a);
  flag_kernel<<<dim3(nb, n_levels), kThreads, 0, st>>>(n_dev, n_max, a);
  scan_counts_kernel<<<dim3(1, n_levels), 1024, 0, st>>>(scan_ws, nb, scan_elems, n_out);
  scatter_kernel<<<dim3(nb, n_levels), kThreads, 0, st>>>(rows, n_dev, n_max, ncols, a);
  dgr_note_launches(4);
}

}  // namespace

void dgr_scan_counts(int32_t* cnt, int64_t nb, cudaStream_t st) {
  scan_counts_kernel<<<1, 1024, 0, st>>>(cnt, nb, 0, nullptr);
}

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

int32_t dgr_float32_in_cells(const void* xyz, int32_t is_f64, int64_t n, const int32_t* cells, int64_t cells_stride,
                             double cell, float* out, void* stream) {
  DGR_ARG_CHECK(cell > 0 && cell < INFINITY, "cell must be positive and finite");
  DGR_ARG_CHECK(n >= 0 && n < (1ll << 40), "row count out of range");
  if (n == 0) return DGR_OK;
  DGR_ARG_CHECK(xyz != nullptr && cells != nullptr && out != nullptr, "null argument");
  DGR_ARG_CHECK(cells_stride >= 3, "cells rows must hold at least 3 ints");
  const unsigned blocks = dgr_blocks(3 * n, kThreads);
  cudaStream_t st = (cudaStream_t)stream;
  if (is_f64)
    float32_in_cells_kernel<double><<<blocks, kThreads, 0, st>>>((const double*)xyz, n, cells, cells_stride, cell, out);
  else
    float32_in_cells_kernel<float><<<blocks, kThreads, 0, st>>>((const float*)xyz, n, cells, cells_stride, cell, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
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
  table_clear_kernel<<<dgr_blocks(cap, kThreads), kThreads, 0, (cudaStream_t)stream>>>(keys, vals, cap);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int64_t dgr_scan_ws_elems(int64_t n) { return (n + kScanElems - 1) / kScanElems + 2; }

int32_t dgr_unique_first(const int32_t* coords, int64_t n, int32_t ncols, const dgr_keyspec_t* spec,
                         uint64_t* keys, int32_t* vals, int64_t cap, int32_t* sel, int32_t* inverse,
                         int32_t* n_unique, int32_t* slot_ws, int32_t* scan_ws, void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(cap >= 2 * n || n == 0, "capacity must be at least 2n");
  DGR_ARG_CHECK(n < (int64_t)INT_MAX, "too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    DGR_CUDA_CHECK(cudaMemsetAsync(n_unique, 0, 2 * sizeof(int32_t), st));
    return DGR_OK;
  }
  const int32_t stride1 = 1;
  first_occurrence(coords, n, nullptr, ncols, spec, 1, &stride1, keys, vals, cap, sel, nullptr, n_unique, slot_ws,
                   scan_ws, st);
  inverse_kernel<<<dgr_blocks(n, kThreads), kThreads, 0, st>>>(slot_ws, vals, n, spec, inverse, n_unique);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_table_build_unique(const int32_t* coords, int64_t n_max, const int32_t* n_dev, int32_t ncols,
                               const dgr_keyspec_t* spec, uint64_t* keys, int32_t* vals, int64_t cap,
                               void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(cap >= 2 * n_max, "capacity must be at least 2 n_max");
  cudaStream_t st = (cudaStream_t)stream;
  table_clear_kernel<<<dgr_blocks(cap, kThreads), kThreads, 0, st>>>(keys, vals, cap);
  if (n_max > 0) {
    Levels a{};                  // one level at stride 1, no slots: distinct rows are all first
    a.stride[0] = 1;
    a.keys[0] = keys;
    a.vals[0] = vals;
    insert_kernel<<<dgr_blocks(n_max, kThreads), kThreads, 0, st>>>(coords, n_dev, n_max, ncols, spec,
                                                                     (uint64_t)cap - 1, a);
  }
  dgr_note_launches(n_max > 0 ? 2 : 1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_coarse_maps(const int32_t* fine, int64_t n_max, const int32_t* n_dev, int32_t ncols,
                        const dgr_keyspec_t* spec, int32_t n_levels, const int32_t* strides, uint64_t* keys,
                        int32_t* vals, int64_t cap, int32_t* coords_out, int32_t* n_out, int32_t* slot_ws,
                        int32_t* scan_ws, void* stream) {
  DGR_ARG_CHECK(n_levels >= 1 && n_levels <= kMaxLevels, "1..4 levels per call");
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0 && cap >= 2 * n_max, "capacity: power of two >= 2 n_max");
  for (int l = 0; l < n_levels; ++l) DGR_ARG_CHECK(strides[l] >= 1, "stride must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  table_clear_kernel<<<dgr_blocks(cap * n_levels, kThreads), kThreads, 0, st>>>(keys, vals, cap * n_levels);
  first_occurrence(fine, n_max, n_dev, ncols, spec, n_levels, strides, keys, vals, cap, nullptr, coords_out, n_out,
                   slot_ws, scan_ws, st);
  dgr_note_launches(1);
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
