// Exact feature nearest neighbour with a tensor-core pre-filter (C % 32 == 0).
//
// The fp32 brute-force kernel (knn.cu) spends 2 instructions per (i, j, c) term on the fp32
// pipe.  Here the same answer - bit-identical indices - is produced in two wgmma sweeps:
//
//   pass 1  D = F0_tile . F1_tile^T on the tensor cores (TF32, fp32 accumulator in registers);
//           the epilogue (each thread holds two F0 rows, two columns of every 8-column group) forms
//           d~2 = |a|^2 + |b|^2 - 2 D and keeps the row minimum m~_i;
//   pass 2  the same products again; every column with d~2 <= m~_i + 2 E_i is a CANDIDATE and
//           only candidates are evaluated with the reference arithmetic
//           (fp32 sum_c (a - b)^2 in ascending c, sqrt(d2 + 1e-7), lowest index on ties) - the
//           very code of the fp32 kernel.
//
// E_i bounds the error of d~2: operands are rounded to TF32 (relative 2^-11 each), so a dot
// product is off by at most 2^-10 |a||b| (+ accumulation slack), and d~2 by twice that.  The
// true nearest neighbour j* satisfies d~2(j*) <= d2(j*) + E <= d2(j) + E <= d~2(j) + 2E for
// every j, hence it is always among the candidates and the result equals the fp32 kernel's.
#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int kThreadsK = 256;        // two warpgroups: F0 rows 0..63 and 64..127 of the tile
constexpr int kRowsA = 128;
constexpr int kColsB = 128;
constexpr int kATile = kRowsA * 128;    // bytes per 32-float chunk
constexpr int kBTile = kColsB * 128;

__global__ void row_norms_kernel(const float* __restrict__ f, int64_t n, int c, float* __restrict__ n2,
                                 unsigned* __restrict__ max_bits) {
  int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;   // 8 lanes per row
  int sub = threadIdx.x & 7;
  float s = 0.f;
  if (row < n)
    for (int k = sub; k < c; k += 8) {
      float v = f[row * c + k];
      s = fmaf(v, v, s);
    }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (row < n && sub == 0) {
    n2[row] = s;
    if (max_bits != nullptr) atomicMax(max_bits, __float_as_uint(s));
  }
}

__global__ void knn_tc_init_kernel(unsigned* __restrict__ rowmin_bits, unsigned long long* __restrict__ packed,
                                   int64_t n0, unsigned* max_bits) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n0) {
    rowmin_bits[i] = 0x7f800000u;
    packed[i] = ~0ull;
  }
  if (i == 0) *max_bits = 0u;
}

// thr_i = m~_i + 2 E_i with E_i = 2 * (dot-product error bound): operands rounded to TF32,
// |a.b error| <= 2^-10 * 1.25 |a||b| (+ accumulation slack), plus the slack of the fp32 norms.
__device__ __forceinline__ float knn_error_bound(float na, float nb) {
  return (0.0009765625f * 1.25f + 4e-5f) * na * nb + 1e-6f * (na + nb) * (na + nb) + 1e-7f;
}
__global__ void knn_tc_threshold_kernel(const unsigned* __restrict__ rowmin_bits, const float* __restrict__ na2,
                                        const unsigned* __restrict__ nb2_max_bits, int64_t n0,
                                        float* __restrict__ thr) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n0) return;
  const float na = sqrtf(na2[i]), nb = sqrtf(__uint_as_float(*nb2_max_bits));
  const float e = knn_error_bound(na, nb);
  // stored in the epilogue's units: candidates satisfy (0.5 |b|^2 - a.b) <= thr'
  thr[i] = 0.5f * (__uint_as_float(rowmin_bits[i]) + 4.f * e - na2[i]);
}

__device__ __forceinline__ void round_store(float4 v, unsigned char* tile, int row, int piece) {
  float4 h;
  h.x = tf32_round(v.x); h.y = tf32_round(v.y); h.z = tf32_round(v.z); h.w = tf32_round(v.w);
  *reinterpret_cast<float4*>(tile + row * 128 + ((piece ^ (row & 7)) << 4)) = h;
}

// exact reference arithmetic for one candidate column, as in knn.cu
template <int C>
__device__ __noinline__ void knn_exact_candidate(const float* __restrict__ f0, const float* __restrict__ f1,
                                                 int gi, int j, float& best_s, float& best_d2, int& best_j) {
  const float4* a = reinterpret_cast<const float4*>(f0 + (size_t)gi * C);
  const float4* b = reinterpret_cast<const float4*>(f1 + (size_t)j * C);
  float d2 = 0.f;
#pragma unroll
  for (int k = 0; k < C / 4; ++k) {
    const float4 x = __ldg(a + k), y = __ldg(b + k);
    float df = x.x - y.x; d2 = fmaf(df, df, d2);
    df = x.y - y.y; d2 = fmaf(df, df, d2);
    df = x.z - y.z; d2 = fmaf(df, df, d2);
    df = x.w - y.w; d2 = fmaf(df, df, d2);
  }
  if (d2 < best_d2) {
    const float sq = sqrtf(d2 + 1e-7f);
    if (sq < best_s) {
      best_s = sq;
      best_d2 = d2;
      best_j = j;
    }
  }
}

template <int C, int PASS>
__global__ void __launch_bounds__(kThreadsK)
knn_tc_kernel(const float* __restrict__ f0, int n0, const float* __restrict__ f1, int n1,
              const float* __restrict__ na2, const float* __restrict__ nb2, int cols_per_split,
              unsigned* __restrict__ rowmin_bits, const float* __restrict__ thr,
              unsigned long long* __restrict__ packed, const unsigned* __restrict__ nb2_max_bits) {
  constexpr int kChunks = C / 32;
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  float* nb_sh = reinterpret_cast<float*>(smem_dyn);          // 0.5 |b|^2 of the tile's columns
  unsigned char* a_tile = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_dyn) + kColsB * sizeof(float) + 1023) & ~(uintptr_t)1023);
  unsigned char* b_tile = a_tile + kChunks * kATile;
  const int t = threadIdx.x, wg = t >> 7, lane = t & 31;
  const int row0 = blockIdx.x * kRowsA;
  const int col_begin = blockIdx.y * cols_per_split;
  const int col_end = min(n1, col_begin + cols_per_split);
  const int n_tiles = (col_end - col_begin + kColsB - 1) / kColsB;
  const int piece = t & 7, rgrp = t >> 3;   // 8 lanes per 128-byte row, 32 row groups

  // the F0 tile, once
#pragma unroll
  for (int ch = 0; ch < kChunks; ++ch)
#pragma unroll
    for (int i = 0; i < kRowsA / 32; ++i) {
      const int r = i * 32 + rgrp;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row0 + r < n0) v = __ldg(reinterpret_cast<const float4*>(f0 + (size_t)(row0 + r) * C + ch * 32 + piece * 4));
      round_store(v, a_tile + ch * kATile, r, piece);
    }
  float4 bv[kChunks][kColsB / 32];
  float nbv = 0.f;
  auto load_b = [&](int it) {
    const int j0 = col_begin + it * kColsB;
#pragma unroll
    for (int ch = 0; ch < kChunks; ++ch)
#pragma unroll
      for (int i = 0; i < kColsB / 32; ++i) {
        const int r = i * 32 + rgrp;
        bv[ch][i] = (j0 + r < col_end)
                        ? __ldg(reinterpret_cast<const float4*>(f1 + (size_t)(j0 + r) * C + ch * 32 + piece * 4))
                        : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    if (t < kColsB) nbv = (j0 + t < col_end) ? nb2[j0 + t] : 0.f;
  };

  // epilogue state: this thread's rows r and r + 8 (h = 0, 1) of its warpgroup
  const int r = wg * 64 + ((t >> 5) & 3) * 16 + (lane >> 2);
  int gi[2];
  bool valid[2];
  float th[2], na2_i[2], e4[2], rmin[2], best_s[2], best_d2[2];
  int best_j[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    gi[h] = row0 + r + 8 * h;
    valid[h] = gi[h] < n0;
    // pass 2 tightens its bound with every exact distance it learns: a later column can only win if its true
    // d2 is below the best exact d2 so far, i.e. if its estimate is below best_d2 + (estimate error)
    th[h] = (PASS == 2 && valid[h]) ? thr[gi[h]] : -__int_as_float(0x7f800000);
    na2_i[h] = (PASS == 2 && valid[h]) ? na2[gi[h]] : 0.f;
    e4[h] = (PASS == 2 && valid[h])
                ? 4.f * knn_error_bound(sqrtf(na2_i[h]), sqrtf(__uint_as_float(*nb2_max_bits)))
                : 0.f;
    rmin[h] = __int_as_float(0x7f800000);     // min over columns of 0.5 |b|^2 - a.b
    best_s[h] = best_d2[h] = __int_as_float(0x7f800000);
    best_j[h] = 0x7fffffff;
  }

  load_b(0);
  for (int it = 0; it < n_tiles; ++it) {
    __syncthreads();     // every thread is done with the previous tile's operands and norms
#pragma unroll
    for (int ch = 0; ch < kChunks; ++ch)
#pragma unroll
      for (int i = 0; i < kColsB / 32; ++i) round_store(bv[ch][i], b_tile + ch * kBTile, i * 32 + rgrp, piece);
    if (t < kColsB) nb_sh[t] = 0.5f * nbv;          // the epilogue works with 0.5 |b|^2 - a.b
    if (it + 1 < n_tiles) load_b(it + 1);           // in flight during the MMAs and the epilogue
    fence_proxy_async();
    __syncthreads();
    float acc[kColsB / 2];
#pragma unroll
    for (int i = 0; i < kColsB / 2; ++i) acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ch = 0; ch < kChunks; ++ch) {
      const uint32_t a = smem_u32(a_tile + ch * kATile) + wg * (kATile / 2), b = smem_u32(b_tile + ch * kBTile);
      mma_chunk<kColsB, false, 1>(acc, a, a, b, b);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(acc);
    // columns in ascending order per row: the exact evaluation keeps the lowest index on ties
    const int j0 = col_begin + it * kColsB;
#pragma unroll
    for (int i = 0; i < kColsB / 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * i + 2 * (lane & 3) + e;
        const int jc = j0 + col;
        if (jc < col_end) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float g = nb_sh[col] - acc[4 * i + 2 * h + e];
            if (PASS == 1) {
              rmin[h] = fminf(rmin[h], g);
            } else if (g <= th[h]) {
              knn_exact_candidate<C>(f0, f1, gi[h], jc, best_s[h], best_d2[h], best_j[h]);
              th[h] = fminf(th[h], 0.5f * (best_d2[h] + e4[h] - na2_i[h]));
            }
          }
        }
      }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (PASS == 1) {
      // the four lanes of a quad share the row
      rmin[h] = fminf(rmin[h], __shfl_xor_sync(0xffffffffu, rmin[h], 1));
      rmin[h] = fminf(rmin[h], __shfl_xor_sync(0xffffffffu, rmin[h], 2));
      if (valid[h] && (lane & 3) == 0)
        atomicMin(rowmin_bits + gi[h], __float_as_uint(fmaxf(fmaf(2.f, rmin[h], na2[gi[h]]), 0.f)));
    } else if (valid[h] && best_j[h] != 0x7fffffff) {
      atomicMin(packed + gi[h], ((unsigned long long)__float_as_uint(best_s[h]) << 32) | (unsigned)best_j[h]);
    }
  }
}

__global__ void knn_tc_unpack_kernel(const unsigned long long* __restrict__ packed, int64_t n,
                                     int32_t* __restrict__ idx, float* __restrict__ dist) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long p = packed[i];
  idx[i] = (int32_t)(p & 0xffffffffu);
  if (dist != nullptr) dist[i] = __uint_as_float((unsigned)(p >> 32));
}

template <int C>
int32_t launch_knn_tc(const float* f0, int64_t n0, const float* f1, int64_t n1, float* na2, float* nb2,
                      unsigned* rowmin, float* thr, unsigned* max_bits, unsigned long long* packed,
                      cudaStream_t st) {
  constexpr int kChunks = C / 32;
  const size_t smem = kColsB * sizeof(float) + 1024 + (size_t)kChunks * (kATile + kBTile);
  DGR_ENSURE_SMEM((knn_tc_kernel<C, 1>), smem);
  DGR_ENSURE_SMEM((knn_tc_kernel<C, 2>), smem);
  int dev = 0, sms = 0;
  DGR_CUDA_CHECK(cudaGetDevice(&dev));
  DGR_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  // split the columns so that the grid fills every SM a few times over
  const int row_tiles = (int)((n0 + kRowsA - 1) / kRowsA);
  const int col_tiles = (int)((n1 + kColsB - 1) / kColsB);
  int splits = (sms * 4 + row_tiles - 1) / row_tiles;
  if (splits > col_tiles) splits = col_tiles;
  if (splits < 1) splits = 1;
  const int cols_per_split = ((col_tiles + splits - 1) / splits) * kColsB;
  splits = (int)((n1 + cols_per_split - 1) / cols_per_split);
  dim3 grid(row_tiles, splits);
  knn_tc_kernel<C, 1><<<grid, kThreadsK, smem, st>>>(f0, (int)n0, f1, (int)n1, na2, nb2, cols_per_split, rowmin, thr,
                                                     packed, max_bits);
  knn_tc_threshold_kernel<<<dgr_blocks(n0, 256), 256, 0, st>>>(rowmin, na2, max_bits, n0, thr);
  knn_tc_kernel<C, 2><<<grid, kThreadsK, smem, st>>>(f0, (int)n0, f1, (int)n1, na2, nb2, cols_per_split, rowmin, thr,
                                                     packed, max_bits);
  return DGR_OK;
}

}  // namespace

extern "C" {

// floats of workspace dgr_knn_top1_tc needs
int64_t dgr_knn_tc_ws_elems(int64_t n0, int64_t n1) { return 3 * n0 + n1 + 8; }

// 1 if the tensor-core pre-filter supports the channel count
int32_t dgr_knn_tc_supported(int32_t c) { return (c == 32 || c == 64) ? 1 : 0; }

// Same result as dgr_knn_top1 (bit-identical indices and distances), two wgmma sweeps
// plus exact fp32 evaluation of the few candidates per row.  ws: dgr_knn_tc_ws_elems floats.
int32_t dgr_knn_top1_tc(const float* f0, int64_t n0, const float* f1, int64_t n1, int32_t c,
                        uint64_t* packed_ws, float* ws, int32_t* idx, float* dist, void* stream) {
  DGR_ARG_CHECK(dgr_knn_tc_supported(c), "channel count not supported by the tensor-core kNN");
  DGR_ARG_CHECK(n1 >= 1 || n0 == 0, "F1 must not be empty");
  DGR_ARG_CHECK(n0 < (1ll << 31) && n1 < (1ll << 31), "too many rows");
  if (n0 == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  float* na2 = ws;
  float* thr = ws + n0;
  unsigned* rowmin = reinterpret_cast<unsigned*>(ws + 2 * n0);
  float* nb2 = ws + 3 * n0;
  unsigned* max_bits = reinterpret_cast<unsigned*>(ws + 3 * n0 + n1);
  unsigned long long* packed = reinterpret_cast<unsigned long long*>(packed_ws);
  knn_tc_init_kernel<<<dgr_blocks(n0, 256), 256, 0, st>>>(rowmin, packed, n0, max_bits);
  row_norms_kernel<<<dgr_blocks(n0 * 8, 256), 256, 0, st>>>(f0, n0, c, na2, nullptr);
  row_norms_kernel<<<dgr_blocks(n1 * 8, 256), 256, 0, st>>>(f1, n1, c, nb2, max_bits);
  int32_t rc = (c == 32) ? launch_knn_tc<32>(f0, n0, f1, n1, na2, nb2, rowmin, thr, max_bits, packed, st)
                         : launch_knn_tc<64>(f0, n0, f1, n1, na2, nb2, rowmin, thr, max_bits, packed, st);
  if (rc != DGR_OK) return rc;
  knn_tc_unpack_kernel<<<dgr_blocks(n0, 256), 256, 0, st>>>(packed, n0, idx, dist);
  dgr_note_launches(7);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
