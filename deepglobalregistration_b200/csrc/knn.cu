// Feature-space nearest neighbour (k = 1): replaces find_knn_gpu (core/knn.py:23-74)
// and its pdist temporary (core/metrics.py:62-65).
//
// Tiled brute force in fp32: a CTA holds a 128-row tile of F0 and a 128-row tile of F1
// in shared memory; every thread owns an 8x8 block of the distance tile in registers
// and accumulates sum_c (a-b)^2 with one FADD + one FFMA per term - the same direct
// difference form as the reference (no ||a||^2+||b||^2-2ab cancellation), so near-ties
// resolve the same way.  Nothing of the [N0, N1] distance matrix ever reaches HBM: the
// compulsory traffic is (N0 + N1) * C * 4 bytes, the kernel is bound by the fp32 pipe.
//
// Reference tie semantics: the compared quantity is sqrt(d2 + 1e-7) in fp32 (distinct d2
// can collapse to the same root) and torch.min returns the lowest index among equals.
// sqrt is monotone, so a candidate can only win if d2 < best_d2; only then is the exact
// root evaluated.  The row result is the lexicographic minimum of (root, index), merged
// across column splits with one 64-bit atomicMin on (root_bits << 32 | index).
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kBM = 128;
constexpr int kBN = 128;

template <int C>
__global__ void __launch_bounds__(kThreads, 2)
knn_top1_kernel(const float* __restrict__ f0, int n0, const float* __restrict__ f1, int n1,
                int cols_per_split, unsigned long long* __restrict__ packed) {
  // A: [C][kBM] transposed; B: [kBN][C + 1] row-major padded
  extern __shared__ __align__(16) float knn_smem[];
  float* As = knn_smem;
  float* Bs = knn_smem + C * kBM;
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const int row0 = blockIdx.x * kBM;
  const int col_begin = blockIdx.y * cols_per_split;
  const int col_end = min(n1, col_begin + cols_per_split);

  for (int e = t; e < kBM * C; e += kThreads) {
    int r = e / C, c = e - r * C;
    As[c * kBM + r] = (row0 + r < n0) ? f0[(int64_t)(row0 + r) * C + c] : 0.f;
  }

  float best_s[8], best_d2[8];
  int best_j[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    best_s[i] = __int_as_float(0x7f800000);
    best_d2[i] = __int_as_float(0x7f800000);
    best_j[i] = 0x7fffffff;
  }

  for (int j0 = col_begin; j0 < col_end; j0 += kBN) {
    __syncthreads();
    for (int e = t; e < kBN * C; e += kThreads) {
      int r = e / C, c = e - r * C;
      Bs[r * (C + 1) + c] = (j0 + r < col_end) ? f1[(int64_t)(j0 + r) * C + c] : 0.f;
    }
    __syncthreads();
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
#pragma unroll 4
    for (int c = 0; c < C; ++c) {
      float4 a0 = *reinterpret_cast<const float4*>(As + c * kBM + ty * 8);
      float4 a1 = *reinterpret_cast<const float4*>(As + c * kBM + ty * 8 + 4);
      float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = Bs[(tx + 16 * j) * (C + 1) + c];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float d = a[i] - b[j];
          acc[i][j] = fmaf(d, d, acc[i][j]);
        }
    }
    // columns of this thread ascend with j, tiles ascend with j0: first minimum wins
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = j0 + tx + 16 * j;
      if (col < col_end) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (acc[i][j] < best_d2[i]) {
            float s = sqrtf(acc[i][j] + 1e-7f);
            if (s < best_s[i]) {
              best_s[i] = s;
              best_d2[i] = acc[i][j];
              best_j[i] = col;
            }
          }
        }
      }
    }
  }
  // merge the 16 threads (tx) that share a row: lexicographic (s, j) minimum
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    unsigned long long p =
        ((unsigned long long)__float_as_uint(best_s[i]) << 32) | (unsigned)best_j[i];
#pragma unroll
    for (int d = 8; d > 0; d >>= 1) {
      unsigned long long o = __shfl_xor_sync(0xffffffffu, p, d);
      p = o < p ? o : p;
    }
    const int row = row0 + ty * 8 + i;
    if (tx == 0 && row < n0) atomicMin(packed + row, p);
  }
}

// any channel count: one thread per (row, column-split) - correctness path for odd C
// live (optional): skip the launch's work when *live == 0
__global__ void knn_top1_generic_kernel(const float* __restrict__ f0, int n0,
                                        const float* __restrict__ f1, int n1, int c,
                                        unsigned long long* __restrict__ packed, const int32_t* __restrict__ live) {
  if (live != nullptr && *live == 0) return;            // uniform per launch
  int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n0) return;
  float best_s = __int_as_float(0x7f800000), best_d2 = best_s;
  int best_j = 0x7fffffff;
  for (int j = 0; j < n1; ++j) {
    float d2 = 0.f;
    for (int k = 0; k < c; ++k) {
      float d = f0[(int64_t)row * c + k] - f1[(int64_t)j * c + k];
      d2 = fmaf(d, d, d2);
    }
    if (d2 < best_d2) {
      float s = sqrtf(d2 + 1e-7f);
      if (s < best_s) { best_s = s; best_d2 = d2; best_j = j; }
    }
  }
  packed[row] = ((unsigned long long)__float_as_uint(best_s) << 32) | (unsigned)best_j;
}

__global__ void knn_init_kernel(unsigned long long* packed, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) packed[i] = ~0ull;
}

__global__ void knn_unpack_kernel(const unsigned long long* __restrict__ packed, int64_t n,
                                  int32_t* __restrict__ idx, float* __restrict__ dist) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long p = packed[i];
  idx[i] = (int32_t)(p & 0xffffffffu);
  if (dist != nullptr) dist[i] = __uint_as_float((unsigned)(p >> 32));
}

}  // namespace

void dgr_knn_top1_packed(const float* f0, int n0, const float* f1, int n1, int c, uint64_t* packed,
                         const int32_t* live, cudaStream_t st) {
  knn_top1_generic_kernel<<<dgr_blocks(n0, 128), 128, 0, st>>>(f0, n0, f1, n1, c,
                                                                reinterpret_cast<unsigned long long*>(packed), live);
}

extern "C" int32_t dgr_knn_top1(const float* f0, int64_t n0, const float* f1, int64_t n1, int32_t c,
                                uint64_t* packed_ws, int32_t* idx, float* dist, void* stream) {
  DGR_ARG_CHECK(n1 >= 1 || n0 == 0, "F1 must not be empty");
  DGR_ARG_CHECK(n0 < (1ll << 31) && n1 < (1ll << 31), "too many rows");
  if (n0 == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* packed = reinterpret_cast<unsigned long long*>(packed_ws);
  knn_init_kernel<<<dgr_blocks(n0, kThreads), kThreads, 0, st>>>(packed, n0);
  const int row_tiles = (int)((n0 + kBM - 1) / kBM);
  // split the columns so that the grid fills 132 SMs x 2 resident CTAs a few times over
  int splits = (132 * 2 * 2 + row_tiles - 1) / row_tiles;
  const int col_tiles = (int)((n1 + kBN - 1) / kBN);
  if (splits > col_tiles) splits = col_tiles;
  if (splits < 1) splits = 1;
  const int cols_per_split = ((col_tiles + splits - 1) / splits) * kBN;
  splits = (int)((n1 + cols_per_split - 1) / cols_per_split);
  dim3 grid(row_tiles, splits);
#define DGR_LAUNCH_KNN(CC)                                                                         \
  do {                                                                                             \
    const int smem = (CC * kBM + kBN * (CC + 1)) * (int)sizeof(float);                             \
    DGR_CUDA_CHECK(cudaFuncSetAttribute(knn_top1_kernel<CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
    knn_top1_kernel<CC><<<grid, kThreads, smem, st>>>(f0, (int)n0, f1, (int)n1, cols_per_split, packed); \
  } while (0)
  switch (c) {
    case 16: DGR_LAUNCH_KNN(16); break;
    case 32: DGR_LAUNCH_KNN(32); break;
    case 64: DGR_LAUNCH_KNN(64); break;
    default:
      knn_top1_generic_kernel<<<dgr_blocks(n0, 128), 128, 0, st>>>(f0, (int)n0, f1, (int)n1, c, packed, nullptr);
  }
  knn_unpack_kernel<<<dgr_blocks(n0, kThreads), kThreads, 0, st>>>(packed, n0, idx, dist);
  dgr_note_launches(3);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}
