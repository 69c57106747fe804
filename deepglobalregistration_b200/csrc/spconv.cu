// Sparse convolution forward and the dense layers around it.
//
//   dgr_spconv_fwd        weight-stationary gather -> sub-GEMM -> scatter-add over the
//                         (kappa, j)-sorted pair lists: one CTA per 128-pair tile of one
//                         kernel offset, input rows gathered with 16-byte cp.async into
//                         shared memory, fp32 FFMA register tiles, vectorised
//                         red.global.add.v4.f32 scatter.
//   dgr_spconv_table_fwd_strided  output-stationary kernel for conv1 (cin <= 8): walks the
//                         dense neighbour table, weights in shared memory, fused BatchNorm.
//   dgr_linear_fwd        1x1 convolutions with fused concat / bias / ReLU / L2-normalise.
//   dgr_affine_act, dgr_cat2, dgr_l2_normalize   elementwise layers.
//
// Replaces MinkowskiConvolution / MinkowskiConvolutionTranspose / MinkowskiBatchNorm /
// MEF.relu / ME.cat as used by model/resunet.py:598-649 and model/residual_block.py:118-134.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTileM = 128;   // pairs (rows) per tile
constexpr int kChunkK = 32;   // input channels per shared-memory stage
constexpr int kAStride = kChunkK + 4;   // floats; keeps 16-byte alignment, breaks bank aliasing

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = valid ? 16 : 0;   // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit_wait() {
  asm volatile("cp.async.commit_group;\n" ::);
  asm volatile("cp.async.wait_group 0;\n" ::);
}
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(a), "f"(b),
               "f"(c), "f"(d)
               : "memory");
}

// One 128 x TN output tile accumulated over `cin` input channels.
// A rows come from `row_ptr(r)` (nullptr -> zero row); W chunk rows from w + c * ldw.
// Thread layout: tx = t % (TN/4) owns 4 consecutive output columns, ty = t / (TN/4)
// owns RPT consecutive rows.
template <int TN>
struct TileCfg {
  static constexpr int kColThreads = TN / 4;
  static constexpr int kRowThreads = kThreads / kColThreads;
  static constexpr int kRpt = kTileM / kRowThreads;
};

template <int TN, bool kAligned, bool kReluIn, typename RowSrc>
__device__ __forceinline__ void tile_mainloop(RowSrc row_src, int cin, const float* __restrict__ w,
                                              int ldw, int n0, int ncols_valid, float* As, float* Ws,
                                              float (&acc)[TileCfg<TN>::kRpt][4]) {
  using Cfg = TileCfg<TN>;
  const int t = threadIdx.x;
  const int tx = t % Cfg::kColThreads, ty = t / Cfg::kColThreads;
  for (int c0 = 0; c0 < cin; c0 += kChunkK) {
    const int cn = min(kChunkK, cin - c0);
    // ---- stage A: 128 rows x 32 channels ------------------------------------------------
    if (kAligned) {
#pragma unroll
      for (int q = 0; q < (kTileM * kChunkK / 4) / kThreads; ++q) {
        int e = q * kThreads + t;
        int r = e >> 3, ch = (e & 7) * 4;
        const float* src = row_src(r);
        bool ok = (src != nullptr) && (ch < cn);
        cp_async16(As + r * kAStride + ch, ok ? src + c0 + ch : w, ok);
      }
    } else {
      for (int e = t; e < kTileM * kChunkK; e += kThreads) {
        int r = e >> 5, ch = e & 31;
        const float* src = row_src(r);
        As[r * kAStride + ch] = (src != nullptr && ch < cn) ? src[c0 + ch] : 0.f;
      }
    }
    // ---- stage W: 32 x TN ---------------------------------------------------------------
    for (int e = t; e < kChunkK * TN / 4; e += kThreads) {
      int kk = e / (TN / 4), col = (e % (TN / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kk < cn) {
        const float* src = w + (int64_t)(c0 + kk) * ldw + n0 + col;
        if (col + 3 < ncols_valid && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
          v = *reinterpret_cast<const float4*>(src);
        } else {
          if (col + 0 < ncols_valid) v.x = src[0];
          if (col + 1 < ncols_valid) v.y = src[1];
          if (col + 2 < ncols_valid) v.z = src[2];
          if (col + 3 < ncols_valid) v.w = src[3];
        }
      }
      *reinterpret_cast<float4*>(Ws + kk * TN + col) = v;
    }
    if (kAligned) cp_async_commit_wait();
    __syncthreads();
    // ---- FFMA ---------------------------------------------------------------------------
#pragma unroll
    for (int kk = 0; kk < kChunkK; kk += 4) {
      float4 b0 = *reinterpret_cast<const float4*>(Ws + (kk + 0) * TN + tx * 4);
      float4 b1 = *reinterpret_cast<const float4*>(Ws + (kk + 1) * TN + tx * 4);
      float4 b2 = *reinterpret_cast<const float4*>(Ws + (kk + 2) * TN + tx * 4);
      float4 b3 = *reinterpret_cast<const float4*>(Ws + (kk + 3) * TN + tx * 4);
#pragma unroll
      for (int r = 0; r < Cfg::kRpt; ++r) {
        float4 a = *reinterpret_cast<const float4*>(As + (ty * Cfg::kRpt + r) * kAStride + kk);
        if (kReluIn) {
          a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
        }
        acc[r][0] = fmaf(a.x, b0.x, acc[r][0]); acc[r][1] = fmaf(a.x, b0.y, acc[r][1]);
        acc[r][2] = fmaf(a.x, b0.z, acc[r][2]); acc[r][3] = fmaf(a.x, b0.w, acc[r][3]);
        acc[r][0] = fmaf(a.y, b1.x, acc[r][0]); acc[r][1] = fmaf(a.y, b1.y, acc[r][1]);
        acc[r][2] = fmaf(a.y, b1.z, acc[r][2]); acc[r][3] = fmaf(a.y, b1.w, acc[r][3]);
        acc[r][0] = fmaf(a.z, b2.x, acc[r][0]); acc[r][1] = fmaf(a.z, b2.y, acc[r][1]);
        acc[r][2] = fmaf(a.z, b2.z, acc[r][2]); acc[r][3] = fmaf(a.z, b2.w, acc[r][3]);
        acc[r][0] = fmaf(a.w, b3.x, acc[r][0]); acc[r][1] = fmaf(a.w, b3.y, acc[r][1]);
        acc[r][2] = fmaf(a.w, b3.z, acc[r][2]); acc[r][3] = fmaf(a.w, b3.w, acc[r][3]);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------
// gather -> sub-GEMM -> scatter-add
// ---------------------------------------------------------------------------------------
template <int TN, bool kAligned, bool kReluIn>
__global__ void __launch_bounds__(kThreads)
spconv_fwd_kernel(const float* __restrict__ in_feat, int cin, const float* __restrict__ weight,
                  int cout, const int32_t* __restrict__ in_idx, const int32_t* __restrict__ out_idx,
                  const int32_t* __restrict__ kofs, const int32_t* __restrict__ tile_k,
                  const int32_t* __restrict__ tile_start, float* __restrict__ out) {
  using Cfg = TileCfg<TN>;
  __shared__ __align__(16) float As[kTileM * kAStride];
  __shared__ __align__(16) float Ws[kChunkK * TN];
  __shared__ int s_in[kTileM];
  __shared__ int s_out[kTileM];
  const int tile = blockIdx.x;
  const int n0 = blockIdx.y * TN;
  const int kappa = tile_k[tile];
  const int p0 = tile_start[tile];
  const int rows = min(kTileM, kofs[kappa + 1] - p0);
  if (threadIdx.x < kTileM) {
    bool ok = threadIdx.x < rows;
    s_in[threadIdx.x] = ok ? in_idx[p0 + threadIdx.x] : -1;
    s_out[threadIdx.x] = ok ? out_idx[p0 + threadIdx.x] : -1;
  }
  __syncthreads();
  float acc[Cfg::kRpt][4];
#pragma unroll
  for (int r = 0; r < Cfg::kRpt; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
  const float* w = weight + (int64_t)kappa * cin * cout;
  auto row_src = [&](int r) -> const float* {
    int i = s_in[r];
    return i >= 0 ? in_feat + (int64_t)i * cin : nullptr;
  };
  tile_mainloop<TN, kAligned, kReluIn>(row_src, cin, w, cout, n0, cout - n0, As, Ws, acc);
  const int tx = threadIdx.x % Cfg::kColThreads, ty = threadIdx.x / Cfg::kColThreads;
  const int col = n0 + tx * 4;
  const bool vec = (cout % 4 == 0) && (col + 3 < cout);
#pragma unroll
  for (int r = 0; r < Cfg::kRpt; ++r) {
    int j = s_out[ty * Cfg::kRpt + r];
    if (j < 0) continue;
    float* dst = out + (int64_t)j * cout + col;
    if (vec) {
      red_add_v4(dst, acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (col + c < cout) atomicAdd(dst + c, acc[r][c]);
    }
  }
}

// ---------------------------------------------------------------------------------------
// 1x1 convolution: out = act(concat(a, b) @ W + bias)
// ---------------------------------------------------------------------------------------
template <int TN>
__global__ void __launch_bounds__(kThreads)
linear_fwd_kernel(const float* __restrict__ a, int ca, const float* __restrict__ b, int cb, int64_t n,
                  const float* __restrict__ weight, int cout, const float* __restrict__ bias, int relu,
                  int normalize, float* __restrict__ out) {
  using Cfg = TileCfg<TN>;
  __shared__ __align__(16) float As[kTileM * kAStride];
  __shared__ __align__(16) float Ws[kChunkK * TN];
  const int64_t r0 = (int64_t)blockIdx.x * kTileM;
  const int n0 = blockIdx.y * TN;
  float acc[Cfg::kRpt][4];
#pragma unroll
  for (int r = 0; r < Cfg::kRpt; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
  {
    auto src_a = [&](int r) -> const float* { return (r0 + r < n) ? a + (r0 + r) * ca : nullptr; };
    if (ca % 4 == 0)
      tile_mainloop<TN, true, false>(src_a, ca, weight, cout, n0, cout - n0, As, Ws, acc);
    else
      tile_mainloop<TN, false, false>(src_a, ca, weight, cout, n0, cout - n0, As, Ws, acc);
  }
  if (b != nullptr && cb > 0) {
    auto src_b = [&](int r) -> const float* { return (r0 + r < n) ? b + (r0 + r) * cb : nullptr; };
    const float* w2 = weight + (int64_t)ca * cout;
    if (cb % 4 == 0)
      tile_mainloop<TN, true, false>(src_b, cb, w2, cout, n0, cout - n0, As, Ws, acc);
    else
      tile_mainloop<TN, false, false>(src_b, cb, w2, cout, n0, cout - n0, As, Ws, acc);
  }
  const int tx = threadIdx.x % Cfg::kColThreads, ty = threadIdx.x / Cfg::kColThreads;
  const int col = n0 + tx * 4;
  float bv[4] = {0.f, 0.f, 0.f, 0.f};
  if (bias != nullptr)
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (col + c < cout) bv[c] = bias[col + c];
#pragma unroll
  for (int r = 0; r < Cfg::kRpt; ++r) {
    const int64_t row = r0 + ty * Cfg::kRpt + r;
    float v[4];
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      v[c] = acc[r][c] + bv[c];
      if (relu) v[c] = fmaxf(v[c], 0.f);
      if (col + c < cout) ss += v[c] * v[c];
    }
    if (normalize) {
      // the row's cout <= TN columns live in the kColThreads consecutive lanes of this row
#pragma unroll
      for (int d = Cfg::kColThreads / 2; d > 0; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
      const float inv = 1.f / (sqrtf(ss) + 1e-8f);
#pragma unroll
      for (int c = 0; c < 4; ++c) v[c] *= inv;
    }
    if (row < n) {
      float* dst = out + row * cout + col;
      if ((cout % 4 == 0) && (col + 3 < cout)) {
        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (col + c < cout) dst[c] = v[c];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// output-stationary convolution for few input channels (conv1)
// ---------------------------------------------------------------------------------------
template <int COUT>
__global__ void __launch_bounds__(kThreads)
spconv_table_kernel(const float* __restrict__ in_feat, int cin, const float* __restrict__ weight,
                    const int32_t* __restrict__ nbr, int K, int64_t n_out, int64_t nbr_stride,
                    const float* __restrict__ scale, const float* __restrict__ shift,
                    float* __restrict__ out) {
  extern __shared__ __align__(16) float w_s[];   // [kc, cin, COUT] chunk of the weights
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  const int kc_max = (44 * 1024 / 4) / (cin * COUT);   // offsets per shared-memory chunk
  for (int k0 = 0; k0 < K; k0 += kc_max) {
    const int kn = min(kc_max, K - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < kn * cin * COUT; e += blockDim.x)
      w_s[e] = weight[(int64_t)k0 * cin * COUT + e];
    __syncthreads();
    if (j < n_out) {
      // the table reads are independent of everything else: keep 8 of them (and, for one input
      // channel, the 8 gathered features) in flight instead of one dependent load per offset
      for (int kb = 0; kb < kn; kb += 8) {
        int idx[8];
        float x0[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          idx[u] = (kb + u < kn) ? __ldcs(nbr + (int64_t)(k0 + kb + u) * nbr_stride + j) : -1;
#pragma unroll
        for (int u = 0; u < 8; ++u) x0[u] = idx[u] >= 0 ? __ldg(in_feat + (int64_t)idx[u] * cin) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (idx[u] < 0) continue;
          for (int ci = 0; ci < cin; ++ci) {
            const float x = ci == 0 ? x0[u] : __ldg(in_feat + (int64_t)idx[u] * cin + ci);
            const float4* wr = reinterpret_cast<const float4*>(w_s + ((kb + u) * cin + ci) * COUT);
#pragma unroll
            for (int c4 = 0; c4 < COUT / 4; ++c4) {
              float4 wv = wr[c4];
              acc[4 * c4 + 0] = fmaf(x, wv.x, acc[4 * c4 + 0]);
              acc[4 * c4 + 1] = fmaf(x, wv.y, acc[4 * c4 + 1]);
              acc[4 * c4 + 2] = fmaf(x, wv.z, acc[4 * c4 + 2]);
              acc[4 * c4 + 3] = fmaf(x, wv.w, acc[4 * c4 + 3]);
            }
          }
        }
      }
    }
  }
  if (j >= n_out) return;
  float4* dst = reinterpret_cast<float4*>(out + j * COUT);
#pragma unroll
  for (int c4 = 0; c4 < COUT / 4; ++c4) {
    float v[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      v[c] = acc[4 * c4 + c];
      if (scale != nullptr) v[c] = v[c] * scale[4 * c4 + c] + shift[4 * c4 + c];
    }
    dst[c4] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// conv1 of the FCGF network on its actual input: ONE input channel whose value is 1 for every voxel
// (core/deep_global_registration.py:96,159: `feats = ones`).  Then out[j, :] = sum over the occupied offsets
// kappa of W[kappa, 0, :]: only the OCCUPANCY of the 7^3 neighbourhood matters, not which row sits there - the
// kernel reads the kernel map's bit masks (bits[kappa][j / 32], one word per warp and offset, broadcast) instead of
// a dense 343 x N index table: 32x less traffic, and the map needs neither pair lists nor a neighbour table.
template <int COUT>
__global__ void __launch_bounds__(kThreads)
spconv_ones_bits_kernel(const float* __restrict__ weight, const uint32_t* __restrict__ bits, int W, int K, int64_t n_out,
                        const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ out) {
  extern __shared__ __align__(16) float w_s[];   // [kc, COUT] chunk of the weights
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int w = (int)(j >> 5), lane = threadIdx.x & 31;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  const int kc_max = (44 * 1024 / 4) / COUT;
  for (int k0 = 0; k0 < K; k0 += kc_max) {
    const int kn = min(kc_max, K - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < kn * COUT; e += blockDim.x) w_s[e] = weight[(int64_t)k0 * COUT + e];
    __syncthreads();
    if (w < W) {
      for (int kb = 0; kb < kn; kb += 8) {
        uint32_t m[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) m[u] = (kb + u < kn) ? __ldg(bits + (int64_t)(k0 + kb + u) * W + w) : 0u;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (!((m[u] >> lane) & 1u)) continue;
          const float4* wr = reinterpret_cast<const float4*>(w_s + (kb + u) * COUT);
#pragma unroll
          for (int c4 = 0; c4 < COUT / 4; ++c4) {
            const float4 wv = wr[c4];
            acc[4 * c4 + 0] += wv.x; acc[4 * c4 + 1] += wv.y; acc[4 * c4 + 2] += wv.z; acc[4 * c4 + 3] += wv.w;
          }
        }
      }
    }
  }
  if (j >= n_out) return;
  float4* dst = reinterpret_cast<float4*>(out + j * COUT);
#pragma unroll
  for (int c4 = 0; c4 < COUT / 4; ++c4) {
    float v[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      v[c] = acc[4 * c4 + c];
      if (scale != nullptr) v[c] = v[c] * scale[4 * c4 + c] + shift[4 * c4 + c];
    }
    dst[c4] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// ---------------------------------------------------------------------------------------
// elementwise
// ---------------------------------------------------------------------------------------
// amax (optional): receives max |out| as float bits (atomicMax on non-negative floats) - the activation scale the
// 3xFP16 convolution that consumes `out` needs, for free in the pass that produces it
__global__ void affine_act_kernel(const float* __restrict__ x, int64_t total, int c,
                                  const float* __restrict__ scale, const float* __restrict__ shift,
                                  const float* __restrict__ residual, int relu, float* out, unsigned* amax) {
  // c % 4 == 0: one float4 per thread
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  float m = 0.f;
  if (i < total) {
    const int ch = (int)(i % c);
    float4 v = *reinterpret_cast<const float4*>(x + i);
    if (scale != nullptr) {
      const float4 s = *reinterpret_cast<const float4*>(scale + ch);
      const float4 b = *reinterpret_cast<const float4*>(shift + ch);
      v.x = v.x * s.x + b.x; v.y = v.y * s.y + b.y; v.z = v.z * s.z + b.z; v.w = v.w * s.w + b.w;
    }
    if (residual != nullptr) {
      const float4 r = *reinterpret_cast<const float4*>(residual + i);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    *reinterpret_cast<float4*>(out + i) = v;
    m = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
  }
  if (amax != nullptr) {               // uniform branch: every thread of the block takes part
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
    __shared__ float wmax[kThreads / 32];
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int w = 1; w < kThreads / 32; ++w) m = fmaxf(m, wmax[w]);
      // one same-address atomic per BLOCK at most, and only from blocks that raise the slot (a plain read
      // filters the rest: same-address atomics serialise at L2)
      if (__float_as_uint(m) > *reinterpret_cast<volatile unsigned*>(amax)) atomicMax(amax, __float_as_uint(m));
    }
  }
}

__global__ void affine_act_scalar_kernel(const float* __restrict__ x, int64_t total, int c,
                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                         const float* __restrict__ residual, int relu, float* out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int ch = (int)(i % c);
  float v = x[i];
  if (scale != nullptr) v = v * scale[ch] + shift[ch];
  if (residual != nullptr) v += residual[i];
  if (relu) v = fmaxf(v, 0.f);
  out[i] = v;
}

__global__ void cat2_kernel(const float* __restrict__ a, int ca, const float* __restrict__ b, int cb,
                            int64_t n, float* __restrict__ out) {
  const int c = ca + cb;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * c) return;
  int64_t r = i / c;
  int ch = (int)(i - r * c);
  out[i] = ch < ca ? a[r * ca + ch] : b[r * cb + (ch - ca)];
}

// one warp per row
__global__ void l2_normalize_kernel(const float* __restrict__ x, int64_t n, int c, float* out) {
  int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (row >= n) return;
  float ss = 0.f;
  for (int ch = lane; ch < c; ch += 32) {
    float v = x[row * c + ch];
    ss += v * v;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
  float inv = 1.f / (sqrtf(ss) + 1e-8f);
  for (int ch = lane; ch < c; ch += 32) out[row * c + ch] = x[row * c + ch] * inv;
}

// ---------------------------------------------------------------------------------------
// weight gradient (training, SURVEY 8f rank 3): dW[kappa] = sum_{p in bucket kappa} in[i_p]^T (x) gout[j_p]
// One block per (kappa, 32 input channels, 64 output channels); pairs are staged 32 at a time in shared
// memory (row gathers, coalesced along the channels); every block sums its bucket in order: deterministic.
// ---------------------------------------------------------------------------------------
constexpr int kWgCi = 32, kWgCo = 64, kWgP = 32;
__global__ void __launch_bounds__(kThreads)
spconv_wgrad_kernel(const float* __restrict__ in_feat, int cin, const float* __restrict__ gout, int cout,
                    const int32_t* __restrict__ in_idx, const int32_t* __restrict__ out_idx,
                    const int32_t* __restrict__ kofs, float* __restrict__ dw) {
  __shared__ float As[kWgP][kWgCi + 1];
  __shared__ float Bs[kWgP][kWgCo];
  const int kappa = blockIdx.x;
  const int ci0 = blockIdx.y * kWgCi, co0 = blockIdx.z * kWgCo;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;      // 16 x 16 threads: 2 ci rows x 4 co columns each
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const int p_begin = kofs[kappa], p_end = kofs[kappa + 1];
  for (int p0 = p_begin; p0 < p_end; p0 += kWgP) {
    const int np = min(kWgP, p_end - p0);
    for (int e = t; e < kWgP * kWgCi; e += kThreads) {
      const int pp = e / kWgCi, c = e % kWgCi;
      As[pp][c] = (pp < np && ci0 + c < cin) ? in_feat[(size_t)in_idx[p0 + pp] * cin + ci0 + c] : 0.f;
    }
    for (int e = t; e < kWgP * kWgCo; e += kThreads) {
      const int pp = e / kWgCo, c = e % kWgCo;
      Bs[pp][c] = (pp < np && co0 + c < cout) ? gout[(size_t)out_idx[p0 + pp] * cout + co0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int pp = 0; pp < kWgP; ++pp) {
      const float a0 = As[pp][2 * ty], a1 = As[pp][2 * ty + 1];
      const float4 b = *reinterpret_cast<const float4*>(&Bs[pp][4 * tx]);
      acc[0][0] = fmaf(a0, b.x, acc[0][0]); acc[0][1] = fmaf(a0, b.y, acc[0][1]);
      acc[0][2] = fmaf(a0, b.z, acc[0][2]); acc[0][3] = fmaf(a0, b.w, acc[0][3]);
      acc[1][0] = fmaf(a1, b.x, acc[1][0]); acc[1][1] = fmaf(a1, b.y, acc[1][1]);
      acc[1][2] = fmaf(a1, b.z, acc[1][2]); acc[1][3] = fmaf(a1, b.w, acc[1][3]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int ci = ci0 + 2 * ty + r;
    if (ci >= cin) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int co = co0 + 4 * tx + c;
      if (co < cout) dw[((size_t)kappa * cin + ci) * cout + co] = acc[r][c];
    }
  }
}

}  // namespace

// =========================================================================================
// C ABI
// =========================================================================================
extern "C" {

int32_t dgr_spconv_fwd(const float* in_feat, int32_t cin, const float* weight, int32_t cout,
                       const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs,
                       const int32_t* tile_k, const int32_t* tile_start, int32_t n_tiles,
                       int32_t tile_rows, int32_t relu_in, float* out, void* stream) {
  DGR_ARG_CHECK(tile_rows == kTileM, "tile_rows must be 128");
  DGR_ARG_CHECK(cin >= 1 && cout >= 1, "channels must be positive");
  if (n_tiles == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool aligned = (cin % 4 == 0);
#define DGR_LAUNCH_SPCONV(TN, AL, RL)                                                          \
  spconv_fwd_kernel<TN, AL, RL><<<dim3(n_tiles, (cout + TN - 1) / TN), kThreads, 0, st>>>(      \
      in_feat, cin, weight, cout, in_idx, out_idx, kofs, tile_k, tile_start, out)
  if (cout <= 32) {
    if (aligned) { if (relu_in) DGR_LAUNCH_SPCONV(32, true, true); else DGR_LAUNCH_SPCONV(32, true, false); }
    else         { if (relu_in) DGR_LAUNCH_SPCONV(32, false, true); else DGR_LAUNCH_SPCONV(32, false, false); }
  } else {
    if (aligned) { if (relu_in) DGR_LAUNCH_SPCONV(64, true, true); else DGR_LAUNCH_SPCONV(64, true, false); }
    else         { if (relu_in) DGR_LAUNCH_SPCONV(64, false, true); else DGR_LAUNCH_SPCONV(64, false, false); }
  }
#undef DGR_LAUNCH_SPCONV
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_spconv_table_fwd_strided(const float* in_feat, int32_t cin, const float* weight, int32_t cout,
                                     const int32_t* nbr, int32_t K, int64_t n_out, int64_t nbr_stride,
                                     const float* scale, const float* shift, float* out, void* stream) {
  DGR_ARG_CHECK(cin >= 1 && cin <= 8, "table convolution supports 1..8 input channels");
  DGR_ARG_CHECK((scale == nullptr) == (shift == nullptr), "scale and shift go together");
  DGR_ARG_CHECK(nbr_stride >= n_out, "row stride of the neighbour table below its row count");
  if (n_out == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = 44 * 1024;
  const unsigned blocks = dgr_blocks(n_out, kThreads);
  if (cout == 32)
    spconv_table_kernel<32><<<blocks, kThreads, smem, st>>>(in_feat, cin, weight, nbr, K, n_out, nbr_stride, scale,
                                                           shift, out);
  else if (cout == 64)
    spconv_table_kernel<64><<<blocks, kThreads, smem, st>>>(in_feat, cin, weight, nbr, K, n_out, nbr_stride, scale,
                                                           shift, out);
  else if (cout == 16)
    spconv_table_kernel<16><<<blocks, kThreads, smem, st>>>(in_feat, cin, weight, nbr, K, n_out, nbr_stride, scale,
                                                           shift, out);
  else {
    dgr_set_error("dgr_spconv_table_fwd_strided: cout must be 16, 32 or 64 (got %d)", cout);
    return DGR_ERR_ARG;
  }
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// conv1 with one all-ones input channel from the kernel map's occupancy masks (dgr_kmap_probe's `bits`):
//   out[j, :] = (sum over kappa with bit (kappa, j) set of weight[kappa, 0, :]) * scale + shift.
// Same summation order over kappa as dgr_spconv_table_fwd_strided on an all-ones input (bit-identical result).
int32_t dgr_spconv_ones_bits_fwd(const float* weight, int32_t cout, const uint32_t* bits, int64_t mask_words, int32_t K,
                                 int64_t n_out, const float* scale, const float* shift, float* out, void* stream) {
  DGR_ARG_CHECK((scale == nullptr) == (shift == nullptr), "scale and shift go together");
  DGR_ARG_CHECK(mask_words * 32 >= n_out, "mask rows shorter than the output");
  if (n_out == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = 44 * 1024;
  const unsigned blocks = dgr_blocks(n_out, kThreads);
  if (cout == 32)
    spconv_ones_bits_kernel<32><<<blocks, kThreads, smem, st>>>(weight, bits, (int)mask_words, K, n_out, scale, shift, out);
  else if (cout == 64)
    spconv_ones_bits_kernel<64><<<blocks, kThreads, smem, st>>>(weight, bits, (int)mask_words, K, n_out, scale, shift, out);
  else if (cout == 16)
    spconv_ones_bits_kernel<16><<<blocks, kThreads, smem, st>>>(weight, bits, (int)mask_words, K, n_out, scale, shift, out);
  else {
    dgr_set_error("dgr_spconv_ones_bits_fwd: cout must be 16, 32 or 64 (got %d)", cout);
    return DGR_ERR_ARG;
  }
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_linear_fwd(const float* a, int32_t ca, const float* b, int32_t cb, int64_t n,
                       const float* weight, int32_t cout, const float* bias, int32_t relu,
                       int32_t normalize, float* out, void* stream) {
  DGR_ARG_CHECK(ca >= 1 && cout >= 1, "channels must be positive");
  DGR_ARG_CHECK(!normalize || cout <= 64, "fused normalisation needs cout <= 64");
  if (n == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned tiles = dgr_blocks(n, kTileM);
  if (cout <= 32)
    linear_fwd_kernel<32><<<dim3(tiles, (cout + 31) / 32), kThreads, 0, st>>>(a, ca, b, cb, n, weight, cout,
                                                                            bias, relu, normalize, out);
  else
    linear_fwd_kernel<64><<<dim3(tiles, (cout + 63) / 64), kThreads, 0, st>>>(a, ca, b, cb, n, weight, cout,
                                                                            bias, relu, normalize, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// dgr_affine_act that also reduces max |out| into amax[0] (device float; the CALLER zeroes it, so that several
// launches may reduce into one slot); requires c % 4 == 0 when amax is given.
int32_t dgr_affine_act_amax(const float* x, int64_t n, int32_t c, const float* scale, const float* shift,
                            const float* residual, int32_t relu, float* out, float* amax, void* stream) {
  DGR_ARG_CHECK((scale == nullptr) == (shift == nullptr), "scale and shift go together");
  DGR_ARG_CHECK(amax == nullptr || c % 4 == 0, "amax needs a channel count divisible by 4");
  const int64_t total = n * c;
  if (total == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (c % 4 == 0)
    affine_act_kernel<<<dgr_blocks(total / 4, kThreads), kThreads, 0, st>>>(x, total, c, scale, shift, residual, relu,
                                                                          out, reinterpret_cast<unsigned*>(amax));
  else
    affine_act_scalar_kernel<<<dgr_blocks(total, kThreads), kThreads, 0, st>>>(x, total, c, scale, shift,
                                                                             residual, relu, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_affine_act(const float* x, int64_t n, int32_t c, const float* scale, const float* shift,
                       const float* residual, int32_t relu, float* out, void* stream) {
  return dgr_affine_act_amax(x, n, c, scale, shift, residual, relu, out, nullptr, stream);
}

int32_t dgr_cat2(const float* a, int32_t ca, const float* b, int32_t cb, int64_t n, float* out,
                 void* stream) {
  if (n == 0) return DGR_OK;
  cat2_kernel<<<dgr_blocks(n * (ca + cb), kThreads), kThreads, 0, (cudaStream_t)stream>>>(a, ca, b, cb, n,
                                                                                       out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// Weight gradient of dgr_spconv_fwd / dgr_spconv_tc_fwd (training): dw[K, cin, cout] is overwritten with
// dw[kappa] = sum over the pairs p of bucket kappa of in_feat[in_idx[p], :]^T (x) grad_out[out_idx[p], :].
// The input gradient needs no kernel of its own: it is dgr_spconv_fwd on grad_out with the index lists
// exchanged and every W[kappa] transposed.
int32_t dgr_spconv_wgrad(const float* in_feat, int32_t cin, const float* grad_out, int32_t cout,
                         const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs, int32_t K, float* dw,
                         void* stream) {
  DGR_ARG_CHECK(K >= 1 && cin >= 1 && cout >= 1, "bad shape");
  DGR_ARG_CHECK((cin + kWgCi - 1) / kWgCi <= 65535 && (cout + kWgCo - 1) / kWgCo <= 65535, "too many channels");
  const dim3 grid(K, (cin + kWgCi - 1) / kWgCi, (cout + kWgCo - 1) / kWgCo);
  spconv_wgrad_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(in_feat, cin, grad_out, cout, in_idx, out_idx, kofs,
                                                                    dw);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_l2_normalize(const float* x, int64_t n, int32_t c, float* out, void* stream) {
  if (n == 0) return DGR_OK;
  l2_normalize_kernel<<<dgr_blocks(n * 32, kThreads), kThreads, 0, (cudaStream_t)stream>>>(x, n, c, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
