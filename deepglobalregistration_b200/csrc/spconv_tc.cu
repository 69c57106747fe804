// Sparse convolution forward on the Hopper tensor cores (wgmma, sm_90a).
//
// Same contract as dgr_spconv_fwd (gather -> per-offset sub-GEMM -> scatter-add over the
// (kappa, j)-sorted pair lists) with the sub-GEMM issued as wgmma.mma_async and the accumulator
// in registers:
//
//   * one CTA = one 128-pair tile of one kernel offset, M = 128 rows (pairs) split over two
//     warpgroups (64 rows each), N = cout (16..256, padded to 32 / 64 / 128 / 256 with zero weight
//     rows), K = cin in chunks of one 128-byte swizzle row (32 TF32 or 64 FP16 channels);
//   * all 256 threads gather the 128 input rows (coalesced 16-byte pieces, 8 lanes per row, the
//     next chunk in flight while the current one multiplies), split every value into a "hi" part and
//     a "lo" residual and store both into shared memory in the canonical K-major SWIZZLE_128B layout;
//     one thread bulk-copies the weight slab of the chunk (TMA engine, completion on an mbarrier);
//   * each warpgroup issues, per k-step, the three products hi*hi + lo*hi + hi*lo (3xTF32 or
//     3xFP16, fp32-accurate to ~2^-21 relative) from two shared-memory stages, so the stores of
//     chunk c+1 overlap the MMAs of chunk c;
//   * the epilogue scatter-adds the accumulator fragments with red.global.add.v2.f32.
//
// Weights come PRE-SPLIT and PRE-SWIZZLED (dgr_pack_weight_tf32 / dgr_pack_weight_f16, cached per layer
// by the host): per (offset, chunk) one contiguous slab holding the hi tile and the lo tile in
// shared-memory image order.
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

#define DGR_TRY_RC(expr)             \
  do {                              \
    int32_t rc__ = (expr);          \
    if (rc__ != DGR_OK) return rc__; \
  } while (0)

constexpr int kThreadsTC = 256;          // two warpgroups: tile rows 0..63 and 64..127
constexpr int kTileM = 128;
constexpr int kChunk = 32;               // TF32 channels per 128-byte row
constexpr int kATileBytes = kTileM * 128;
constexpr int kStages = 2;

struct TcShared {
  unsigned long long full[kStages];     // weight slab of the stage has landed (bulk-copy bytes)
};

// shared-memory bytes of spconv_tc_kernel<NT, *>
constexpr size_t tc_smem_bytes(int nt) {
  return sizeof(TcShared) + 1024 + (size_t)kStages * (2 * kATileBytes + 2 * nt * 128);
}

// kF16: 3xFP16 instead of 3xTF32 (64 channels per 128-byte stage row; `wt` then holds the fp16 slabs of
// dgr_pack_weight_f16, amax_in the input tensor's absolute maximum, w_inv_scale the inverse of the weight scale)
template <int NT, bool kF16, int kPasses>
__global__ void __launch_bounds__(kThreadsTC, 1)
spconv_tc_kernel(const float* __restrict__ in_feat, int cin, const unsigned char* __restrict__ wt, int cout,
                 const int32_t* __restrict__ in_idx, const int32_t* __restrict__ out_idx,
                 const int32_t* __restrict__ kofs, const int32_t* __restrict__ tile_k,
                 const int32_t* __restrict__ tile_start, const float* __restrict__ amax_in,
                 const float* __restrict__ w_inv_scale, float* __restrict__ out) {
  constexpr int kCh = kF16 ? 64 : kChunk;        // channels per stage (one 128-byte swizzle row)
  constexpr int kV = kF16 ? 2 : 1;               // float4 loads per (thread, row, chunk)
  constexpr int kBTileBytes = NT * 128;          // B tile in shared memory: rows >= cout stay zero
  constexpr int kStageBytes = 2 * kATileBytes + 2 * kBTileBytes;
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  TcShared& sh = *reinterpret_cast<TcShared*>(smem_dyn);
  // stage buffers start at the next 1024-byte boundary (SWIZZLE_128B atom alignment)
  unsigned char* stage0 = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_dyn) + sizeof(TcShared) + 1023) & ~(uintptr_t)1023);
  const int t = threadIdx.x, wg = t >> 7;
  const int n_chunks = cin / kCh;
  const uint32_t b_tile_bytes = (uint32_t)cout * 128;   // one tile (hi or lo) of the packed slab
  const uint32_t slab_bytes = 2 * b_tile_bytes;
  const int kappa = tile_k[blockIdx.x];
  const int p0 = tile_start[blockIdx.x];
  const int rows = min(kTileM, kofs[kappa + 1] - p0);   // <= 0 for the padding tiles of a paired list

  if (t == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(smem_u32(&sh.full[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (NT > cout) {     // zero the padding rows of every B tile once: the bulk copies never write them
    const int pad_pieces = (NT - cout) * 8;
    for (int i = t; i < kStages * 2 * pad_pieces; i += kThreadsTC) {
      const int tile = i / pad_pieces, e = i % pad_pieces;
      *reinterpret_cast<uint4*>(stage0 + (tile >> 1) * kStageBytes + 2 * kATileBytes + (tile & 1) * kBTileBytes +
                                (cout + (e >> 3)) * 128 + (e & 7) * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
  }

  // gather: 8 lanes cover one 128-byte row; 32 row groups, rows rgrp + 32 i
  const int piece = t & 7, rgrp = t >> 3;
  const uint32_t a_off = (uint32_t)(rgrp * 128 + ((piece ^ (rgrp & 7)) << 4));   // + i * 4096
  int src[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = i * 32 + rgrp;
    src[i] = (r < rows) ? __ldg(in_idx + p0 + r) : -1;
  }
  float4 v[4][kV];
  auto load_a = [&](int c) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int u = 0; u < kV; ++u)
        v[i][u] = src[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(in_feat + (size_t)src[i] * cin + c * kCh +
                                                                       piece * (4 * kV) + 4 * u))
                              : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  const float sx = kF16 ? f16_scale_for(__ldg(amax_in)) : 1.f;
  const unsigned char* slab = wt + (size_t)kappa * n_chunks * slab_bytes;

  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
  load_a(0);
  for (int c = 0; c < n_chunks; ++c) {
    const int s = c % kStages;
    const uint32_t ph = (c / kStages) & 1;
    unsigned char* a_hi = stage0 + (size_t)s * kStageBytes;
    unsigned char* a_lo = a_hi + kATileBytes;
    unsigned char* b_hi = a_lo + kATileBytes;
    // every warpgroup has retired the MMAs of chunk c - kStages (wgmma_wait below): stage s is free
    __syncthreads();
    if (t == 0) {
      const unsigned char* bsrc = slab + (size_t)c * slab_bytes;
      mbar_arrive_expect_tx(smem_u32(&sh.full[s]), kPasses == 3 ? slab_bytes : b_tile_bytes);
      bulk_g2s(smem_u32(b_hi), bsrc, b_tile_bytes, smem_u32(&sh.full[s]));
      if (kPasses == 3) bulk_g2s(smem_u32(b_hi + kBTileBytes), bsrc + b_tile_bytes, b_tile_bytes, smem_u32(&sh.full[s]));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (kF16) split_store_f16(v[i][0], v[i][kV - 1], sx, a_hi, a_lo, a_off + i * 4096);
      else split_store(v[i][0], a_hi, a_lo, a_off + i * 4096);
    }
    if (c + 1 < n_chunks) load_a(c + 1);          // in flight while chunk c multiplies
    fence_proxy_async();
    __syncthreads();
    mbar_wait(smem_u32(&sh.full[s]), ph);
    wgmma_fence();
    const uint32_t a0 = smem_u32(a_hi) + wg * (kATileBytes / 2);
    mma_chunk<NT, kF16, kPasses>(acc, a0, a0 + kATileBytes, smem_u32(b_hi), smem_u32(b_hi) + kBTileBytes);
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  fence_acc(acc);

  // epilogue: thread holds rows r0 and r0 + 8 of its warpgroup, two adjacent columns per 8-column group
  // kF16: the accumulator holds (sx * x) . (sw * w); both scales are powers of two, undone exactly here
  const float inv = kF16 ? __ldg(w_inv_scale) / sx : 1.f;
  const int lane = t & 31;
  const int r0 = wg * 64 + ((t >> 5) & 3) * 16 + (lane >> 2);
  const int j0 = r0 < rows ? out_idx[p0 + r0] : -1;
  const int j1 = r0 + 8 < rows ? out_idx[p0 + r0 + 8] : -1;
  float* o0 = out + (size_t)(j0 < 0 ? 0 : j0) * cout;
  float* o1 = out + (size_t)(j1 < 0 ? 0 : j1) * cout;
#pragma unroll
  for (int i = 0; i < NT / 8; ++i) {
    const int col = 8 * i + 2 * (lane & 3);
    if (col < cout) {
      if (j0 >= 0) red_add_v2(o0 + col, acc[4 * i] * inv, acc[4 * i + 1] * inv);
      if (j1 >= 0) red_add_v2(o1 + col, acc[4 * i + 2] * inv, acc[4 * i + 3] * inv);
    }
  }
}

// one instantiation per kernel: DGR_ENSURE_SMEM keeps its attribute state per call site
template <int NT, bool kF16, int kPasses>
int32_t launch_spconv_tc(const float* in_feat, int cin, const void* wt, int cout, const int32_t* in_idx,
                         const int32_t* out_idx, const int32_t* kofs, const int32_t* tile_k, const int32_t* tile_start,
                         int n_tiles, const float* amax_in, const float* w_inv_scale, float* out, cudaStream_t st) {
  const size_t smem = tc_smem_bytes(NT);
  DGR_ENSURE_SMEM((spconv_tc_kernel<NT, kF16, kPasses>), smem);
  spconv_tc_kernel<NT, kF16, kPasses><<<n_tiles, kThreadsTC, smem, st>>>(
      in_feat, cin, (const unsigned char*)wt, cout, in_idx, out_idx, kofs, tile_k, tile_start, amax_in, w_inv_scale, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// the narrowest instantiated accumulator width >= cout (zero weight rows pad the rest)
template <bool kF16, int kPasses>
int32_t launch_spconv_tc(const float* in_feat, int cin, const void* wt, int cout, const int32_t* in_idx,
                         const int32_t* out_idx, const int32_t* kofs, const int32_t* tile_k, const int32_t* tile_start,
                         int n_tiles, const float* amax_in, const float* w_inv_scale, float* out, cudaStream_t st) {
  auto launch = cout <= 32 ? launch_spconv_tc<32, kF16, kPasses> : cout <= 64 ? launch_spconv_tc<64, kF16, kPasses>
                : cout <= 128 ? launch_spconv_tc<128, kF16, kPasses> : launch_spconv_tc<256, kF16, kPasses>;
  return launch(in_feat, cin, wt, cout, in_idx, out_idx, kofs, tile_k, tile_start, n_tiles, amax_in, w_inv_scale, out, st);
}

// W[K, cin, cout] fp32  ->  packed[K][cin/32][2][cout][32]: for every (kappa, 32-channel chunk) the
// K-major SWIZZLE_128B shared-memory image of the B operand, TF32 "hi" tile followed by the "lo"
// residual tile - exactly what one bulk copy drops into a pipeline stage.
__global__ void pack_weight_kernel(const float* __restrict__ w, int cin, int cout, float* __restrict__ packed) {
  const int n_chunks = cin / kChunk;
  const int64_t total = (int64_t)n_chunks * cout * 8;          // 16-byte pieces per kappa
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int kappa = blockIdx.y;
  const int n = (int)(e % cout);                                 // output channel = B row (fastest: coalesced)
  const int q = (int)((e / cout) % 8);                           // 16-byte piece inside the 128-byte row
  const int ch = (int)(e / ((int64_t)cout * 8));
  const float* src = w + ((size_t)kappa * cin + ch * kChunk + q * 4) * cout + n;
  float4 v = make_float4(src[0], src[cout], src[2 * (size_t)cout], src[3 * (size_t)cout]);
  float4 h, l;
  h.x = tf32_round(v.x); h.y = tf32_round(v.y); h.z = tf32_round(v.z); h.w = tf32_round(v.w);
  l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
  float* slab = packed + ((size_t)kappa * n_chunks + ch) * 2 * cout * 32;
  const int off = n * 32 + ((q ^ (n & 7)) << 2);                 // floats
  *reinterpret_cast<float4*>(slab + off) = h;
  *reinterpret_cast<float4*>(slab + (size_t)cout * 32 + off) = l;
}

// |x| maximum of a tensor as float bits (non-negative floats order like unsigned ints)
__global__ void absmax_kernel(const float* __restrict__ x, int64_t n, unsigned* __restrict__ out) {
  float m = 0.f;
  const int64_t n4 = n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) m = fmaxf(m, fabsf(x[(n4 << 2) + threadIdx.x]));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

// W[K, cin, cout] fp32 -> packed[K][cin/64][2][cout][64 halves]: per (kappa, 64-channel chunk) the K-major
// SWIZZLE_128B image of the B operand, fp16 hi tile then fp16 lo tile of (sw * W); scale[0] = 1 / sw.
__global__ void pack_weight_f16_kernel(const float* __restrict__ w, int cin, int cout, const float* __restrict__ amax,
                                       unsigned char* __restrict__ packed, float* __restrict__ scale) {
  const int n_chunks = cin / 64;
  const int64_t total = (int64_t)n_chunks * cout * 8;          // 16-byte pieces (8 halves) per kappa
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float sw = f16_scale_for(*amax);
  if (e == 0 && blockIdx.y == 0) scale[0] = 1.f / sw;
  if (e >= total) return;
  const int kappa = blockIdx.y;
  const int n = (int)(e % cout);
  const int q = (int)((e / cout) % 8);
  const int ch = (int)(e / ((int64_t)cout * 8));
  const float* src = w + ((size_t)kappa * cin + ch * 64 + q * 8) * cout + n;
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float x0 = src[(size_t)(2 * i) * cout] * sw, x1 = src[(size_t)(2 * i + 1) * cout] * sw;
    const __half2 hh = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(hh);
    const __half2 ll = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hh);
    l[i] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  unsigned char* slab = packed + ((size_t)kappa * n_chunks + ch) * 2 * cout * 128;
  const int off = n * 128 + ((q ^ (n & 7)) << 4);
  *reinterpret_cast<uint4*>(slab + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(slab + (size_t)cout * 128 + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

}  // namespace

extern "C" {

// Layout transform the tensor-core path needs once per layer: W[K, cin, cout] ->
// packed[K][cin/32][2][cout][32] (TF32 hi / lo tiles in shared-memory image order), 2x the size.
int32_t dgr_pack_weight_tf32(const float* w, int32_t K, int32_t cin, int32_t cout, float* packed, void* stream) {
  DGR_ARG_CHECK(K >= 1 && cin >= 32 && cin % 32 == 0 && cout >= 8 && cout % 8 == 0, "bad weight shape");
  DGR_ARG_CHECK(K <= 65535, "K too large");
  const int64_t per_k = (int64_t)(cin / kChunk) * cout * 8;
  dim3 grid(dgr_blocks(per_k, 256), K);
  pack_weight_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, cin, cout, packed);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}


// 1 if dgr_spconv_tc_fwd supports the shape (cin % 32 == 0, cout % 16 == 0, 16 <= cout <= 256).
int32_t dgr_spconv_tc_supported(int32_t cin, int32_t cout) {
  return (cin >= 32 && cin % 32 == 0 && cout >= 16 && cout <= 256 && cout % 16 == 0) ? 1 : 0;
}

// Tensor-core variant of dgr_spconv_fwd.  weight_t is the packed layout of dgr_pack_weight_tf32.
// passes = 3: 3xTF32 (fp32-accurate, default); passes = 1: single TF32 product (~1e-3 rel.).
int32_t dgr_spconv_tc_fwd(const float* in_feat, int32_t cin, const float* weight_t, int32_t cout,
                          const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs,
                          const int32_t* tile_k, const int32_t* tile_start, int32_t n_tiles,
                          int32_t tile_rows, int32_t passes, float* out, void* stream) {
  DGR_ARG_CHECK(tile_rows == kTileM, "tile_rows must be 128");
  DGR_ARG_CHECK(dgr_spconv_tc_supported(cin, cout), "shape not supported by the tensor-core path");
  DGR_ARG_CHECK(passes == 1 || passes == 3, "passes must be 1 or 3");
  if (n_tiles == 0) return DGR_OK;
  auto launch = passes == 3 ? launch_spconv_tc<false, 3> : launch_spconv_tc<false, 1>;
  return launch(in_feat, cin, weight_t, cout, in_idx, out_idx, kofs, tile_k, tile_start, n_tiles, nullptr, nullptr, out,
                (cudaStream_t)stream);
}

// amax[0] (device float) = max |x| over n floats; the slot is zeroed by the call.
int32_t dgr_absmax_f32(const float* x, int64_t n, float* amax, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DGR_CUDA_CHECK(cudaMemsetAsync(amax, 0, sizeof(float), st));
  if (n <= 0) return DGR_OK;
  int dev = 0, sms = 0;
  DGR_CUDA_CHECK(cudaGetDevice(&dev));
  DGR_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  unsigned blocks = dgr_blocks(n / 4 + 1, 256);
  if (blocks > 4u * sms) blocks = 4u * sms;      // grid-stride: four blocks per SM
  absmax_kernel<<<blocks, 256, 0, st>>>(x, n, reinterpret_cast<unsigned*>(amax));
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// 1 if dgr_spconv_tc_f16_fwd supports the shape: the 3xFP16 mode of the kernel
int32_t dgr_spconv_tc_f16_supported(int32_t cin, int32_t cout) {
  return (cin >= 64 && cin % 64 == 0 && cout >= 32 && cout <= 256 && cout % 32 == 0) ? 1 : 0;
}

// W[K, cin, cout] -> fp16 hi|lo slabs [K][cin/64][2][cout][64] (4 * K * cin * cout BYTES, half of the TF32
// slabs) of sw * W with sw the power of two that maps max|W| into [2^14, 2^15); scale_ws (device float[2]):
// [0] = 1 / sw (read by the kernel's epilogue), [1] = max |W| (workspace).
int32_t dgr_pack_weight_f16(const float* w, int32_t K, int32_t cin, int32_t cout, void* packed, float* scale_ws,
                            void* stream) {
  DGR_ARG_CHECK(K >= 1 && K <= 65535 && dgr_spconv_tc_f16_supported(cin, cout), "bad weight shape");
  DGR_TRY_RC(dgr_absmax_f32(w, (int64_t)K * cin * cout, scale_ws + 1, stream));
  const int64_t per_k = (int64_t)(cin / 64) * cout * 8;
  dim3 grid(dgr_blocks(per_k, 256), K);
  pack_weight_f16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, cin, cout, scale_ws + 1, (unsigned char*)packed,
                                                               scale_ws);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// dgr_spconv_tc_fwd with every product evaluated as hi*hi + lo*hi + hi*lo on FP16 splits of power-of-two-scaled
// operands (same 2^-21 accuracy as 3xTF32, half the weight bytes, twice the tensor rate).
// amax_in: device float = max |in_feat| (dgr_absmax_f32, or an upper bound); w_scale: scale_ws of
// dgr_pack_weight_f16.  Takes the plain or the paired tile list (dgr_kernel_map_tiles).
int32_t dgr_spconv_tc_f16_fwd(const float* in_feat, int32_t cin, const void* weight_h, int32_t cout,
                              const int32_t* in_idx, const int32_t* out_idx, const int32_t* kofs,
                              const int32_t* tile_k, const int32_t* tile_start, int32_t n_tiles, int32_t tile_rows,
                              const float* amax_in, const float* w_scale, float* out, void* stream) {
  DGR_ARG_CHECK(tile_rows == kTileM, "tile_rows must be 128");
  DGR_ARG_CHECK(dgr_spconv_tc_f16_supported(cin, cout), "shape not supported by the 3xFP16 path");
  DGR_ARG_CHECK(amax_in != nullptr && w_scale != nullptr, "scales missing");
  if (n_tiles == 0) return DGR_OK;
  return launch_spconv_tc<true, 3>(in_feat, cin, weight_h, cout, in_idx, out_idx, kofs, tile_k, tile_start, n_tiles,
                                   amax_in, w_scale, out, (cudaStream_t)stream);
}

}  // extern "C"
