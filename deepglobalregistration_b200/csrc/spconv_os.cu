// Output-stationary sparse convolution on the tensor cores, with the layer's epilogue fused
// (eval BatchNorm scale / shift, residual add, ReLU) - for the stride-1 3^3 layers of the 3-D network
// (every BasicBlock convolution of the FCGF ResUNet: model/residual_block.py:118-134).
//
// dgr_spconv_tc_fwd is weight-stationary: a tile is 128 PAIRS of one kernel offset, results are
// scatter-added into the output with red.global.add (P x Cout x 4 bytes of atomic traffic on a
// pre-zeroed buffer, P/N ~ 17 for these layers), and BatchNorm / residual / ReLU need a second
// pass.  With only 27 offsets and ~64 % of the (row, offset) slots occupied, the output-stationary
// order is the better one:
//
//   tile          = 128 consecutive OUTPUT rows; the accumulator (registers of two warpgroups, fp32) lives through all
//                   27 offsets x Cin/32 chunks: D[128, Cout] += A_kappa[128, 32] . W[kappa][32, Cout]
//   A_kappa       = input rows nbr[kappa][j] gathered by all threads (missing neighbours are
//                   zero rows), split hi / lo as in the 3xTF32 kernel, K-major SWIZZLE_128B tiles
//   weights       = the same packed hi | lo slabs, one cp.async.bulk per stage
//   epilogue      = y = acc * scale + shift (+ residual), ReLU on the accumulator fragments: every output
//                   row is written exactly once with plain stores - no atomics, no memset, deterministic
//
// 1.56x the MMA work of the pair lists (zero rows are multiplied too) on layers whose tensor pipe is
// ~6-13 % busy; gather bytes unchanged (P x Cin x 4), output bytes N x Cout x 4 instead of the
// atomics' P x Cout x 4 (17x fewer), and the elementwise pass disappears.
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int kThreadsOS = 256;          // two warpgroups: tile rows 0..63 and 64..127
constexpr int kTileM = 128;
constexpr int kChunk = 32;
constexpr int kATileBytes = kTileM * 128;
constexpr int kStages = 2;

struct OsShared {
  unsigned long long full[kStages];     // weight slab of the stage has landed (bulk-copy bytes)
};

constexpr size_t os_smem_bytes(int nt) {
  return sizeof(OsShared) + 1024 + (size_t)kStages * (2 * kATileBytes + 2 * nt * 128);
}

template <int NT>
__global__ void __launch_bounds__(kThreadsOS, 1)
spconv_os_kernel(const float* __restrict__ in_feat, int cin, const float* __restrict__ wt, int cout,
                 const int32_t* __restrict__ nbr, int64_t nbr_stride, int K, int n_out,
                 const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ residual,
                 int relu, float* __restrict__ out) {
  constexpr int kBTileBytes = NT * 128;          // B tile in shared memory: rows >= cout stay zero
  constexpr int kStageBytes = 2 * kATileBytes + 2 * kBTileBytes;
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  OsShared& sh = *reinterpret_cast<OsShared*>(smem_dyn);
  unsigned char* stage0 = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_dyn) + sizeof(OsShared) + 1023) & ~(uintptr_t)1023);
  const int t = threadIdx.x, wg = t >> 7;
  const int n_chunks = cin / kChunk;
  const int steps = K * n_chunks;                 // (kappa, chunk) steps of the tile
  const uint32_t b_tile_bytes = (uint32_t)cout * 128;
  const uint32_t slab_bytes = 2 * b_tile_bytes;
  const int j0 = blockIdx.x * kTileM;

  if (t == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(smem_u32(&sh.full[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (NT > cout) {     // zero the padding rows of every B tile once: the bulk copies never write them
    const int pad_pieces = (NT - cout) * 8;
    for (int i = t; i < kStages * 2 * pad_pieces; i += kThreadsOS) {
      const int tile = i / pad_pieces, e = i % pad_pieces;
      *reinterpret_cast<uint4*>(stage0 + (tile >> 1) * kStageBytes + 2 * kATileBytes + (tile & 1) * kBTileBytes +
                                (cout + (e >> 3)) * 128 + (e & 7) * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
  }

  // gather: 8 lanes cover one 128-byte row; 32 row groups, rows rgrp + 32 i
  const int piece = t & 7, rgrp = t >> 3;
  const uint32_t a_off = (uint32_t)(rgrp * 128 + ((piece ^ (rgrp & 7)) << 4));
  int src[4];
  auto rows_of = [&](int kappa) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = j0 + i * 32 + rgrp;
      src[i] = (r < n_out) ? __ldg(nbr + (int64_t)kappa * nbr_stride + r) : -1;
    }
  };
  float4 v[4];
  auto load_a = [&](int c) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      v[i] = src[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(in_feat + (size_t)src[i] * cin + c * kChunk + piece * 4))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
  };

  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
  rows_of(0);
  load_a(0);
  for (int step = 0; step < steps; ++step) {
    const int s = step % kStages;
    const uint32_t ph = (step / kStages) & 1;
    unsigned char* a_hi = stage0 + (size_t)s * kStageBytes;
    unsigned char* a_lo = a_hi + kATileBytes;
    unsigned char* b_hi = a_lo + kATileBytes;
    __syncthreads();       // every warpgroup has retired the MMAs of step - kStages: stage s is free
    if (t == 0) {
      const unsigned char* bsrc = reinterpret_cast<const unsigned char*>(wt) + (size_t)step * slab_bytes;
      mbar_arrive_expect_tx(smem_u32(&sh.full[s]), slab_bytes);
      bulk_g2s(smem_u32(b_hi), bsrc, b_tile_bytes, smem_u32(&sh.full[s]));
      bulk_g2s(smem_u32(b_hi + kBTileBytes), bsrc + b_tile_bytes, b_tile_bytes, smem_u32(&sh.full[s]));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) split_store(v[i], a_hi, a_lo, a_off + i * 4096);
    if (step + 1 < steps) {                 // the next step's rows are in flight while this one multiplies
      const int c = (step + 1) % n_chunks;
      if (c == 0) rows_of((step + 1) / n_chunks);
      load_a(c);
    }
    fence_proxy_async();
    __syncthreads();
    mbar_wait(smem_u32(&sh.full[s]), ph);
    wgmma_fence();
    const uint32_t a0 = smem_u32(a_hi) + wg * (kATileBytes / 2);
    mma_chunk<NT, false, 3>(acc, a0, a0 + kATileBytes, smem_u32(b_hi), smem_u32(b_hi) + kBTileBytes);
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  fence_acc(acc);

  // epilogue: thread holds rows r and r + 8 of its warpgroup, two adjacent columns per 8-column group
  const int lane = t & 31;
  const int r = j0 + wg * 64 + ((t >> 5) & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < NT / 8; ++i) {
    const int col = 8 * i + 2 * (lane & 3);
    if (col < cout) {
      const float2 sc = scale != nullptr ? __ldg(reinterpret_cast<const float2*>(scale + col)) : make_float2(1.f, 1.f);
      const float2 sf = shift != nullptr ? __ldg(reinterpret_cast<const float2*>(shift + col)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = r + 8 * h;
        if (j < n_out) {
          float2 x = make_float2(fmaf(acc[4 * i + 2 * h], sc.x, sf.x), fmaf(acc[4 * i + 2 * h + 1], sc.y, sf.y));
          const size_t o = (size_t)j * cout + col;
          if (residual != nullptr) {
            const float2 r2 = __ldg(reinterpret_cast<const float2*>(residual + o));
            x.x += r2.x; x.y += r2.y;
          }
          if (relu) {
            x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f);
          }
          *reinterpret_cast<float2*>(out + o) = x;
        }
      }
    }
  }
}

// one instantiation per kernel: DGR_ENSURE_SMEM keeps its attribute state per call site
template <int NT>
int32_t launch_spconv_os(const float* in_feat, int cin, const float* wt, int cout, const int32_t* nbr,
                         int64_t nbr_stride, int K, int n_out, const float* scale, const float* shift,
                         const float* residual, int relu, float* out, cudaStream_t st) {
  const size_t smem = os_smem_bytes(NT);
  DGR_ENSURE_SMEM(spconv_os_kernel<NT>, smem);
  spconv_os_kernel<NT><<<(n_out + kTileM - 1) / kTileM, kThreadsOS, smem, st>>>(
      in_feat, cin, wt, cout, nbr, nbr_stride, K, n_out, scale, shift, residual, relu, out);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // namespace

extern "C" {

// 1 if dgr_spconv_os_fwd supports the shape (cin % 32 == 0, cout % 32 == 0, 32 <= cout <= 256)
int32_t dgr_spconv_os_supported(int32_t cin, int32_t cout) {
  return (cin >= 32 && cin % 32 == 0 && cout >= 32 && cout <= 256 && cout % 32 == 0) ? 1 : 0;
}

// Output-stationary tensor-core convolution with the fused layer epilogue:
//   out[j, :] = act((sum_kappa in_feat[nbr[kappa * nbr_stride + j], :] @ W[kappa]) * scale + shift + residual[j, :])
// nbr: dense neighbour table (dgr_kmap_dense; -1 = no neighbour), weight_t: the packed TF32
// hi | lo slabs of dgr_pack_weight_tf32 (3xTF32, fp32-accurate).  scale / shift / residual may be NULL; `out` need
// not be initialised and must not alias in_feat (it may alias nothing that is read).  Deterministic.
int32_t dgr_spconv_os_fwd(const float* in_feat, int32_t cin, const float* weight_t, int32_t cout, const int32_t* nbr,
                          int64_t nbr_stride, int32_t K, int64_t n_out, const float* scale, const float* shift,
                          const float* residual, int32_t relu, float* out, void* stream) {
  DGR_ARG_CHECK(dgr_spconv_os_supported(cin, cout), "shape not supported by the output-stationary kernel");
  DGR_ARG_CHECK((scale == nullptr) == (shift == nullptr), "scale and shift go together");
  DGR_ARG_CHECK(K >= 1 && nbr_stride >= n_out && n_out < (1ll << 31), "bad neighbour table extents");
  if (n_out == 0) return DGR_OK;
  auto launch = cout <= 32 ? launch_spconv_os<32> : cout <= 64 ? launch_spconv_os<64>
                : cout <= 128 ? launch_spconv_os<128> : launch_spconv_os<256>;
  return launch(in_feat, cin, weight_t, cout, nbr, nbr_stride, K, (int)n_out, scale, shift, residual, relu, out,
                (cudaStream_t)stream);
}

}  // extern "C"
