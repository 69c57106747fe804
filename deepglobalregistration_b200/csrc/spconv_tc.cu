// Sparse convolution forward on the Hopper tensor cores (wgmma, sm_90a).
//
// Same contract as dgr_spconv_fwd (gather -> per-offset sub-GEMM -> scatter-add over the
// (kappa, j)-sorted pair lists) with the sub-GEMM issued as wgmma.mma_async and the accumulator
// in registers:
//
//   * a tile is 128 pairs of one kernel offset: M = 128 rows split over two consumer warpgroups (64 rows
//     each), N = cout (16..256, padded to 32 / 64 / 128 / 256 with zero weight rows), K = cin in chunks of
//     one 128-byte swizzle row (32 TF32 or 64 FP16 channels);
//   * a CTA works through a run of consecutive tiles (spconv_ring::tile_run of them) as three warpgroups:
//     one producer, two consumers, coupled only by the full / empty mbarriers of a two-stage ring whose
//     position keeps running across tile boundaries (spconv_ring.h);
//   * the producer gathers the 128 input rows of a chunk (coalesced 16-byte pieces, 8 lanes per row, the
//     next chunk - of this tile or the next - in flight while the current one is stored), splits every
//     value into a "hi" part and a "lo" residual and stores both into shared memory in the canonical
//     K-major SWIZZLE_128B layout; one of its threads bulk-copies the weight slab of the chunk (TMA engine,
//     completion on the stage's full barrier).  It also parks the tile's out rows in shared memory.  While
//     the consumers drain the accumulators of tile t, the first chunks of tile t + 1 are already landing;
//   * each consumer warpgroup issues, per k-step, the three products hi*hi + lo*hi + hi*lo (3xTF32 or
//     3xFP16, fp32-accurate to ~2^-21 relative) and hands a stage back once the MMAs that read it retired;
//   * the epilogue scatter-adds the accumulator fragments with red.global.add.v2.f32.
//
// Weights come PRE-SPLIT and PRE-SWIZZLED (dgr_pack_weight_tf32 / dgr_pack_weight_f16, cached per layer
// by the host): per (offset, chunk) one contiguous slab holding the hi tile and the lo tile in
// shared-memory image order.
#include <stdlib.h>

#include "common.cuh"
#include "spconv_ring.h"
#include "tc_common.cuh"

namespace {

using namespace tc;
using namespace spconv_ring;

#define DGR_TRY_RC(expr)             \
  do {                              \
    int32_t rc__ = (expr);          \
    if (rc__ != DGR_OK) return rc__; \
  } while (0)

constexpr int kConsumerWarps = 8;        // two warpgroups: tile rows 0..63 and 64..127
constexpr int kProducerThreads = 128;    // the third warpgroup
constexpr int kThreadsTC = kConsumerWarps * 32 + kProducerThreads;
constexpr int kTileM = 128;
constexpr int kChunk = 32;               // TF32 channels per 128-byte row
constexpr int kATileBytes = kTileM * 128;
constexpr int kGatherRows = kTileM / (kProducerThreads / 8);   // rows per producer thread and chunk
static_assert(kMaxRun <= 32, "one warp lists the tiles of a run");

struct TileDesc {
  int kappa, p0, rows;
};

struct TcShared {
  unsigned long long full[kStages];     // gathered rows stored and weight slab landed (bulk-copy bytes)
  unsigned long long empty[kStages];    // every consumer warp has retired the MMAs that read the stage
  int n_run;                            // non-empty tiles of the run
  TileDesc tiles[kMaxRun];
  int out_rows[kIdxSlots][kTileM];      // out row of every pair of a tile, -1 beyond the tile's rows
};

// shared-memory bytes of spconv_tc_kernel<NT, *>
constexpr size_t tc_smem_bytes(int nt) {
  return sizeof(TcShared) + 1024 + (size_t)kStages * (2 * kATileBytes + 2 * nt * 128);
}

// NT >= 128: one CTA per SM, the register file re-divided between producer and consumers (setmaxnreg);
// narrower accumulators leave room for two CTAs, whose 80 registers the TF32 producer fits and the FP16 one
// (twice the rows per chunk) does not
constexpr int tc_min_ctas(int nt, bool f16) { return nt >= 128 || f16 ? 1 : 2; }
constexpr int kProducerRegs = 104, kConsumerRegs = 200;     // 128 * 104 + 256 * 200 = 384 * 168

// kF16: 3xFP16 instead of 3xTF32 (64 channels per 128-byte stage row; `wt` then holds the fp16 slabs of
// dgr_pack_weight_f16, amax_in the input tensor's absolute maximum, w_inv_scale the inverse of the weight scale).
// CTA b owns tiles [b * run, min((b + 1) * run, n_tiles)).
template <int NT, bool kF16, int kPasses>
__global__ void __launch_bounds__(kThreadsTC, tc_min_ctas(NT, kF16))
spconv_tc_kernel(const float* __restrict__ in_feat, int cin, const unsigned char* __restrict__ wt, int cout,
                 const int32_t* __restrict__ in_idx, const int32_t* __restrict__ out_idx,
                 const int32_t* __restrict__ kofs, const int32_t* __restrict__ tile_k,
                 const int32_t* __restrict__ tile_start, int n_tiles, int run, const float* __restrict__ amax_in,
                 const float* __restrict__ w_inv_scale, float* __restrict__ out) {
  constexpr int kCh = kF16 ? 64 : kChunk;        // channels per stage (one 128-byte swizzle row)
  constexpr int kV = kF16 ? 2 : 1;               // float4 loads per (thread, row, chunk)
  // a producer thread keeps eight float4 in flight: a whole chunk of its rows in TF32, half of them in FP16
  constexpr int kBatches = kV, kBatchRows = kGatherRows / kBatches;
  constexpr int kBTileBytes = NT * 128;          // B tile in shared memory: rows >= cout stay zero
  constexpr int kStageBytes = 2 * kATileBytes + 2 * kBTileBytes;
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  TcShared& sh = *reinterpret_cast<TcShared*>(smem_dyn);
  // stage buffers start at the next 1024-byte boundary (SWIZZLE_128B atom alignment)
  unsigned char* stage0 = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_dyn) + sizeof(TcShared) + 1023) & ~(uintptr_t)1023);
  // warp index through a shuffle: the compiler then knows it is warp-uniform, as the wgmma paths need
  const int t = threadIdx.x, warp = __shfl_sync(0xffffffffu, t >> 5, 0), lane = t & 31;
  const int n_chunks = cin / kCh;
  const uint32_t b_tile_bytes = (uint32_t)cout * 128;   // one tile (hi or lo) of the packed slab
  const uint32_t slab_bytes = 2 * b_tile_bytes;
  const uint32_t full0 = smem_u32(&sh.full[0]), empty0 = smem_u32(&sh.empty[0]);

  if (t == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full0 + 8 * s, kProducerThreads + 1);     // every producer thread + the slab's expect-tx arrival
      mbar_init(empty0 + 8 * s, kConsumerWarps);
    }
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
  if (warp == 0) {     // the run's tiles, without the padding tiles (rows <= 0) of a paired list
    const int tile = blockIdx.x * run + lane;
    TileDesc d = {0, 0, 0};
    if (lane < run && tile < n_tiles) {
      d.kappa = tile_k[tile];
      d.p0 = tile_start[tile];
      d.rows = min(kTileM, kofs[d.kappa + 1] - d.p0);
    }
    const unsigned live = __ballot_sync(0xffffffffu, d.rows > 0);
    if (d.rows > 0) sh.tiles[__popc(live & ((1u << lane) - 1u))] = d;
    if (lane == 0) sh.n_run = __popc(live);
  }
  __syncthreads();     // the last block-wide barrier: the roles split here
  const int n_run = sh.n_run;
  if (n_run == 0) return;

  if (warp >= kConsumerWarps) {     // producer warpgroup
    if (NT >= 128) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    // gather: 8 lanes cover one 128-byte row; 16 row groups, rows rgrp + 16 i
    const int pt = t - kConsumerWarps * 32, piece = pt & 7, rgrp = pt >> 3;
    const uint32_t a_off = (uint32_t)(rgrp * 128 + ((piece ^ (rgrp & 7)) << 4));   // + i * 2048
    const float sx = kF16 ? f16_scale_for(__ldg(amax_in)) : 1.f;
    // in rows of the thread's kGatherRows rows and the out row of pair `pt`, of run tile ti
    auto load_idx = [&](int ti, int (&src)[kGatherRows], int& oj) {
      const TileDesc d = sh.tiles[ti < n_run ? ti : 0];
      const int rows = ti < n_run ? d.rows : 0;
#pragma unroll
      for (int i = 0; i < kGatherRows; ++i) {
        const int r = i * 16 + rgrp;
        src[i] = r < rows ? __ldg(in_idx + d.p0 + r) : -1;
      }
      oj = pt < rows ? __ldg(out_idx + d.p0 + pt) : -1;
    };
    int src[kGatherRows], src_next[kGatherRows], oj, oj_next;
    float4 v[kBatchRows][kV];
    // rows h * kBatchRows ... of chunk c of the tile `src` belongs to
    auto load_a = [&](int c, int h) {
#pragma unroll
      for (int i = 0; i < kBatchRows; ++i)
#pragma unroll
        for (int u = 0; u < kV; ++u) {
          const int row = src[h * kBatchRows + i];
          v[i][u] = row >= 0 ? __ldg(reinterpret_cast<const float4*>(in_feat + (size_t)row * cin + c * kCh +
                                                                      piece * (4 * kV) + 4 * u))
                             : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    load_idx(0, src, oj);
    load_idx(1, src_next, oj_next);     // indices stay one tile ahead of the rows they address
    load_a(0, 0);
    unsigned g = 0;                     // chunks of the run so far: the ring position
    for (int ti = 0; ti < n_run; ++ti) {
      const unsigned char* slab = wt + (size_t)sh.tiles[ti].kappa * n_chunks * slab_bytes;
      for (int c = 0; c < n_chunks; ++c, ++g) {
        const int s = stage_of(g);
        unsigned char* a_hi = stage0 + (size_t)s * kStageBytes;
        unsigned char* a_lo = a_hi + kATileBytes;
        unsigned char* b_hi = a_lo + kATileBytes;
        if (g >= kStages) mbar_wait(empty0 + 8 * s, empty_parity(g));
        if (pt == 0) {
          const unsigned char* bsrc = slab + (size_t)c * slab_bytes;
          mbar_arrive_expect_tx(full0 + 8 * s, kPasses == 3 ? slab_bytes : b_tile_bytes);
          bulk_g2s(smem_u32(b_hi), bsrc, b_tile_bytes, full0 + 8 * s);
          if (kPasses == 3) bulk_g2s(smem_u32(b_hi + kBTileBytes), bsrc + b_tile_bytes, b_tile_bytes, full0 + 8 * s);
        }
        if (c == 0) sh.out_rows[idx_slot(ti)][pt] = oj;
#pragma unroll
        for (int h = 0; h < kBatches; ++h) {
#pragma unroll
          for (int i = 0; i < kBatchRows; ++i) {
            const uint32_t off = a_off + (h * kBatchRows + i) * 2048;
            if (kF16) split_store_f16(v[i][0], v[i][kV - 1], sx, a_hi, a_lo, off);
            else split_store(v[i][0], a_hi, a_lo, off);
          }
          // the next rows - of this chunk, the next chunk or the next tile - are in flight while these multiply
          if (h + 1 < kBatches) {
            load_a(c, h + 1);
          } else if (c + 1 < n_chunks) {
            load_a(c + 1, 0);
          } else if (ti + 1 < n_run) {
#pragma unroll
            for (int i = 0; i < kGatherRows; ++i) src[i] = src_next[i];
            oj = oj_next;
            load_a(0, 0);
            load_idx(ti + 2, src_next, oj_next);
          }
        }
        fence_proxy_async();
        mbar_arrive(full0 + 8 * s);
      }
    }
    return;
  }

  if (NT >= 128) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
  // consumers: thread holds rows r0 and r0 + 8 of the tile, two adjacent columns per 8-column group
  const int wg = warp >> 2;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  // kF16: the accumulator holds (sx * x) . (sw * w); both scales are powers of two, undone exactly in the epilogue
  const float inv = kF16 ? __ldg(w_inv_scale) / f16_scale_for(__ldg(amax_in)) : 1.f;
  auto release = [&](unsigned gq) {
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * stage_of(gq));
  };
  unsigned g = 0;
  for (int ti = 0; ti < n_run; ++ti) {
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    for (int c = 0; c < n_chunks; ++c, ++g) {
      const uint32_t a_hi = smem_u32(stage0 + (size_t)stage_of(g) * kStageBytes);
      const uint32_t b_hi = a_hi + 2 * kATileBytes;
      mbar_wait(full0 + 8 * stage_of(g), full_parity(g));
      wgmma_fence();
      const uint32_t a0 = a_hi + wg * (kATileBytes / 2);
      mma_chunk<NT, kF16, kPasses>(acc, a0, a0 + kATileBytes, b_hi, b_hi + kBTileBytes);
      wgmma_commit();
      wgmma_wait<1>();
      if (c > 0) release(g - 1);          // the MMAs of the previous chunk have retired: its stage is free
    }
    wgmma_wait<0>();
    fence_acc(acc);
    release(g - 1);

    const int* rows_of = sh.out_rows[idx_slot(ti)];
    const int j0 = rows_of[r0], j1 = rows_of[r0 + 8];
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
}

// CTAs of the kernel a device holds at once (SMs x CTAs per SM); 0 if the query fails
template <int NT, bool kF16, int kPasses>
int tc_resident_ctas(size_t smem) {
  int dev = 0, sms = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, spconv_tc_kernel<NT, kF16, kPasses>, kThreadsTC, smem) !=
          cudaSuccess)
    return 0;
  return sms * per_sm;
}

// one instantiation per kernel: DGR_ENSURE_SMEM keeps its attribute state per call site
template <int NT, bool kF16, int kPasses>
int32_t launch_spconv_tc(const float* in_feat, int cin, const void* wt, int cout, const int32_t* in_idx,
                         const int32_t* out_idx, const int32_t* kofs, const int32_t* tile_k, const int32_t* tile_start,
                         int n_tiles, const float* amax_in, const float* w_inv_scale, float* out, cudaStream_t st) {
  const size_t smem = tc_smem_bytes(NT);
  DGR_ENSURE_SMEM((spconv_tc_kernel<NT, kF16, kPasses>), smem);
  static const int resident = tc_resident_ctas<NT, kF16, kPasses>(smem);
  if (resident <= 0) {
    dgr_set_error("spconv_tc_kernel does not fit the device");
    return DGR_ERR_CUDA;
  }
  const int run = tile_run(n_tiles, resident);
  spconv_tc_kernel<NT, kF16, kPasses><<<(n_tiles + run - 1) / run, kThreadsTC, smem, st>>>(
      in_feat, cin, (const unsigned char*)wt, cout, in_idx, out_idx, kofs, tile_k, tile_start, n_tiles, run, amax_in,
      w_inv_scale, out);
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
