// Exact feature nearest neighbour with a tensor-core pre-filter (C = 32 or 64).
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
//           arithmetic of the fp32 kernel.  The row result is the lexicographic minimum of
//           (bits of the root, column) over the candidates, so the order in which they are evaluated
//           does not change it.
//
// E_i bounds the error of d~2: operands are rounded to TF32 (relative 2^-11 each), so a dot
// product is off by at most 2^-10 |a||b| (+ accumulation slack), and d~2 by twice that.  The
// true nearest neighbour j* satisfies d~2(j*) <= d2(j*) + E <= d2(j) + E <= d~2(j) + 2E for
// every j, hence it is always among the candidates and the result equals the fp32 kernel's.
//
// Schedule (four launches):
//   prep    F0 and F1 are written once, TF32-rounded, as 128-row tiles in the K-major SWIZZLE_128B
//           shared-memory image (tail rows zero), with |a|^2 per F0 row, 0.5 |b|^2 per F1 column
//           (+inf past n1, so tail columns are never a minimum or a candidate) and max |b|^2 per
//           column tile; the row minima and packed results are reset.
//   sweeps  one persistent kernel per pass, grid = SMs x resident CTAs.  CTA b takes the b-th
//           contiguous share of the row-major (row tile, column tile) sequence; a work item is the part
//           of that share inside one row tile.  The assignment is static, so every run makes the same
//           schedule.  One producer thread streams the B tiles and their 0.5 |b|^2 through a ring of
//           kStages stages with cp.async.bulk (full / empty mbarriers) and the A tile once per item
//           (double-buffered).  Two consumer warpgroups own 64 rows each and double-buffer the
//           accumulator over pairs of tiles: the MMAs of tiles t and t + 1 are issued together and the
//           epilogue of t runs while t + 1 multiplies.  No MMA stays in flight across the loop's back
//           edge: ptxas then serialises every wgmma (C7514).  The epilogue of t + 1 overlaps the other
//           warpgroup's MMAs instead; the two warpgroups only share the ring.  Pass 2 computes
//           its thresholds in its prologue, takes a warp-uniform fast path through tiles in which no row
//           of the warp has a candidate, and otherwise queues the candidates per warp in shared memory,
//           evaluated one lane per candidate.  The threshold is not tightened as exact distances arrive:
//           the bench pair's features have about 1.3 candidates per row, so there is nothing to save.
//   unpack  packed (root, column) -> idx, dist.
#include <algorithm>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int kRows = 128;                   // rows of an A tile = columns of a B tile
constexpr int kTileBytes = kRows * 128;      // one 32-channel chunk of a tile
constexpr int kTileFloats = kTileBytes / 4;
constexpr int kConsumerWarps = 8;            // two warpgroups: A-tile rows 0..63 and 64..127
constexpr int kThreads = kConsumerWarps * 32 + 128;  // + the producer warpgroup (one thread issues the copies)
constexpr int kQueue = 256;                  // pass-2 candidate queue per consumer warp
constexpr float kInf = __builtin_huge_valf();

template <int C>
struct KnnCfg {
  static constexpr int kChunks = C / 32;
  static constexpr int kStages = C == 32 ? 4 : 3;
  static constexpr int kOpBytes = kChunks * kTileBytes;   // one A or B tile, every chunk
  // A double buffer, B ring, 0.5 |b|^2 ring, candidate queues, per-row best, mbarriers, max |b|^2
  static constexpr size_t kSmem = 1024 + (size_t)(2 + kStages) * kOpBytes + kStages * kRows * 4 +
                                  kConsumerWarps * (kQueue + 16) * 8 + (2 * kStages + 4) * 8 + 16;
};

// workspace carve-up; every part starts on a 16-byte boundary (bulk-copy sources)
struct KnnWs {
  float* a_img;        // [row_tiles][chunks][128 x 128 B] TF32 image of F0
  float* b_img;        // [col_tiles][chunks][128 x 128 B] TF32 image of F1
  float* na2;          // [n0] |a|^2
  unsigned* rowmin;    // [n0] bits of max(m~_i, 0) (pass 1)
  float* nbh;          // [col_tiles * 128] 0.5 |b|^2, +inf past n1
  float* bmax;         // [col_tiles] max |b|^2 of the tile's columns
};
inline int64_t up4(int64_t x) { return (x + 3) & ~(int64_t)3; }
inline int64_t ceil_tiles(int64_t n) { return (n + kRows - 1) / kRows; }
// float offsets of the parts: a_img, b_img, na2, rowmin, nbh, bmax, end
void ws_offsets(int64_t n0, int64_t n1, int c, int64_t (&o)[7]) {
  const int64_t tile = (int64_t)(c / 32) * kTileFloats;
  o[0] = 0;
  o[1] = o[0] + ceil_tiles(n0) * tile;
  o[2] = o[1] + ceil_tiles(n1) * tile;
  o[3] = o[2] + up4(n0);
  o[4] = o[3] + up4(n0);
  o[5] = o[4] + ceil_tiles(n1) * kRows;
  o[6] = o[5] + up4(ceil_tiles(n1));
}
KnnWs carve_ws(float* ws, int64_t n0, int64_t n1, int c) {
  int64_t o[7];
  ws_offsets(n0, n1, c, o);
  return KnnWs{ws + o[0], ws + o[1], ws + o[2], reinterpret_cast<unsigned*>(ws + o[3]), ws + o[4], ws + o[5]};
}

// thr_i = m~_i + 2 E_i with E_i = 2 * (dot-product error bound): operands rounded to TF32,
// |a.b error| <= 2^-10 * 1.25 |a||b| (+ accumulation slack), plus the slack of the fp32 norms.
__device__ __forceinline__ float knn_error_bound(float na, float nb) {
  return (0.0009765625f * 1.25f + 4e-5f) * na * nb + 1e-6f * (na + nb) * (na + nb) + 1e-7f;
}

// One block per 128-row tile: blocks [0, row_tiles) take F0, the rest F1.  8 lanes per row.
template <int C>
__global__ void __launch_bounds__(kRows * 8)
knn_prep_kernel(const float* __restrict__ f0, int n0, const float* __restrict__ f1, int n1, int row_tiles, KnnWs w,
                unsigned long long* __restrict__ packed) {
  constexpr int kChunks = C / 32;
  const bool is_a = (int)blockIdx.x < row_tiles;
  const int tile = is_a ? blockIdx.x : blockIdx.x - row_tiles;
  const float* f = is_a ? f0 : f1;
  const int n = is_a ? n0 : n1;
  const int r = threadIdx.x >> 3, sub = threadIdx.x & 7;
  const int row = tile * kRows + r;
  const bool valid = row < n;
  // |x|^2: lane `sub` sums channels sub, sub + 8, ... in order, then a butterfly over the 8 lanes
  float s = 0.f;
  if (valid)
    for (int k = sub; k < C; k += 8) {
      const float v = f[(size_t)row * C + k];
      s = fmaf(v, v, s);
    }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  float* img = (is_a ? w.a_img : w.b_img) + (size_t)tile * kChunks * kTileFloats;
#pragma unroll
  for (int ch = 0; ch < kChunks; ++ch) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid) v = __ldg(reinterpret_cast<const float4*>(f + (size_t)row * C + ch * 32 + sub * 4));
    v.x = tf32_round(v.x); v.y = tf32_round(v.y); v.z = tf32_round(v.z); v.w = tf32_round(v.w);
    *reinterpret_cast<float4*>(img + ch * kTileFloats + r * 32 + ((sub ^ (r & 7)) << 2)) = v;
  }
  if (is_a) {
    if (valid && sub == 0) {
      w.na2[row] = s;
      w.rowmin[row] = 0x7f800000u;
      packed[row] = ~0ull;
    }
    return;
  }
  if (sub == 0) w.nbh[row] = valid ? 0.5f * s : kInf;
  __shared__ float wmax[kRows * 8 / 32];
  float m = valid ? s : 0.f;
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = wmax[threadIdx.x];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
    if (threadIdx.x == 0) w.bmax[tile] = m;
  }
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// exact reference arithmetic for one (row, column) pair, as in knn.cu
template <int C>
__device__ __forceinline__ unsigned long long knn_exact_key(const float* __restrict__ f0, const float* __restrict__ f1,
                                                            int gi, int j) {
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
  return ((unsigned long long)__float_as_uint(sqrtf(d2 + 1e-7f)) << 32) | (unsigned)j;
}

// one work item: row tile rt, column tiles [ct0, ct1)
struct Item {
  int rt, ct0, ct1;
};
__device__ __forceinline__ Item item_at(long long k, long long k_end, int col_tiles) {
  Item it;
  it.rt = (int)(k / col_tiles);
  it.ct0 = (int)(k - (long long)it.rt * col_tiles);
  it.ct1 = (int)min((long long)col_tiles, it.ct0 + (k_end - k));
  return it;
}

template <int C, int PASS>
__global__ void __launch_bounds__(kThreads, 1)
knn_sweep_kernel(const float* __restrict__ f0, int n0, const float* __restrict__ f1, int row_tiles, int col_tiles,
                 KnnWs w, unsigned long long* __restrict__ packed) {
  using K = KnnCfg<C>;
  constexpr int kStages = K::kStages, kOpBytes = K::kOpBytes;
  extern __shared__ __align__(16) unsigned char smem_dyn[];
  unsigned char* a_buf = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) &
                                                          ~(uintptr_t)1023);
  unsigned char* b_buf = a_buf + 2 * kOpBytes;
  float* nb_buf = reinterpret_cast<float*>(b_buf + kStages * kOpBytes);                    // [kStages][128]
  unsigned long long* queue = reinterpret_cast<unsigned long long*>(nb_buf + kStages * kRows);  // [8][kQueue]
  unsigned long long* best = queue + kConsumerWarps * kQueue;                              // [8][16]
  uint64_t* bars = reinterpret_cast<uint64_t*>(best + kConsumerWarps * 16);
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * kStages;
  const uint32_t a_full0 = empty0 + 8 * kStages, a_empty0 = a_full0 + 16;
  float* nbmax_sh = reinterpret_cast<float*>(bars + 2 * kStages + 4);

  // warp index through a shuffle: the compiler then knows it is warp-uniform, as the wgmma paths need
  const int t = threadIdx.x, warp = __shfl_sync(0xffffffffu, t >> 5, 0), lane = t & 31;
  const long long total = (long long)row_tiles * col_tiles;
  const long long k_begin = total * blockIdx.x / gridDim.x, k_end = total * (blockIdx.x + 1) / gridDim.x;

  if (t == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, kConsumerWarps);
    }
    for (int p = 0; p < 2; ++p) {
      mbar_init(a_full0 + 8 * p, 1);
      mbar_init(a_empty0 + 8 * p, kConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (PASS == 2 && warp == 0) {     // max |b|^2 over every column: the error bound's |b|
    float m = 0.f;
    for (int i = lane; i < col_tiles; i += 32) m = fmaxf(m, w.bmax[i]);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
    if (lane == 0) *nbmax_sh = m;
  }
  if (PASS == 2 && t < kConsumerWarps * 16) best[t] = ~0ull;
  __syncthreads();     // the last block-wide barrier: the roles split here

  if (warp >= kConsumerWarps) {     // producer warpgroup
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kConsumerWarps && lane == 0) {
      long long kt = 0;
      int it = 0;
      for (long long k = k_begin; k < k_end; ++it) {
        const Item item = item_at(k, k_end, col_tiles);
        const int p = it & 1;
        if (it >= 2) mbar_wait(a_empty0 + 8 * p, ((it >> 1) - 1) & 1);
        mbar_arrive_expect_tx(a_full0 + 8 * p, kOpBytes);
        bulk_g2s(smem_u32(a_buf + p * kOpBytes), w.a_img + (size_t)item.rt * (kOpBytes / 4), kOpBytes, a_full0 + 8 * p);
        for (int ct = item.ct0; ct < item.ct1; ++ct, ++kt) {
          const int s = (int)(kt % kStages);
          if (kt >= kStages) mbar_wait(empty0 + 8 * s, (uint32_t)((kt / kStages - 1) & 1));
          mbar_arrive_expect_tx(full0 + 8 * s, kOpBytes + kRows * 4);
          bulk_g2s(smem_u32(b_buf + s * kOpBytes), w.b_img + (size_t)ct * (kOpBytes / 4), kOpBytes, full0 + 8 * s);
          bulk_g2s(smem_u32(nb_buf + s * kRows), w.nbh + (size_t)ct * kRows, kRows * 4, full0 + 8 * s);
        }
        k += item.ct1 - item.ct0;
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // consumers: thread holds rows rw and rw + 8 of its warp's 16, two adjacent columns of every 8-column group
  const int wg = warp >> 2;
  const int rw = lane >> 2;
  const int row_in_tile = wg * 64 + (warp & 3) * 16;    // first of the warp's 16 rows
  const float nb_root = PASS == 2 ? sqrtf(*nbmax_sh) : 0.f;
  unsigned long long* q = queue + warp * kQueue;
  unsigned long long* bw = best + warp * 16;
  int qn = 0;     // queued candidates (warp-uniform)

  // evaluate every queued candidate, one lane each; the row keeps the (root, column) minimum
  auto drain = [&](int row0) {
    __syncwarp();
    for (int b = 0; b < qn; b += 32)
      if (b + lane < qn) {
        const unsigned long long e = q[b + lane];
        const int r = (int)(e >> 32), j = (int)(unsigned)e;
        atomicMin(bw + r, knn_exact_key<C>(f0, f1, row0 + r, j));
      }
    qn = 0;
    __syncwarp();
  };

  long long kt = 0;
  int it = 0;
  for (long long k = k_begin; k < k_end; ++it) {
    const Item item = item_at(k, k_end, col_tiles);
    const int p = it & 1;
    const int row0 = item.rt * kRows + row_in_tile;    // global row of the warp's row 0
    int gi[2];
    float th[2], rmin[2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      gi[h] = row0 + rw + 8 * h;
      th[h] = -kInf;
      if (PASS == 2 && gi[h] < n0) {
        const float na2 = w.na2[gi[h]];
        const float e = knn_error_bound(sqrtf(na2), nb_root);
        // in the epilogue's units: candidates satisfy (0.5 |b|^2 - a.b) <= th
        th[h] = 0.5f * (__uint_as_float(w.rowmin[gi[h]]) + 4.f * e - na2);
      }
      rmin[h][0] = rmin[h][1] = kInf;     // min over columns of 0.5 |b|^2 - a.b
    }
    mbar_wait(a_full0 + 8 * p, (it >> 1) & 1);
    const uint32_t a_s = smem_u32(a_buf + p * kOpBytes) + wg * (kTileBytes / 2);

    auto issue = [&](float(&acc)[64], long long kq) {
      const int s = (int)(kq % kStages);
      mbar_wait(full0 + 8 * s, (uint32_t)((kq / kStages) & 1));
      const uint32_t b_s = smem_u32(b_buf + s * kOpBytes);
      wgmma_fence();
#pragma unroll
      for (int ch = 0; ch < K::kChunks; ++ch)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          Wgmma<128, false>::mma(acc, wgmma_desc(a_s + ch * kTileBytes + ks * 32),
                                 wgmma_desc(b_s + ch * kTileBytes + ks * 32), (ch | ks) != 0);
      wgmma_commit();
    };
    auto epilogue = [&](float(&acc)[64], long long kq, int ct) {
      fence_acc(acc);
      const int s = (int)(kq % kStages);
      const float* nbs = nb_buf + s * kRows + 2 * (lane & 3);
      float tmin[2][2] = {{kInf, kInf}, {kInf, kInf}};
#pragma unroll
      for (int i = 0; i < kRows / 8; ++i) {
        const float2 nb = *reinterpret_cast<const float2*>(nbs + 8 * i);
#pragma unroll
        for (int h = 0; h < 2; ++h)
          tmin[h][i & 1] = fminf(tmin[h][i & 1], fminf(nb.x - acc[4 * i + 2 * h], nb.y - acc[4 * i + 2 * h + 1]));
      }
      if (PASS == 1) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          rmin[h][0] = fminf(rmin[h][0], tmin[h][0]);
          rmin[h][1] = fminf(rmin[h][1], tmin[h][1]);
        }
      } else if (__any_sync(0xffffffffu, fminf(tmin[0][0], tmin[0][1]) <= th[0] ||
                                             fminf(tmin[1][0], tmin[1][1]) <= th[1])) {
        // some row of the warp has a candidate in this tile: queue them all.  Bit 4 i + 2 h + e of the mask is
        // acc[4 i + 2 h + e]; the queueing loop below is rolled (this path is cold: it must stay small)
        unsigned long long mask = 0;
#pragma unroll
        for (int i = 0; i < kRows / 8; ++i) {
          const float2 nb = *reinterpret_cast<const float2*>(nbs + 8 * i);
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if ((e ? nb.y : nb.x) - acc[4 * i + 2 * h + e] <= th[h]) mask |= 1ull << (4 * i + 2 * h + e);
        }
        const int cnt = __popcll(mask);
        int pos = cnt;     // inclusive prefix sum over the lanes, then exclusive
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, pos, d);
          if (lane >= d) pos += y;
        }
        const int total = __shfl_sync(0xffffffffu, pos, 31);
        pos -= cnt;
        if (qn + total > kQueue) drain(row0);
        // rounds of at most kQueue entries: more than that only when most of the tile's pairs are candidates
        for (int base = 0; base < total; base += kQueue) {
          unsigned long long m = mask;
          for (int idx = pos; m != 0; ++idx, m &= m - 1) {
            const int b = __ffsll((long long)m) - 1;
            if (idx >= base && idx < base + kQueue)
              q[qn + idx - base] = ((unsigned long long)(rw + 8 * ((b >> 1) & 1)) << 32) |
                                   (unsigned)(ct * kRows + 8 * (b >> 2) + 2 * (lane & 3) + (b & 1));
          }
          qn += min(kQueue, total - base);
          if (base + kQueue < total) drain(row0);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);
    };

    float acc0[64], acc1[64];
    const int n = item.ct1 - item.ct0;
    for (int i = 0; i < n; i += 2) {
      issue(acc0, kt + i);
      if (i + 1 < n) {
        issue(acc1, kt + i + 1);
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      epilogue(acc0, kt + i, item.ct0 + i);
      if (i + 1 == n) break;
      wgmma_wait<0>();
      epilogue(acc1, kt + i + 1, item.ct0 + i + 1);
    }
    wgmma_wait<0>();     // nothing is pending; ptxas cannot tell from the loop and would add waits of its own
    __syncwarp();
    if (lane == 0) mbar_arrive(a_empty0 + 8 * p);     // every MMA of the item has completed
    kt += n;
    k += n;

    if (PASS == 1) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // the four lanes of a quad share the row
        float m = fminf(rmin[h][0], rmin[h][1]);
        m = fminf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fminf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        if (gi[h] < n0 && (lane & 3) == 0)
          atomicMin(w.rowmin + gi[h], __float_as_uint(fmaxf(fmaf(2.f, m, w.na2[gi[h]]), 0.f)));
      }
    } else {
      if (qn > 0) drain(row0);
      if (lane < 16) {
        const unsigned long long v = bw[lane];
        if (v != ~0ull && row0 + lane < n0) atomicMin(packed + row0 + lane, v);
        bw[lane] = ~0ull;
      }
      __syncwarp();
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
int32_t launch_knn_tc(const float* f0, int64_t n0, const float* f1, int64_t n1, const KnnWs& w,
                      unsigned long long* packed, cudaStream_t st) {
  constexpr size_t smem = KnnCfg<C>::kSmem;
  DGR_ENSURE_SMEM((knn_sweep_kernel<C, 1>), smem);
  DGR_ENSURE_SMEM((knn_sweep_kernel<C, 2>), smem);
  int dev = 0, sms = 0, per_sm1 = 0, per_sm2 = 0;
  DGR_CUDA_CHECK(cudaGetDevice(&dev));
  DGR_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  DGR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm1, knn_sweep_kernel<C, 1>, kThreads, smem));
  DGR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, knn_sweep_kernel<C, 2>, kThreads, smem));
  const int row_tiles = (int)ceil_tiles(n0), col_tiles = (int)ceil_tiles(n1);
  const long long total = (long long)row_tiles * col_tiles;
  // persistent: one CTA per resident slot, never more CTAs than (row tile, column tile) pairs
  const int grid = (int)std::min<long long>(total, (long long)sms * std::max(1, std::min(per_sm1, per_sm2)));
  knn_prep_kernel<C><<<row_tiles + col_tiles, kRows * 8, 0, st>>>(f0, (int)n0, f1, (int)n1, row_tiles, w, packed);
  knn_sweep_kernel<C, 1><<<grid, kThreads, smem, st>>>(f0, (int)n0, f1, row_tiles, col_tiles, w, packed);
  knn_sweep_kernel<C, 2><<<grid, kThreads, smem, st>>>(f0, (int)n0, f1, row_tiles, col_tiles, w, packed);
  return DGR_OK;
}

}  // namespace

extern "C" {

// floats of workspace dgr_knn_top1_tc needs at a supported c: both operand images, the norms and the row minima
int64_t dgr_knn_tc_ws_elems(int64_t n0, int64_t n1, int32_t c) {
  int64_t o[7];
  ws_offsets(n0, n1, c, o);
  return o[6];
}

// 1 if the tensor-core pre-filter supports the channel count
int32_t dgr_knn_tc_supported(int32_t c) { return (c == 32 || c == 64) ? 1 : 0; }

// Same result as dgr_knn_top1 (bit-identical indices and distances), two wgmma sweeps
// plus exact fp32 evaluation of the few candidates per row.  ws: dgr_knn_tc_ws_elems floats.
int32_t dgr_knn_top1_tc(const float* f0, int64_t n0, const float* f1, int64_t n1, int32_t c,
                        uint64_t* packed_ws, float* ws, int32_t* idx, float* dist, void* stream) {
  DGR_ARG_CHECK(dgr_knn_tc_supported(c), "channel count not supported by the tensor-core kNN");
  DGR_ARG_CHECK(n1 >= 1 || n0 == 0, "F1 must not be empty");
  DGR_ARG_CHECK(n0 < (1ll << 31) && n1 < (1ll << 31), "too many rows");
  DGR_ARG_CHECK(((uintptr_t)ws & 15) == 0, "workspace must be 16-byte aligned");
  if (n0 == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const KnnWs w = carve_ws(ws, n0, n1, c);
  unsigned long long* packed = reinterpret_cast<unsigned long long*>(packed_ws);
  int32_t rc = (c == 32) ? launch_knn_tc<32>(f0, n0, f1, n1, w, packed, st)
                         : launch_knn_tc<64>(f0, n0, f1, n1, w, packed, st);
  if (rc != DGR_OK) return rc;
  knn_tc_unpack_kernel<<<dgr_blocks(n0, 256), 256, 0, st>>>(packed, n0, idx, dist);
  dgr_note_launches(4);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
