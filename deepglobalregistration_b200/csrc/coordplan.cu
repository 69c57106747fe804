// Coordinate planning with DEVICE-SIDE row counts: the integer work of one network forward
// (coarse coordinate maps, kernel maps) enqueued without a single host round trip.  The coarse
// maps and the table of the input rows come from the first-occurrence pass in coords.cu.
//
// Every kernel takes (n_max, n_dev): a host-side upper bound that sizes buffers and grids,
// and a device pointer to the actual count that the kernels read (NULL: n_max is the count,
// as on the operator path of me/coords.py).  The native executor (exec.cu) enqueues the whole
// coordinate phase of a network, then reads ONE small meta block (rows per level, pairs /
// tiles per map, key overflow) and launches the fill + convolution phase.
//
// Kernel maps do not go through a dense neighbour table nbr[K][N_out] (150 MB per 6-D map,
// 99.7 % of it -1): the probe pass stores one BIT per (offset, output row) - a ballot word
// per (offset, warp of 32 rows), 32x smaller - together with per-(offset, block) hit counts;
// after an exclusive scan the fill pass walks the set bits, re-probes those (hits only) and
// writes the (kappa, j)-sorted pair lists, bit-identical to the oracle's buckets.  A dense
// table is built (dgr_kmap_dense) only where a convolution reads one.
// Misses, 96-99.7 % of all probes of a 6-D map, are answered by a blocked Bloom filter of the
// input table held in SHARED memory (one 32-bit word holds both bits of a key: one
// shared-memory load per probe) instead of an L2 round trip.
//
// Replaces the MinkowskiEngine coordinate manager / kernel-map builder behind
// model/residual_block.py:31-80 and model/resunet.py:598-649 (reference call sites); the pair
// list semantics are those frozen in oracle/sparse_ops.py.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kCntWords = 256;        // mask words per counted block of a kernel map (one fill block, one word per thread)
constexpr int kProbeThreads = 512;    // 16 warps = 512 output rows per probe block

// ---------------------------------------------------------------------------------------
// voxel compaction of a scan pair (device count of kept points)
// ---------------------------------------------------------------------------------------
template <typename T0, typename T1>
__global__ void compact_voxels_kernel(const int32_t* __restrict__ raw, const int32_t* __restrict__ sel,
                                      const int32_t* __restrict__ n_unique, int64_t n_raw0,
                                      const T0* __restrict__ xyz0, const T1* __restrict__ xyz1, double cell,
                                      int32_t* __restrict__ coords, float* __restrict__ xyz,
                                      int32_t* __restrict__ counts) {
  const int n = n_unique[0];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    // sel is ascending: rows of cloud 0 come first; N0 = lower_bound(sel, n_raw0)
    int lo = 0, hi = n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sel[mid] < n_raw0) lo = mid + 1; else hi = mid;
    }
    counts[0] = n;
    counts[1] = lo;
    counts[2] = n - lo;
    counts[3] = n_unique[1];     // key-overflow flag
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = sel[i];
    const int4 k = reinterpret_cast<const int4*>(raw)[r];
    reinterpret_cast<int4*>(coords)[i] = k;
    double x, y, z;
    if (r < n_raw0) {
      x = (double)xyz0[3 * r]; y = (double)xyz0[3 * r + 1]; z = (double)xyz0[3 * r + 2];
    } else {
      const int64_t q = r - n_raw0;
      x = (double)xyz1[3 * q]; y = (double)xyz1[3 * q + 1]; z = (double)xyz1[3 * q + 2];
    }
    // the rows the pair's ICP searches its voxel hash with: in the cells they are keyed under (DESIGN.md §3)
    xyz[3 * i] = dgr_float32_in_cell(x, k.y, cell);
    xyz[3 * i + 1] = dgr_float32_in_cell(y, k.z, cell);
    xyz[3 * i + 2] = dgr_float32_in_cell(z, k.w, cell);
  }
}

// ---------------------------------------------------------------------------------------
// blocked Bloom filter of a table: both bits of a key live in ONE 32-bit word
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t bloom_mix(uint64_t key) {
  uint32_t h = (uint32_t)key ^ ((uint32_t)(key >> 32) * 0x9E3779B1u);
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}
__device__ __forceinline__ uint32_t bloom_bits(uint32_t h) { return (1u << ((h >> 20) & 31)) | (1u << ((h >> 26) & 31)); }

__global__ void bloom2_build_kernel(const uint64_t* __restrict__ keys, int64_t cap, uint32_t* words,
                                    uint32_t word_mask) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  const uint64_t k = keys[i];
  if (k == DGR_EMPTY_KEY) return;
  const uint32_t h = bloom_mix(k);
  atomicOr(words + (h & word_mask), bloom_bits(h));
}

// ---------------------------------------------------------------------------------------
// kernel maps: probe -> bit masks + block counts, scan, fill
// ---------------------------------------------------------------------------------------
// Probe kernel.  grid (row blocks of 512 rows, kappa chunks); thread = output row.
//
// Two phases per warp, decoupled by a shared-memory queue:
//   generate  every lane tests its row's neighbour key against the Bloom filter (shared memory, no global
//             traffic); lanes whose key MAY exist push (kappa, lane) into the warp's queue;
//   drain     whenever 32 candidates are queued, every lane takes ONE and does the hash-table lookup (L2):
//             all 32 lanes busy, 32 independent L2 chains in flight.
// Probing in place instead would make the whole warp wait for an L2 round trip whenever ANY of its 32 lanes
// passes the filter (a 3 % pass rate per lane is 62 % per warp) with one or two lanes doing useful work.
// Output: kDense ? nbr[kappa * nbr_stride + j] = input row or -1
//                : bits[kappa * W + w] = ballot of warp w's rows (+ per-(kappa, 256-word block) counts)
// kSym (a same-stride map: the input table is the output table, the offsets a centred odd cube, so offset
// k_last - kappa is the negation of offset kappa): only the buckets kappa < k_last / 2 are probed (K of them).
// A hit j -> i of bucket kappa is also the pair i -> j of the mirror bucket k_last - kappa: bit i of that bucket
// is set with a global atomicOr (its words zeroed by the caller).  The centre bucket k_last / 2 (offset 0) holds
// every live row and is written from the row count without a probe.  kmap_count_kernel counts both afterwards.
template <bool kBloom, bool kDense, bool kSym>
__global__ void __launch_bounds__(kProbeThreads, 2)
kmap_probe_kernel(const int32_t* __restrict__ out_coords, const int32_t* __restrict__ n_out_dev, int64_t n_out_max,
                  int ncols, const dgr_keyspec_t* __restrict__ spec_p, const uint64_t* __restrict__ keys,
                  const int32_t* __restrict__ vals, uint64_t mask, const uint32_t* __restrict__ bloom,
                  uint32_t n_bloom_words, const int32_t* __restrict__ offsets, int K, int k_per_block,
                  uint32_t* __restrict__ bits, int W, int32_t* block_cnt, int bpk, int32_t* __restrict__ nbr,
                  int64_t nbr_stride, int32_t* hit_count, int k_last) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int kWarps = kProbeThreads / 32;
  long long* delta = reinterpret_cast<long long*>(smem_raw);                               // [k_per_block]
  uint32_t* mtile = reinterpret_cast<uint32_t*>(smem_raw + (size_t)k_per_block * 8);       // [kWarps][k_per_block]
  uint16_t* queue = reinterpret_cast<uint16_t*>(mtile + (size_t)kWarps * k_per_block);     // [kWarps][64]
  uint32_t* bloom_s = reinterpret_cast<uint32_t*>(queue + kWarps * 64);                    // [n_bloom_words]
  const int n_out = dgr_dev_count(n_out_dev, n_out_max);
  const int k0 = blockIdx.y * k_per_block;
  const int kn = min(k_per_block, K - k0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if ((int64_t)blockIdx.x * kProbeThreads >= n_out) {
    // rows beyond the actual count: their mask words must still read as zero (a dense table is never read there)
    if (!kDense) {
      const int w = blockIdx.x * kWarps + warp;
      if (lane == 0 && w < W)
        for (int kk = 0; kk < kn; ++kk) bits[(int64_t)(k0 + kk) * W + w] = 0u;
    }
    return;
  }
  const dgr_keyspec_t s = *spec_p;
  for (int kk = threadIdx.x; kk < kn; kk += blockDim.x) {
    long long d = 0;
    const int32_t* o = offsets + (int64_t)(k0 + kk) * (ncols - 1);
    for (int a = 0; a < ncols - 1; ++a) d += (long long)o[a] * (1ll << s.shift[a + 1]);
    delta[kk] = d;
  }
  if (!kDense)
    for (int e = threadIdx.x; e < kWarps * k_per_block; e += blockDim.x) mtile[e] = 0u;
  if (kBloom)
    for (uint32_t i = threadIdx.x; i < n_bloom_words; i += blockDim.x) bloom_s[i] = bloom[i];
  __syncthreads();
  const int64_t j = (int64_t)blockIdx.x * kProbeThreads + threadIdx.x;
  const bool live = j < n_out;
  const uint64_t key = live ? dgr_pack_key(out_coords + j * ncols, s) : 0;
  const uint32_t key_lo = (uint32_t)key, key_hi = (uint32_t)(key >> 32);
  const int64_t row0 = j - lane;                       // first row of this warp
  const uint32_t wm = n_bloom_words - 1;
  uint16_t* q = queue + warp * 64;
  uint32_t* mt = mtile + warp * k_per_block;
  int qn = 0;                                          // queued candidates (warp-uniform)
  auto mirror = [&](int kappa, int32_t i) {            // kSym: hit (kappa, in i, out j) is the pair (k_last - kappa, in j, out i)
    atomicOr(bits + (int64_t)(k_last - kappa) * W + (i >> 5), 1u << (i & 31));
  };
  if (kSym && blockIdx.y == 0) {                       // centre bucket: the identity pair of every live row
    const uint32_t m = __ballot_sync(0xffffffffu, live);
    if (lane == 0 && (j >> 5) < W) bits[(int64_t)(k_last / 2) * W + (j >> 5)] = m;
  }

  auto drain = [&](int count) {                        // lanes < count take one candidate each
    __syncwarp();
    const uint32_t e = lane < count ? q[lane] : 0u;
    const int src = e & 31, kq = e >> 5;
    const uint32_t lo = __shfl_sync(0xffffffffu, key_lo, src), hi = __shfl_sync(0xffffffffu, key_hi, src);
    if (lane < count) {
      const uint64_t qq = (((uint64_t)hi << 32) | lo) + (uint64_t)delta[kq];
      const int32_t i = dgr_hash_lookup(keys, vals, mask, qq);
      if (kDense) {
        nbr[(int64_t)(k0 + kq) * nbr_stride + row0 + src] = i;
        if (hit_count != nullptr) {
          const uint32_t act = __activemask();
          const uint32_t hits = __ballot_sync(act, i >= 0);
          if (lane == (__ffs(act) - 1) && hits) atomicAdd(hit_count, __popc(hits));
        }
      } else if (i >= 0) {
        atomicOr(mt + kq, 1u << src);
        if (kSym) mirror(k0 + kq, i);
      }
    }
    __syncwarp();
    // move the (at most 31) entries behind the drained ones to the front
    const uint32_t rest = (lane + 32 < qn) ? q[lane + 32] : 0u;
    __syncwarp();
    if (lane + 32 < qn) q[lane] = (uint16_t)rest;
    qn = qn > 32 ? qn - 32 : 0;
    __syncwarp();
  };

  if (!kBloom && !kDense) {
    // no filter (3^3 kernels: ~60 % of the probes hit): probe in place, four independent lookups in flight
    const int w = (int)(j >> 5);
    const int cnt_col = w / kCntWords;
    for (int kk = 0; kk < kn; kk += 4) {
      int32_t found[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        found[u] = live && kk + u < kn ? dgr_hash_lookup(keys, vals, mask, key + (uint64_t)delta[min(kk + u, kn - 1)]) : -1;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (kk + u >= kn) break;                                     // uniform
        if (kSym && found[u] >= 0) mirror(k0 + kk + u, found[u]);
        const uint32_t m = __ballot_sync(0xffffffffu, found[u] >= 0);
        if (lane == 0 && w < W) {
          bits[(int64_t)(k0 + kk + u) * W + w] = m;
          if (m) atomicAdd(block_cnt + (int64_t)(k0 + kk + u) * bpk + cnt_col, __popc(m));
        }
      }
    }
    return;
  }
  for (int kk = 0; kk < kn; ++kk) {
    bool maybe = live;
    if (kBloom && live) {
      const uint32_t h = bloom_mix(key + (uint64_t)delta[kk]);
      const uint32_t b = bloom_bits(h);
      maybe = (bloom_s[h & wm] & b) == b;
    }
    if (kDense && live && !maybe) nbr[(int64_t)(k0 + kk) * nbr_stride + j] = -1;
    const uint32_t cand = __ballot_sync(0xffffffffu, maybe);
    if (cand) {
      if (maybe) q[qn + __popc(cand & ((1u << lane) - 1u))] = (uint16_t)((kk << 5) | lane);
      qn += __popc(cand);
      if (qn >= 32) drain(32);
    }
  }
  if (qn > 0) drain(qn);
  if (!kDense) {
    __syncwarp();
    const int w = (int)(j >> 5);
    if (w < W) {
      const int cnt_col = w / kCntWords;
      for (int kk = lane; kk < kn; kk += 32) {
        const uint32_t m = mt[kk];
        bits[(int64_t)(k0 + kk) * W + w] = m;
        if (m) atomicAdd(block_cnt + (int64_t)(k0 + kk) * bpk + cnt_col, __popc(m));
      }
    }
  }
}

// Down map (kernel 3, input tensor stride s, output stride 2s) enumerated from the input side.
// Output rows are multiples of 2s and input rows multiples of s, so input row c reaches output o = c - offset
// only where, on every spatial axis, o = c if c / s is even and o = c -/+ s (offset +s / -s) if it is odd:
// 2^(odd axes) candidates per input row (one of them, the floor parent, always exists), each looked up in the
// OUTPUT table.  kDownLanes lanes share a row and take its candidates in turn, so a row with every axis odd
// (64 candidates in 6-D) is not one thread's chain of 64 dependent L2 round trips.  A hit sets bit o of bucket
// kappa with atomicOr (words zeroed by the caller): the masks equal those of probing all 3^D offsets per output
// row.  Offsets are enumerated axis 0 fastest, digit 0 / 1 / 2 = offset -s / 0 / +s.
constexpr int kDownLanes = 8;
__global__ void __launch_bounds__(kThreads)
kmap_down_kernel(const int32_t* __restrict__ in_coords, const int32_t* __restrict__ n_in_dev, int64_t n_in_max,
                 int ncols, int stride, const dgr_keyspec_t* __restrict__ spec_p, const uint64_t* __restrict__ out_keys,
                 const int32_t* __restrict__ out_vals, uint64_t out_mask, uint32_t* __restrict__ bits, int W) {
  const int n_in = dgr_dev_count(n_in_dev, n_in_max);
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t i = t / kDownLanes;
  if (i >= n_in) return;
  const dgr_keyspec_t s = *spec_p;
  const int32_t* c = in_coords + i * ncols;
  const uint64_t key = dgr_pack_key(c, s);
  uint32_t odd = 0;
#pragma unroll
  for (int a = 1; a < DGR_MAX_COLS; ++a)
    if (a < ncols) odd |= (uint32_t)((c[a] / stride) & 1) << a;   // exact division; & 1 is floor parity for c < 0 too
  const uint32_t n_cand = 1u << __popc(odd);
  for (uint32_t sub = (uint32_t)(t % kDownLanes); sub < n_cand; sub += kDownLanes) {
    int kappa = 0, p = 1, b = 0;
    long long d = 0;
#pragma unroll
    for (int a = 1; a < DGR_MAX_COLS; ++a) {
      if (a < ncols) {
        int digit = 1;
        if ((odd >> a) & 1u) {
          const long long step = (long long)stride << s.shift[a];
          if ((sub >> b++) & 1u) { digit = 2; d -= step; }      // offset +s: o = c - s
          else { digit = 0; d += step; }                        // offset -s: o = c + s
        }
        kappa += digit * p;
        p *= 3;
      }
    }
    const int32_t o = dgr_hash_lookup(out_keys, out_vals, out_mask, key + (uint64_t)d);
    if (o >= 0) atomicOr(bits + (int64_t)kappa * W + (o >> 5), 1u << (o & 31));
  }
}

// Per-(kappa, 256-word block) pair counts of the buckets k_lo + blockIdx.y from their finished masks (the buckets
// the down and mirror paths set with atomicOr); grid (bpk, buckets).
__global__ void __launch_bounds__(kThreads)
kmap_count_kernel(const uint32_t* __restrict__ bits, int W, int bpk, int k_lo, int32_t* __restrict__ block_cnt) {
  const int64_t kappa = k_lo + blockIdx.y;
  const int w = blockIdx.x * kCntWords + threadIdx.x;
  int total;
  dgr_block_exclusive_scan<kThreads>(w < W ? __popc(bits[kappa * W + w]) : 0, &total);
  if (threadIdx.x == 0) block_cnt[kappa * bpk + blockIdx.x] = total;
}

// exclusive scan of the K x bpk block counts (one block), bucket offsets, work-list sizes
// meta[0..4] = (pairs P, tiles, tiles with every offset rounded up to an even count,
//              non-empty offsets, key-overflow flag of spec)
__global__ void kmap_scan_kernel(int32_t* cnt, int K, int bpk, int tile_rows, int32_t* kofs,
                                 int32_t* meta, const dgr_keyspec_t* spec) {
  const int64_t nb = (int64_t)K * bpk;
  const int total = dgr_block_scan_inplace(cnt, nb);
  if (threadIdx.x == 0) cnt[nb] = total;
  __syncthreads();
  __shared__ int red[3][32];
  int tiles = 0, ptiles = 0, nonempty = 0;
  for (int k = threadIdx.x; k <= K; k += blockDim.x) {
    const int lo = cnt[(int64_t)k * bpk];        // k == K reads cnt[nb] = total
    kofs[k] = lo;
    if (k < K) {
      const int hi = (k + 1 < K) ? cnt[(int64_t)(k + 1) * bpk] : total;
      const int t = (hi - lo + tile_rows - 1) / tile_rows;
      tiles += t;
      ptiles += (t + 1) & ~1;
      nonempty += (hi > lo);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    tiles += __shfl_xor_sync(0xffffffffu, tiles, d);
    ptiles += __shfl_xor_sync(0xffffffffu, ptiles, d);
    nonempty += __shfl_xor_sync(0xffffffffu, nonempty, d);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = tiles;
    red[1][threadIdx.x >> 5] = ptiles;
    red[2][threadIdx.x >> 5] = nonempty;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, b = 0, c = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += red[0][w]; b += red[1][w]; c += red[2][w]; }
    const int ovf = spec != nullptr ? spec->overflow : 0;
    kofs[K + 1] = ovf;
    meta[0] = total; meta[1] = a; meta[2] = b; meta[3] = c; meta[4] = ovf;
  }
}

// Fill: grid (bpk, K); block (b, kappa) owns the 256 mask words [b * 256, +256) of bucket kappa, one per thread;
// its output offset is the scanned count of exactly that block, so blocks without a hit leave at once (a 6-D
// map at stride 1 has a hit in ~10 % of its blocks).  A word's 32 hits are resolved by the 32 LANES of a warp in
// parallel (each lane: one hash lookup, consecutive output positions): the longest serial chain is the 32 words
// of a warp, not the hits of a thread.
__global__ void __launch_bounds__(kThreads)
kmap_fill_kernel(const uint32_t* __restrict__ bits, int W, int bpk, const int32_t* __restrict__ block_ofs,
                 const int32_t* __restrict__ out_coords, int ncols, const dgr_keyspec_t* __restrict__ spec_p,
                 const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask,
                 const int32_t* __restrict__ offsets, int32_t* __restrict__ in_idx, int32_t* __restrict__ out_idx) {
  __shared__ uint32_t s_mask[kThreads];
  __shared__ int s_base[kThreads];
  const int kappa = blockIdx.y;
  const int64_t e = (int64_t)kappa * bpk + blockIdx.x;
  const int base = block_ofs[e];
  if (block_ofs[e + 1] == base) return;                        // no pair in this block (uniform)
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int w_own = blockIdx.x * kCntWords + t;
  const uint32_t m_own = w_own < W ? bits[(int64_t)kappa * W + w_own] : 0u;
  const int excl = dgr_block_exclusive_scan<256>(__popc(m_own), nullptr);
  s_mask[t] = m_own;
  s_base[t] = base + excl;
  __syncthreads();
  const dgr_keyspec_t s = *spec_p;
  long long d = 0;
  const int32_t* o = offsets + (int64_t)kappa * (ncols - 1);
  for (int a = 0; a < ncols - 1; ++a) d += (long long)o[a] * (1ll << s.shift[a + 1]);
  const int w_first = blockIdx.x * kCntWords + warp * 32;      // this warp resolves its own 32 words
  for (int u = 0; u < 32; ++u) {
    const uint32_t m = s_mask[warp * 32 + u];
    if (m == 0u) continue;                                     // uniform
    if ((m >> lane) & 1u) {
      const int64_t j = (int64_t)(w_first + u) * 32 + lane;
      const int pos = s_base[warp * 32 + u] + __popc(m & ((1u << lane) - 1u));
      const uint64_t qq = dgr_pack_key(out_coords + j * ncols, s) + (uint64_t)d;
      in_idx[pos] = dgr_hash_lookup(keys, vals, mask, qq);
      out_idx[pos] = (int32_t)j;
    }
  }
}

// Work list of a kernel map (one block): bucket k gets ceil(count_k / tile_rows) tiles, rounded up to an even
// number when `pair` is set (CTA pairs; the last tile may then be empty); tile t covers pairs
// [tile_start[t], +tile_rows) of bucket tile_k[t].
__global__ void tiles_kernel(const int32_t* __restrict__ kofs, int K, int tile_rows, int n_tiles, int pair,
                             int32_t* __restrict__ tile_k, int32_t* __restrict__ tile_start) {
  extern __shared__ int tofs[];   // K + 1 exclusive tile offsets
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int v = (kofs[k + 1] - kofs[k] + tile_rows - 1) / tile_rows;
    tofs[k] = pair ? (v + 1) & ~1 : v;
  }
  __syncthreads();
  const int total = dgr_block_scan_inplace(tofs, K);
  if (threadIdx.x == 0) tofs[K] = total;
  __syncthreads();
  for (int t = threadIdx.x; t < n_tiles; t += blockDim.x) {
    int lo = 0, hi = K;   // largest k with tofs[k] <= t (non-empty: tofs[k + 1] > t)
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
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

int32_t dgr_compact_voxel_pair(const int32_t* raw_coords, const int32_t* sel, const int32_t* n_unique,
                               int64_t n_raw0, int64_t n_raw1, const void* xyz0, int32_t is_f64_0,
                               const void* xyz1, int32_t is_f64_1, double cell, int32_t* coords, float* xyz,
                               int32_t* counts, void* stream) {
  DGR_ARG_CHECK(cell > 0 && cell < INFINITY, "cell must be positive and finite");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n_max = n_raw0 + n_raw1;
  unsigned blocks = dgr_blocks(n_max > 0 ? n_max : 1, kThreads);
  if (blocks > 1184) blocks = 1184;
#define DGR_CV(T0, T1)                                                                                         \
  compact_voxels_kernel<T0, T1><<<blocks, kThreads, 0, st>>>(raw_coords, sel, n_unique, n_raw0, (const T0*)xyz0, \
                                                             (const T1*)xyz1, cell, coords, xyz, counts)
  if (is_f64_0 && is_f64_1) DGR_CV(double, double);
  else if (is_f64_0) DGR_CV(double, float);
  else if (is_f64_1) DGR_CV(float, double);
  else DGR_CV(float, float);
#undef DGR_CV
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_bloom2_build(const uint64_t* keys, int64_t cap, uint32_t* words, int64_t n_words, void* stream) {
  DGR_ARG_CHECK(cap > 0 && (cap & (cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(n_words >= 32 && (n_words & (n_words - 1)) == 0, "n_words must be a power of two");
  cudaStream_t st = (cudaStream_t)stream;
  DGR_CUDA_CHECK(cudaMemsetAsync(words, 0, (size_t)n_words * 4, st));
  bloom2_build_kernel<<<dgr_blocks(cap, kThreads), kThreads, 0, st>>>(keys, cap, words, (uint32_t)n_words - 1);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

/* Filter size of a table of n_max keys: about 10 bits per key, a power of two in [1024, 16384] words, so that it
 * fits the 32768-word shared-memory limit of dgr_kmap_probe / dgr_kmap_dense. */
int64_t dgr_bloom2_words(int64_t n_max) {
  int64_t words = 1;
  while (words < (n_max * 10 + 31) / 32) words <<= 1;
  return words < 1024 ? 1024 : (words > 16384 ? 16384 : words);
}

/* words per offset of the bit-mask representation (one word per 32 output rows) */
int64_t dgr_kmap_mask_words(int64_t n_out_max) {
  const int64_t w = (n_out_max + 31) / 32;
  return w < 1 ? 1 : w;
}
/* ints of the block-count workspace: K * ceil(W / 2048) + 2 */
int64_t dgr_kmap_cnt_elems(int32_t K, int64_t n_out_max) {
  const int64_t W = dgr_kmap_mask_words(n_out_max);
  return (int64_t)K * ((W + kCntWords - 1) / kCntWords) + 2;
}

static size_t probe_smem_bytes(int k_per_block, int64_t n_bloom_words) {
  return (size_t)k_per_block * 8 + (size_t)(kProbeThreads / 32) * k_per_block * 4 + (size_t)(kProbeThreads / 32) * 64 * 2 +
         (size_t)n_bloom_words * 4;
}
static int probe_k_per_block(int K, unsigned row_blocks) {
  // kappa chunks: enough blocks for ~2 waves of the 132 SMs at 2 blocks per SM, at most 96 offsets per block
  int k_per_block = K;
  while (k_per_block > 16 && (int64_t)row_blocks * ((K + k_per_block - 1) / k_per_block) < 528) k_per_block = (k_per_block + 1) / 2;
  if (k_per_block > 96) k_per_block = 96;
  return (k_per_block + 3) & ~3;
}

int32_t dgr_kmap_probe_mode(int32_t mode, const int32_t* out_coords, int64_t n_out_max, const int32_t* n_out_dev,
                            int32_t ncols, const dgr_keyspec_t* spec, const uint64_t* in_keys, const int32_t* in_vals,
                            int64_t in_cap, const uint32_t* bloom_words, int64_t n_bloom_words, const int32_t* offsets,
                            int32_t K, const int32_t* in_coords, int64_t n_in_max, const int32_t* n_in_dev,
                            int32_t in_stride, const uint64_t* out_keys, const int32_t* out_vals, int64_t out_cap,
                            uint32_t* bits, int32_t* block_cnt, int32_t* kofs, int32_t* meta, void* stream) {
  DGR_ARG_CHECK(mode == DGR_KMAP_GENERAL || mode == DGR_KMAP_SAME || mode == DGR_KMAP_DOWN, "unknown probe mode");
  DGR_ARG_CHECK(in_cap > 0 && (in_cap & (in_cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(K >= 1 && K <= 65535, "K out of range");
  DGR_ARG_CHECK(bloom_words == nullptr || (n_bloom_words >= 32 && (n_bloom_words & (n_bloom_words - 1)) == 0 &&
                                           n_bloom_words <= 32768),
                "bloom: power of two, 32..32768 words");
  DGR_ARG_CHECK(mode != DGR_KMAP_SAME || (K > 1 && (K & 1)), "same-stride mode: a centred odd cube of offsets");
  if (mode == DGR_KMAP_DOWN) {
    int64_t k3 = 1;
    for (int a = 1; a < ncols; ++a) k3 *= 3;
    DGR_ARG_CHECK(K == k3, "down mode: kernel size 3");
    DGR_ARG_CHECK(in_coords != nullptr && in_stride >= 1 && n_in_max >= 0, "down mode: input rows and stride");
    DGR_ARG_CHECK(out_keys != nullptr && out_vals != nullptr && out_cap > 0 && (out_cap & (out_cap - 1)) == 0,
                  "down mode: output table, capacity a power of two");
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t nmx = n_out_max > 0 ? n_out_max : 1;
  const int W = (int)dgr_kmap_mask_words(nmx);
  const int bpk = (W + kCntWords - 1) / kCntWords;
  DGR_CUDA_CHECK(cudaMemsetAsync(block_cnt, 0, (size_t)dgr_kmap_cnt_elems(K, nmx) * sizeof(int32_t), st));
  int k_counted = K;                                   // buckets [k_counted, K) are counted from their masks
  if (mode == DGR_KMAP_DOWN) {
    DGR_CUDA_CHECK(cudaMemsetAsync(bits, 0, (size_t)K * W * sizeof(uint32_t), st));
    if (n_in_max > 0)
      kmap_down_kernel<<<dgr_blocks(n_in_max * kDownLanes, kThreads), kThreads, 0, st>>>(
          in_coords, n_in_dev, n_in_max, ncols, in_stride, spec, out_keys, out_vals, (uint64_t)out_cap - 1, bits, W);
    k_counted = 0;
  } else {
    // same-stride mode: probe the buckets below the centre, the rest are mirrored (and set with atomicOr)
    const bool sym = mode == DGR_KMAP_SAME;
    const int Kp = sym ? (K - 1) / 2 : K;
    if (sym) DGR_CUDA_CHECK(cudaMemsetAsync(bits + (int64_t)Kp * W, 0, (size_t)(K - Kp) * W * sizeof(uint32_t), st));
    k_counted = Kp;
    const unsigned row_blocks = dgr_blocks(nmx, kProbeThreads);
    const int k_per_block = probe_k_per_block(Kp, row_blocks);
    const dim3 grid(row_blocks, (Kp + k_per_block - 1) / k_per_block);
    const uint32_t* bw = bloom_words;
    const uint32_t nbw = bloom_words != nullptr ? (uint32_t)n_bloom_words : 1u;
    const size_t smem = probe_smem_bytes(k_per_block, bloom_words != nullptr ? n_bloom_words : 0);
#define DGR_PROBE(B, S)                                                                                             \
  do {                                                                                                              \
    DGR_ENSURE_SMEM((kmap_probe_kernel<B, false, S>), smem);                                                       \
    kmap_probe_kernel<B, false, S><<<grid, kProbeThreads, smem, st>>>(                                              \
        out_coords, n_out_dev, n_out_max, ncols, spec, in_keys, in_vals, (uint64_t)in_cap - 1, bw, nbw, offsets, Kp, \
        k_per_block, bits, W, block_cnt, bpk, nullptr, 0, nullptr, K - 1);                                          \
  } while (0)
    if (bloom_words != nullptr) {
      if (sym) DGR_PROBE(true, true); else DGR_PROBE(true, false);
    } else {
      if (sym) DGR_PROBE(false, true); else DGR_PROBE(false, false);
    }
#undef DGR_PROBE
  }
  if (k_counted < K) kmap_count_kernel<<<dim3(bpk, K - k_counted), kThreads, 0, st>>>(bits, W, bpk, k_counted, block_cnt);
  kmap_scan_kernel<<<1, 1024, 0, st>>>(block_cnt, K, bpk, 128, kofs, meta, spec);
  dgr_note_launches(k_counted < K ? 3 : 2);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_kmap_probe(const int32_t* out_coords, int64_t n_out_max, const int32_t* n_out_dev, int32_t ncols,
                       const dgr_keyspec_t* spec, const uint64_t* in_keys, const int32_t* in_vals, int64_t in_cap,
                       const uint32_t* bloom_words, int64_t n_bloom_words, const int32_t* offsets, int32_t K,
                       uint32_t* bits, int32_t* block_cnt, int32_t* kofs, int32_t* meta, void* stream) {
  return dgr_kmap_probe_mode(DGR_KMAP_GENERAL, out_coords, n_out_max, n_out_dev, ncols, spec, in_keys, in_vals, in_cap,
                             bloom_words, n_bloom_words, offsets, K, nullptr, 0, nullptr, 0, nullptr, nullptr, 0, bits,
                             block_cnt, kofs, meta, stream);
}

int32_t dgr_kmap_fill(const uint32_t* bits, const int32_t* block_cnt, int32_t K, int64_t n_out_max,
                      const int32_t* out_coords, int32_t ncols, const dgr_keyspec_t* spec,
                      const uint64_t* in_keys, const int32_t* in_vals, int64_t in_cap, const int32_t* offsets,
                      int32_t* in_idx, int32_t* out_idx, void* stream) {
  const int64_t nmx = n_out_max > 0 ? n_out_max : 1;
  const int W = (int)dgr_kmap_mask_words(nmx);
  const int bpk = (W + kCntWords - 1) / kCntWords;
  kmap_fill_kernel<<<dim3(bpk, K), kThreads, 0, (cudaStream_t)stream>>>(bits, W, bpk, block_cnt, out_coords, ncols,
                                                                            spec, in_keys, in_vals, (uint64_t)in_cap - 1,
                                                                            offsets, in_idx, out_idx);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_kmap_dense(const int32_t* out_coords, int64_t n_out_max, const int32_t* n_out_dev, int32_t ncols,
                       const dgr_keyspec_t* spec, const uint64_t* in_keys, const int32_t* in_vals, int64_t in_cap,
                       const uint32_t* bloom_words, int64_t n_bloom_words, const int32_t* offsets, int32_t K,
                       int32_t* nbr, int64_t nbr_stride, int32_t* hit_count, void* stream) {
  DGR_ARG_CHECK(in_cap > 0 && (in_cap & (in_cap - 1)) == 0, "capacity must be a power of two");
  DGR_ARG_CHECK(nbr_stride >= n_out_max, "row stride below the row bound");
  if (hit_count != nullptr) DGR_CUDA_CHECK(cudaMemsetAsync(hit_count, 0, sizeof(int32_t), (cudaStream_t)stream));
  DGR_ARG_CHECK(bloom_words == nullptr || (n_bloom_words >= 32 && (n_bloom_words & (n_bloom_words - 1)) == 0 &&
                                           n_bloom_words <= 32768),
                "bloom: power of two, 32..32768 words");
  if (n_out_max == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned row_blocks = dgr_blocks(n_out_max, kProbeThreads);
  const int k_per_block = probe_k_per_block(K, row_blocks);
  const dim3 grid(row_blocks, (K + k_per_block - 1) / k_per_block);
  if (bloom_words != nullptr) {
    const size_t smem = probe_smem_bytes(k_per_block, n_bloom_words);
    DGR_ENSURE_SMEM((kmap_probe_kernel<true, true, false>), smem);
    kmap_probe_kernel<true, true, false><<<grid, kProbeThreads, smem, st>>>(
        out_coords, n_out_dev, n_out_max, ncols, spec, in_keys, in_vals, (uint64_t)in_cap - 1, bloom_words,
        (uint32_t)n_bloom_words, offsets, K, k_per_block, nullptr, 0, nullptr, 0, nbr, nbr_stride, hit_count, 0);
  } else {
    const size_t smem = probe_smem_bytes(k_per_block, 0);
    kmap_probe_kernel<false, true, false><<<grid, kProbeThreads, smem, st>>>(
        out_coords, n_out_dev, n_out_max, ncols, spec, in_keys, in_vals, (uint64_t)in_cap - 1, nullptr, 1u, offsets, K,
        k_per_block, nullptr, 0, nullptr, 0, nbr, nbr_stride, hit_count, 0);
  }
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_kernel_map_tiles(const int32_t* kofs, int32_t K, int32_t tile_rows, int32_t n_tiles, int32_t pair,
                             int32_t* tile_k, int32_t* tile_start, void* stream) {
  DGR_ARG_CHECK(tile_rows >= 1, "tile_rows must be positive");
  if (n_tiles == 0) return DGR_OK;
  tiles_kernel<<<1, 1024, (K + 1) * sizeof(int), (cudaStream_t)stream>>>(kofs, K, tile_rows, n_tiles, pair, tile_k,
                                                                        tile_start);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
