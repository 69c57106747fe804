// Safeguard registration: RANSAC over a fixed correspondence list, the job open3d's
// registration_ransac_based_on_correspondence does for the reference
// (core/deep_global_registration.py:50-64, called from :302-315 when the weight sum is below
// the gate).  ransac_n = 4, TransformationEstimationPointToPoint(with_scaling=False), no
// checkers; a hypothesis is better when it has more inliers (|T p - q| < max_dist over ALL
// correspondences) or as many with a lower inlier RMSE.  The reference passes
// RANSACConvergenceCriteria(4000000, num_iterations = 80000): the 80000 lands in the
// confidence slot, open3d clamps it to 1, the early-exit estimate log(1 - confidence) / ... is
// never reached and all max_iteration hypotheses are evaluated - which is what happens here.
//
// One thread owns kHyp hypotheses (R, t in registers); the correspondences stream through
// shared memory in tiles and every thread reads the same element (broadcast), so the kernel
// is bound by the fp32 pipe: ~19 instructions per (hypothesis, correspondence).
// Sampling is a counter-based hash of (seed, hypothesis, slot): reproducible, and restated
// in oracle/ransac.py so the CPU checker draws the very same hypotheses.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kabsch.cuh"

namespace {

constexpr int kRansacThreads = 256;
constexpr int kHyp = 4;        // hypotheses per thread
constexpr int kTile = 512;     // correspondences per shared-memory tile (16 KB)

__global__ void ransac_pack_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                   const int32_t* __restrict__ idx0, const int32_t* __restrict__ idx1,
                                   int64_t n, float4* __restrict__ src, float4* __restrict__ tgt) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t a = idx0 != nullptr ? (int64_t)idx0[i] : i;
  int64_t b = idx1 != nullptr ? (int64_t)idx1[i] : i;
  src[i] = make_float4(x[3 * a], x[3 * a + 1], x[3 * a + 2], 0.f);
  tgt[i] = make_float4(y[3 * b], y[3 * b + 1], y[3 * b + 2], 0.f);
}

// slot-th sample of hypothesis h: uniform in [0, n) (with replacement, like open3d's
// per-iteration uniform_int_distribution draws)
__device__ __forceinline__ uint32_t ransac_pick(uint64_t seed, uint64_t h, int slot, uint32_t n) {
  return dgr_counter_pick(seed, h * 4 + (uint64_t)slot, n);
}

// Umeyama without scaling: the pose (R, t) minimising sum |R p_j + t - q_j|^2 over 4 pairs, fp64
__device__ void ransac_fit4(const double p[4][3], const double q[4][3], double R[3][3], double t[3]) {
  double mp[3] = {0, 0, 0}, mq[3] = {0, 0, 0};
  for (int j = 0; j < 4; ++j)
    for (int c = 0; c < 3; ++c) { mp[c] += p[j][c]; mq[c] += q[j][c]; }
  for (int c = 0; c < 3; ++c) { mp[c] *= 0.25; mq[c] *= 0.25; }
  double S[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double acc = 0;
      for (int j = 0; j < 4; ++j) acc += (q[j][r] - mq[r]) * (p[j][c] - mp[c]);
      S[r][c] = acc * 0.25;
    }
  kabsch_rotation(S, R);
  for (int r = 0; r < 3; ++r) t[r] = mq[r] - (R[r][0] * mp[0] + R[r][1] * mp[1] + R[r][2] * mp[2]);
}

// the pose of hypothesis h over the packed correspondence list
__device__ void ransac_hypothesis(const float4* __restrict__ src, const float4* __restrict__ tgt, uint32_t n,
                                  uint64_t seed, uint64_t h, double R[3][3], double t[3]) {
  double p[4][3], q[4][3];
  for (int j = 0; j < 4; ++j) {
    uint32_t i = ransac_pick(seed, h, j, n);
    float4 a = __ldg(src + i), b = __ldg(tgt + i);
    p[j][0] = a.x; p[j][1] = a.y; p[j][2] = a.z;
    q[j][0] = b.x; q[j][1] = b.y; q[j][2] = b.z;
  }
  ransac_fit4(p, q, R, t);
}

// (inliers, sum d^2) -> a key whose unsigned order is open3d's IsBetterRANSACThan: more
// inliers first; at equal count the smaller squared-error sum (= smaller RMSE)
__device__ __forceinline__ unsigned long long ransac_key(uint32_t cnt, float err2) {
  return ((unsigned long long)cnt << 32) | (unsigned long long)(0xFFFFFFFFu - __float_as_uint(err2));
}

__global__ void __launch_bounds__(kRansacThreads)
ransac_eval_kernel(const float4* __restrict__ src, const float4* __restrict__ tgt, uint32_t n, uint64_t seed,
                   uint64_t num_hyp, float max_d2, unsigned long long* __restrict__ blk_key,
                   unsigned long long* __restrict__ blk_hyp) {
  __shared__ float4 s_src[kTile], s_tgt[kTile];
  __shared__ unsigned long long s_key[kRansacThreads / 32], s_hyp[kRansacThreads / 32];
  const int tid = threadIdx.x;
  const uint64_t h0 = ((uint64_t)blockIdx.x * kRansacThreads + tid) * kHyp;

  float R[kHyp][9], t[kHyp][3];
#pragma unroll
  for (int h = 0; h < kHyp; ++h) {
    if (h0 + h < num_hyp) {
      double Rd[3][3], td[3];
      ransac_hypothesis(src, tgt, n, seed, h0 + h, Rd, td);
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) R[h][3 * r + c] = (float)Rd[r][c];
        t[h][r] = (float)td[r];
      }
    } else {      // past the end: a pose nothing can be an inlier of
      for (int k = 0; k < 9; ++k) R[h][k] = 0.f;
      t[h][0] = t[h][1] = t[h][2] = 3.0e18f;
    }
  }

  uint32_t cnt[kHyp];
  float err[kHyp];
#pragma unroll
  for (int h = 0; h < kHyp; ++h) { cnt[h] = 0; err[h] = 0.f; }

  for (uint32_t base = 0; base < n; base += kTile) {
    const int m = (int)min((uint32_t)kTile, n - base);
    __syncthreads();
    for (int i = tid; i < m; i += kRansacThreads) {
      s_src[i] = __ldg(src + base + i);
      s_tgt[i] = __ldg(tgt + base + i);
    }
    __syncthreads();
#pragma unroll 4
    for (int i = 0; i < m; ++i) {
      const float4 a = s_src[i], b = s_tgt[i];
#pragma unroll
      for (int h = 0; h < kHyp; ++h) {
        float dx = fmaf(R[h][0], a.x, fmaf(R[h][1], a.y, fmaf(R[h][2], a.z, t[h][0] - b.x)));
        float dy = fmaf(R[h][3], a.x, fmaf(R[h][4], a.y, fmaf(R[h][5], a.z, t[h][1] - b.y)));
        float dz = fmaf(R[h][6], a.x, fmaf(R[h][7], a.y, fmaf(R[h][8], a.z, t[h][2] - b.z)));
        float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        bool in = d2 < max_d2;
        cnt[h] += in ? 1u : 0u;
        err[h] += in ? d2 : 0.f;
      }
    }
  }

  // best of the thread, the warp, the block; ties go to the lowest hypothesis number
  unsigned long long key = 0, hyp = ~0ull;
#pragma unroll
  for (int h = 0; h < kHyp; ++h) {
    unsigned long long k = cnt[h] ? ransac_key(cnt[h], err[h]) : 0ull;
    if (k > key) { key = k; hyp = h0 + h; }
  }
  for (int d = 16; d > 0; d >>= 1) {
    unsigned long long ok = __shfl_xor_sync(0xffffffffu, key, d);
    unsigned long long oh = __shfl_xor_sync(0xffffffffu, hyp, d);
    if (ok > key || (ok == key && oh < hyp)) { key = ok; hyp = oh; }
  }
  if ((tid & 31) == 0) { s_key[tid >> 5] = key; s_hyp[tid >> 5] = hyp; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kRansacThreads / 32; ++w)
      if (s_key[w] > key || (s_key[w] == key && s_hyp[w] < hyp)) { key = s_key[w]; hyp = s_hyp[w]; }
    blk_key[blockIdx.x] = key;
    blk_hyp[blockIdx.x] = hyp;
  }
}

// winner over the blocks, its pose regenerated in fp64 and re-scored in fp64 for the report
__global__ void __launch_bounds__(1024)
ransac_final_kernel(const float4* __restrict__ src, const float4* __restrict__ tgt, uint32_t n, uint64_t seed,
                    const unsigned long long* __restrict__ blk_key, const unsigned long long* __restrict__ blk_hyp,
                    uint32_t n_blk, double max_dist, double* __restrict__ result) {
  __shared__ unsigned long long s_key[32], s_hyp[32];
  __shared__ double s_T[12], s_red[32][2];
  const int tid = threadIdx.x;
  unsigned long long key = 0, hyp = ~0ull;
  for (uint32_t b = tid; b < n_blk; b += blockDim.x) {
    unsigned long long k = blk_key[b], h = blk_hyp[b];
    if (k > key || (k == key && h < hyp)) { key = k; hyp = h; }
  }
  for (int d = 16; d > 0; d >>= 1) {
    unsigned long long ok = __shfl_xor_sync(0xffffffffu, key, d);
    unsigned long long oh = __shfl_xor_sync(0xffffffffu, hyp, d);
    if (ok > key || (ok == key && oh < hyp)) { key = ok; hyp = oh; }
  }
  if ((tid & 31) == 0) { s_key[tid >> 5] = key; s_hyp[tid >> 5] = hyp; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (s_key[w] > key || (s_key[w] == key && s_hyp[w] < hyp)) { key = s_key[w]; hyp = s_hyp[w]; }
    s_key[0] = key;
    s_hyp[0] = hyp;
    double R[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}, t[3] = {0, 0, 0};
    if (key != 0) ransac_hypothesis(src, tgt, n, seed, hyp, R, t);
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) s_T[4 * r + c] = R[r][c];
      s_T[4 * r + 3] = t[r];
    }
  }
  __syncthreads();
  key = s_key[0];
  hyp = s_hyp[0];
  double ce[2] = {0, 0};                                  // inlier count, sum d^2
  if (key != 0) {
    for (uint32_t i = tid; i < n; i += blockDim.x) {
      float4 a = src[i], b = tgt[i];
      double dx = s_T[0] * a.x + s_T[1] * a.y + s_T[2] * a.z + s_T[3] - b.x;
      double dy = s_T[4] * a.x + s_T[5] * a.y + s_T[6] * a.z + s_T[7] - b.y;
      double dz = s_T[8] * a.x + s_T[9] * a.y + s_T[10] * a.z + s_T[11] - b.z;
      double d2 = dx * dx + dy * dy + dz * dz;
      if (sqrt(d2) < max_dist) { ce[0] += 1.0; ce[1] += d2; }
    }
  }
  const double cnt = dgr_block_sum<1024>(ce, s_red);
  const double err = __shfl_down_sync(0xffffffffu, cnt, 1);    // thread 1's sum
  if (tid == 0) {
    for (int k = 0; k < 12; ++k) result[k] = s_T[k];
    result[12] = 0; result[13] = 0; result[14] = 0; result[15] = 1;
    result[16] = n ? cnt / (double)n : 0.0;                 // fitness
    result[17] = cnt > 0 ? sqrt(err / cnt) : 0.0;           // inlier RMSE
    result[18] = key != 0 ? (double)hyp : -1.0;             // winning hypothesis
    result[19] = (double)(uint32_t)(key >> 32);             // its fp32 inlier count
  }
}

inline uint32_t ransac_blocks(int64_t num_hyp) {
  const int64_t per_block = (int64_t)kRansacThreads * kHyp;
  return (uint32_t)((num_hyp + per_block - 1) / per_block);
}

struct RansacWs {
  float4* src;                 // [n_corr] packed correspondences
  float4* tgt;
  unsigned long long* blk_key; // [n_blk] best key and hypothesis per evaluation block
  unsigned long long* blk_hyp;
};

// workspace size in 8-byte words; carves `base` into the regions when it is not null
int64_t ransac_layout(int64_t n_corr, int64_t num_hyp, uint64_t* base, RansacWs* w) {
  const int64_t n_blk = ransac_blocks(num_hyp);
  DgrCarver c(base);
  RansacWs r;
  r.src = c.take<float4>(n_corr);
  r.tgt = c.take<float4>(n_corr);
  r.blk_key = c.take<unsigned long long>(n_blk);
  r.blk_hyp = c.take<unsigned long long>(n_blk);
  c.take<uint64_t>(2);                                  // 2 unused words, part of the size reported since the start
  if (w != nullptr) *w = r;
  return c.words;
}

// ---------------------------------------------------------------------------------------
// Feature-matching RANSAC: open3d 0.10's registration_ransac_based_on_feature_matching as the reference
// calls it (core/deep_global_registration.py:29-47), restated in oracle/ransac_fm.py.  Hypothesis h draws
// 4 SOURCE points with ransac_pick and pairs each with its nearest target feature (nn, computed once by the
// caller); the checkers run before / after the fp64 Umeyama fit; the first max_validation hypotheses that
// pass every checker are scored on ALL source points (nearest target point strictly within max_dist of
// R s + t, through the target's voxel hash).  Five launches, no host read:
//   fm_hypothesis_kernel  one thread per hypothesis: draw, edge checker, fit, distance checker -> flag, pose
//   dgr_scan_counts       exclusive scan of the per-block validated counts (coords.cu)
//   dgr_select_first      the first V validated hypothesis numbers, in hypothesis order (coords.cu)
//   fm_score_kernel       (selected hypothesis x 1024-point chunk) per block, 8 lanes per point
//                         (dgr_voxel_nearest8, shared with the ICP); fixed-order block partials
//   fm_final_kernel       partials summed in chunk order, best by (count, smaller sum d^2, lower h)
// The scoring is fp64 end to end and its partials are reduced in a fixed order, so the (count, sum d^2)
// a hypothesis is ranked by are the numbers the result reports, and a call is bit-reproducible.
// ---------------------------------------------------------------------------------------
constexpr int kFmThreads = 256;
constexpr int kFmChunk = 1024;          // source points per scoring block: 32 groups of 8 lanes x 32 rounds
constexpr int64_t kFmMaxChunks = 65535; // gridDim.y of the scoring launch

struct FmWs {
  double* pose;       // [M][12] row-major [R | t] of every hypothesis that reached the fit
  int32_t* flag;      // [M] passed every checker
  int32_t* blk;       // [n_hblk + 1] validated per hypothesis block -> exclusive offsets; [n_hblk] = total
  int32_t* sel;       // [Vc] selected hypothesis numbers
  double* part;       // [Vc][n_chunk][2] (matched, sum d^2) per scoring block
};

// workspace size in 8-byte words; carves `base` into the regions when it is not null
int64_t fm_layout(int64_t n_src, int64_t M, int64_t V, uint64_t* base, FmWs* w) {
  const int64_t Vc = V < M ? V : M;
  const int64_t n_hblk = (M + kFmThreads - 1) / kFmThreads;
  const int64_t n_chunk = (n_src + kFmChunk - 1) / kFmChunk;
  DgrCarver c(base);
  FmWs r;
  r.pose = c.take<double>(12 * M);
  r.flag = c.take<int32_t>(M);
  r.blk = c.take<int32_t>(n_hblk + 1);
  r.sel = c.take<int32_t>(Vc);
  r.part = c.take<double>(2 * Vc * n_chunk);
  if (w != nullptr) *w = r;
  return c.words;
}

__global__ void __launch_bounds__(kFmThreads)
fm_hypothesis_kernel(const float* __restrict__ src, uint32_t n_src, const float* __restrict__ tgt,
                     const int32_t* __restrict__ nn, uint64_t seed, int64_t M, double edge_ratio, double check_dist,
                     double* __restrict__ pose, int32_t* __restrict__ flag, int32_t* __restrict__ blk_cnt) {
  const int64_t h = (int64_t)blockIdx.x * kFmThreads + threadIdx.x;
  int ok = 0;
  if (h < M) {
    double p[4][3], q[4][3];
    for (int j = 0; j < 4; ++j) {
      const int64_t i = ransac_pick(seed, (uint64_t)h, j, n_src);
      const int64_t k = __ldg(nn + i);
      for (int c = 0; c < 3; ++c) { p[j][c] = __ldg(src + 3 * i + c); q[j][c] = __ldg(tgt + 3 * k + c); }
    }
    ok = 1;
    // CorrespondenceCheckerBasedOnEdgeLength: every edge of the sample similar in length on both sides
    if (edge_ratio > 0) {
      for (int a = 1; a < 4; ++a)
        for (int b = 0; b < a; ++b) {
          double ds = 0, dt = 0;
          for (int c = 0; c < 3; ++c) {
            ds += (p[a][c] - p[b][c]) * (p[a][c] - p[b][c]);
            dt += (q[a][c] - q[b][c]) * (q[a][c] - q[b][c]);
          }
          ds = sqrt(ds);
          dt = sqrt(dt);
          if (ds < edge_ratio * dt || dt < edge_ratio * ds) ok = 0;
        }
    }
    if (ok) {
      double R[3][3], t[3];
      ransac_fit4(p, q, R, t);
      // CorrespondenceCheckerBasedOnDistance: every sampled pair within check_dist after alignment
      if (check_dist > 0) {
        for (int j = 0; j < 4; ++j) {
          double e2 = 0;
          for (int r = 0; r < 3; ++r) {
            const double e = R[r][0] * p[j][0] + R[r][1] * p[j][1] + R[r][2] * p[j][2] + t[r] - q[j][r];
            e2 += e * e;
          }
          if (sqrt(e2) > check_dist) ok = 0;
        }
      }
      double* T = pose + 12 * h;
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) T[4 * r + c] = R[r][c];
        T[4 * r + 3] = t[r];
      }
    }
    flag[h] = ok;
  }
  const int cnt = __syncthreads_count(ok);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = cnt;
}

__global__ void __launch_bounds__(kFmThreads, 4)   // <= 64 registers: 32 warps per SM hide the probe latency
fm_score_kernel(const float* __restrict__ src, int64_t n_src, const float* __restrict__ tgt,
                const dgr_keyspec_t* __restrict__ spec_p, const uint64_t* __restrict__ keys,
                const int32_t* __restrict__ vals, uint64_t mask, int32_t batch, double cell, double max_dist,
                const double* __restrict__ pose, const int32_t* __restrict__ sel, const int32_t* __restrict__ n_valid,
                int64_t Vc, double* __restrict__ part) {
  const int64_t slot = blockIdx.x;
  if (slot >= min((int64_t)*n_valid, Vc)) return;      // uniform per block
  const dgr_keyspec_t s = *spec_p;
  double T[12];
  const double* Tp = pose + 12 * (int64_t)sel[slot];
#pragma unroll
  for (int k = 0; k < 12; ++k) T[k] = __ldg(Tp + k);
  const int reach = (int)ceil(max_dist / cell);
  const int sub = threadIdx.x & 7;
  const int64_t lo = (int64_t)blockIdx.y * kFmChunk, hi = min(n_src, lo + kFmChunk);
  const int64_t end = lo + ((hi - lo + kFmThreads / 8 - 1) / (kFmThreads / 8)) * (kFmThreads / 8);
  uint32_t cnt = 0;
  double err = 0.0;
  for (int64_t i0 = lo + (threadIdx.x >> 3); i0 < end; i0 += kFmThreads / 8) {
    const bool have = i0 < hi;                         // whole warps stay in the loop for the shuffles
    const int64_t i = have ? i0 : lo;
    const double x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
    const double p[3] = {T[0] * x + T[1] * y + T[2] * z + T[3], T[4] * x + T[5] * y + T[6] * z + T[7],
                         T[8] * x + T[9] * y + T[10] * z + T[11]};
    double best = max_dist * max_dist;
    int best_j;
    dgr_voxel_nearest8(p, have, sub, tgt, s, keys, vals, mask, batch, cell, reach, best, best_j);
    if (have && sub == 0 && best_j >= 0) {
      ++cnt;
      err += best;
    }
  }
  // fixed reduction order (butterfly, then warps in order): the partial does not depend on scheduling
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    err += __shfl_xor_sync(0xffffffffu, err, d);
  }
  __shared__ uint32_t s_cnt[kFmThreads / 32];
  __shared__ double s_err[kFmThreads / 32];
  if ((threadIdx.x & 31) == 0) { s_cnt[threadIdx.x >> 5] = cnt; s_err[threadIdx.x >> 5] = err; }
  __syncthreads();
  if (threadIdx.x == 0) {
    cnt = 0;
    err = 0.0;
    for (int w = 0; w < kFmThreads / 32; ++w) { cnt += s_cnt[w]; err += s_err[w]; }
    double* o = part + 2 * (slot * gridDim.y + blockIdx.y);
    o[0] = (double)cnt;
    o[1] = err;
  }
}

// (c2, e2, s2) ranks before (c1, e1, s1): open3d's IsBetterRANSACThan with the earlier hypothesis keeping a
// tie; slot -1 = nothing (open3d's initial result, fitness 0, which no hypothesis without a match beats)
__device__ __forceinline__ bool fm_better(double c2, double e2, int s2, double c1, double e1, int s1) {
  return s2 >= 0 && (s1 < 0 || c2 > c1 || (c2 == c1 && (e2 < e1 || (e2 == e1 && s2 < s1))));
}

__global__ void __launch_bounds__(1024)
fm_final_kernel(const double* __restrict__ pose, const int32_t* __restrict__ sel, const int32_t* __restrict__ n_valid,
                int64_t Vc, int64_t V, int64_t M, int64_t n_chunk, const double* __restrict__ part, int64_t n_src,
                double* __restrict__ result) {
  __shared__ double s_c[32], s_e[32];
  __shared__ int s_s[32];
  const int total = *n_valid;
  const int64_t nv = min((int64_t)total, Vc);
  double bc = 0, be = 0;
  int bs = -1;
  for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) {
    double c = 0, e = 0;
    for (int64_t k = 0; k < n_chunk; ++k) {
      c += part[2 * (v * n_chunk + k)];
      e += part[2 * (v * n_chunk + k) + 1];
    }
    if (c > 0 && fm_better(c, e, (int)v, bc, be, bs)) { bc = c; be = e; bs = (int)v; }
  }
  for (int d = 16; d > 0; d >>= 1) {
    const double oc = __shfl_xor_sync(0xffffffffu, bc, d), oe = __shfl_xor_sync(0xffffffffu, be, d);
    const int os = __shfl_xor_sync(0xffffffffu, bs, d);
    if (fm_better(oc, oe, os, bc, be, bs)) { bc = oc; be = oe; bs = os; }
  }
  if ((threadIdx.x & 31) == 0) { s_c[threadIdx.x >> 5] = bc; s_e[threadIdx.x >> 5] = be; s_s[threadIdx.x >> 5] = bs; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
    if (fm_better(s_c[w], s_e[w], s_s[w], bc, be, bs)) { bc = s_c[w]; be = s_e[w]; bs = s_s[w]; }
  const int64_t h = bs >= 0 ? (int64_t)sel[bs] : -1;
  for (int k = 0; k < 12; ++k) result[k] = h >= 0 ? pose[12 * h + k] : (k % 5 == 0 ? 1.0 : 0.0);
  result[12] = 0; result[13] = 0; result[14] = 0; result[15] = 1;
  result[16] = bs >= 0 ? bc / (double)n_src : 0.0;         // fitness
  result[17] = bs >= 0 ? sqrt(be / bc) : 0.0;              // inlier RMSE
  result[18] = (double)h;                                  // winning hypothesis
  result[19] = bc;                                         // matched source points
  result[20] = (double)nv;                                 // validated hypotheses scored
  result[21] = total >= V ? (double)(sel[V - 1] + 1) : (double)M;   // drawn until the V-th validation
  for (int k = 22; k < 24; ++k) result[k] = 0;
}

}  // namespace

extern "C" {

int32_t dgr_ransac_ws_elems(int64_t n_corr, int64_t num_hyp, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_corr >= 0 && num_hyp >= 0, "bad arguments");
  *n_elems = ransac_layout(n_corr, num_hyp, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_ransac_correspondence(const float* x, const float* y, const int32_t* idx0, const int32_t* idx1,
                                  int64_t n_corr, double max_dist, int64_t num_hyp, uint64_t seed, uint64_t* ws,
                                  double* result, void* stream) {
  DGR_ARG_CHECK(x != nullptr && y != nullptr && ws != nullptr && result != nullptr, "null pointer");
  DGR_ARG_CHECK(n_corr >= 1 && n_corr < (1ll << 31), "correspondence count out of range");
  DGR_ARG_CHECK(num_hyp >= 1 && num_hyp <= (1ll << 40), "hypothesis count out of range");
  DGR_ARG_CHECK(max_dist > 0, "max_dist must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  RansacWs w;
  ransac_layout(n_corr, num_hyp, ws, &w);
  const uint32_t n_blk = ransac_blocks(num_hyp);
  ransac_pack_kernel<<<dgr_blocks(n_corr, 256), 256, 0, st>>>(x, y, idx0, idx1, n_corr, w.src, w.tgt);
  ransac_eval_kernel<<<n_blk, kRansacThreads, 0, st>>>(w.src, w.tgt, (uint32_t)n_corr, seed, (uint64_t)num_hyp,
                                                       (float)(max_dist * max_dist), w.blk_key, w.blk_hyp);
  ransac_final_kernel<<<1, 1024, 0, st>>>(w.src, w.tgt, (uint32_t)n_corr, seed, w.blk_key, w.blk_hyp, n_blk, max_dist,
                                          result);
  dgr_note_launches(3);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_ransac_fm_ws_elems(int64_t n_src, int64_t max_iteration, int64_t max_validation, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0 && max_iteration >= 0 && max_validation >= 0, "bad arguments");
  *n_elems = fm_layout(n_src, max_iteration, max_validation, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_ransac_feature_matching(const float* src, int64_t n_src, const float* tgt, const int32_t* nn,
                                    const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals, int64_t cap,
                                    int32_t batch, double cell, double max_dist, double edge_ratio, double check_dist,
                                    int64_t max_iteration, int64_t max_validation, uint64_t seed, uint64_t* ws,
                                    double* result, void* stream) {
  DGR_ARG_CHECK(src != nullptr && tgt != nullptr && nn != nullptr && spec != nullptr && keys != nullptr &&
                vals != nullptr && ws != nullptr && result != nullptr, "null pointer");
  DGR_ARG_CHECK(n_src >= 1 && n_src <= kFmChunk * kFmMaxChunks, "source point count out of range");
  DGR_ARG_CHECK(max_iteration >= 1 && max_iteration <= (1ll << 30), "hypothesis count out of range");
  DGR_ARG_CHECK(max_validation >= 1, "max_validation must be positive");
  DGR_TRY(dgr_check_hash_search(cap, cell, max_dist, 4));
  DGR_ARG_CHECK(edge_ratio >= 0, "edge_ratio must be >= 0 (0 = no edge-length checker)");
  cudaStream_t st = (cudaStream_t)stream;
  FmWs w;
  fm_layout(n_src, max_iteration, max_validation, ws, &w);
  const int64_t Vc = max_validation < max_iteration ? max_validation : max_iteration;
  const uint32_t n_hblk = (uint32_t)((max_iteration + kFmThreads - 1) / kFmThreads);
  const int64_t n_chunk = (n_src + kFmChunk - 1) / kFmChunk;
  fm_hypothesis_kernel<<<n_hblk, kFmThreads, 0, st>>>(src, (uint32_t)n_src, tgt, nn, seed, max_iteration, edge_ratio,
                                                      check_dist, w.pose, w.flag, w.blk);
  dgr_scan_counts(w.blk, n_hblk, st);
  dgr_select_first(w.flag, w.blk, max_iteration, Vc, 0, w.sel, nullptr, st);
  fm_score_kernel<<<dim3((unsigned)Vc, (unsigned)n_chunk), kFmThreads, 0, st>>>(
      src, n_src, tgt, spec, keys, vals, (uint64_t)cap - 1, batch, cell, max_dist, w.pose, w.sel, w.blk + n_hblk, Vc,
      w.part);
  fm_final_kernel<<<1, 1024, 0, st>>>(w.pose, w.sel, w.blk + n_hblk, Vc, max_validation, max_iteration, n_chunk, w.part,
                                      n_src, result);
  dgr_note_launches(5);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
