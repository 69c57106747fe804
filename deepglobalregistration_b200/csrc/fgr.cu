// Fast Global Registration (Zhou, Park & Koltun, ECCV 2016) over feature matches: open3d's
// registration_fast_based_on_feature_matching, restated in oracle/fgr.py (which pins every boundary convention).
// The caller supplies both feature kNN directions (dgr_knn_top1 / dgr_knn_top1_tc); the rest runs here with no
// host read and no atomics, so a call gives the same bits on every run:
//   dgr_cloud_stats     one CTA per cloud: fp64 mean and max |x - mean| in a fixed order (frame.cu)
//   fgr_mutual_kernel   one thread per row of the larger cloud ("first"; the source on a tie): mutual flag
//   dgr_scan_counts     exclusive scan of the per-block counts (coords.cu); [nb] = n_mut
//   dgr_select_first    the mutual list in first-cloud order (coords.cu, shared with the RANSAC)
//   per chunk of kFgrChunk tuple trials (grids sized from the host bound 100 min(n_s, n_t)):
//     fgr_tuple_kernel       one thread per trial: 3 counter-hash draws, the three edge-ratio tests
//     fgr_tuple_scan_kernel  scan offset by the acceptances so far; marks the chunk dead once K are in
//     dgr_select_first       the first K accepted trials, in trial order
//   Every kernel of a chunk that starts after the K-th acceptance (or past 100 n_mut) returns at once, and the
//   workspace is one chunk's flags whatever the trial count.
//   fgr_solve_kernel    one launch for all iterations: one CTA (a cluster of 8 when the mutual list is long and
//                       the tuple test is off); J^T J / J^T r reduced in a fixed order, the 6x6 Cholesky on one
//                       thread, the pose kept in shared memory.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "frame.cuh"
#include "kabsch.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kFgrThreads = 256;                        // flag kernels (dgr_select_first's blocks)
constexpr int64_t kFgrChunk = 1 << 18;                  // tuple trials per chunk
constexpr int kFgrChunkBlocks = (int)(kFgrChunk / kFgrThreads);
constexpr int kFgrSolveThreads = 512;
constexpr int kFgrCluster = 8;
constexpr int64_t kFgrClusterMin = 16384;               // mutual-list bound from which the solver runs on a cluster
constexpr int kNv = 27;                                 // J^T J upper triangle (21) + J^T r (6)

struct FgrWs {
  double* stat;      // [2][4] per cloud: mean xyz, max |x - mean|
  int32_t* mflag;    // [n_first] mutual flag per first-cloud row
  int32_t* mblk;     // [n_mblk + 1] per-block counts -> exclusive offsets; [n_mblk] = n_mut
  int32_t* mut;      // [n_min] first-cloud rows of the mutual pairs, ascending
  int32_t* tflag;    // [kFgrChunk] accepted flag of the current chunk's trials
  int32_t* tblk;     // [kFgrChunkBlocks + 1]
  int32_t* tsel;     // [Kc] accepted trial numbers, in order
  int32_t* tstate;   // [2] accepted so far, current chunk live
  double* corr;      // [n_corr_max][6] normalised (source, target) points of the correspondences
};

// K capped by the trial count bound: at most 100 min(n_s, n_t) trials exist
inline int64_t fgr_kc(int64_t n_min, int64_t K) { return K < 100 * n_min ? K : 100 * n_min; }

inline int64_t fgr_corr_max(int64_t n_min, int64_t K, int tuple_test) {
  return tuple_test ? 3 * fgr_kc(n_min, K) : n_min;
}

// workspace size in 8-byte words; carves `base` into the regions when it is not null
int64_t fgr_layout(int64_t n_src, int64_t n_tgt, int64_t K, int tuple_test, uint64_t* base, FgrWs* w) {
  const int64_t n_first = n_src > n_tgt ? n_src : n_tgt, n_min = n_src < n_tgt ? n_src : n_tgt;
  const int64_t n_mblk = (n_first + kFgrThreads - 1) / kFgrThreads;
  const int64_t t = tuple_test ? 1 : 0;
  DgrCarver c(base);
  FgrWs r;
  r.stat = c.take<double>(8);
  r.mflag = c.take<int32_t>(n_first);
  r.mblk = c.take<int32_t>(n_mblk + 1);
  r.mut = c.take<int32_t>(n_min);
  r.tflag = c.take<int32_t>(t * kFgrChunk);
  r.tblk = c.take<int32_t>(t * (kFgrChunkBlocks + 1));
  r.tsel = c.take<int32_t>(t * fgr_kc(n_min, K));
  r.tstate = c.take<int32_t>(2);
  r.corr = c.take<double>(6 * fgr_corr_max(n_min, K, tuple_test));
  if (w != nullptr) *w = r;
  return c.words;
}

// the normalisation of oracle/fgr.py::normalise: x -> (x - mean) / scale
struct FgrFrame {
  double ms[3], mt[3];
  double s;          // largest |x - mean| over both clouds (1 when both clouds are a single point)
  double scale;      // s, or 1 with use_absolute_scale
};

__device__ __forceinline__ FgrFrame fgr_frame(const double* __restrict__ stat, int absolute) {
  FgrFrame f;
  for (int c = 0; c < 3; ++c) { f.ms[c] = stat[c]; f.mt[c] = stat[4 + c]; }
  f.s = dgr_frame_scale(stat);
  f.scale = absolute ? 1.0 : f.s;
  return f;
}

// (source row, target row) of the mutual pair whose first-cloud row is f
__device__ __forceinline__ void fgr_pair(int32_t f, int swapped, const int32_t* __restrict__ nn_st,
                                         const int32_t* __restrict__ nn_ts, int32_t& i, int32_t& j) {
  if (swapped) { j = f; i = __ldg(nn_ts + f); }
  else { i = f; j = __ldg(nn_st + f); }
}

__global__ void __launch_bounds__(kFgrThreads)
fgr_mutual_kernel(const int32_t* __restrict__ nn_first, const int32_t* __restrict__ nn_other, int64_t n_first,
                  int64_t n_other, int32_t* __restrict__ flag, int32_t* __restrict__ blk, int32_t* __restrict__ tstate) {
  const int64_t f = (int64_t)blockIdx.x * kFgrThreads + threadIdx.x;
  if (f == 0) { tstate[0] = 0; tstate[1] = 0; }     // no trial accepted yet, for the tuple chunks that follow
  int ok = 0;
  if (f < n_first) {
    const int32_t j = __ldg(nn_first + f);
    ok = j >= 0 && j < n_other && __ldg(nn_other + j) == f;
    flag[f] = ok;
  }
  const int cnt = __syncthreads_count(ok);
  if (threadIdx.x == 0) blk[blockIdx.x] = cnt;
}

// trials [h0, h0 + kFgrChunk) of 100 n_mut: trial k draws list positions 3k .. 3k + 2 of the counter hash and is
// accepted when every edge satisfies l_s tuple_scale < l_t < l_s / tuple_scale on the normalised points
__global__ void __launch_bounds__(kFgrThreads)
fgr_tuple_kernel(const float* __restrict__ src, const float* __restrict__ tgt, const int32_t* __restrict__ nn_st,
                 const int32_t* __restrict__ nn_ts, int swapped, const int32_t* __restrict__ mut,
                 const int32_t* __restrict__ n_mut_p, const double* __restrict__ stat, int absolute, uint64_t seed,
                 int64_t h0, double tuple_scale, int64_t Kc, const int32_t* __restrict__ tstate,
                 int32_t* __restrict__ flag, int32_t* __restrict__ blk) {
  const int64_t n_mut = *n_mut_p;
  const int64_t n_trials = n_mut >= 3 ? 100 * n_mut : 0;
  if (tstate[0] >= Kc || h0 >= n_trials) return;        // uniform per launch: K accepted, or no trial left
  const int64_t local = (int64_t)blockIdx.x * kFgrThreads + threadIdx.x, k = h0 + local;
  int ok = 0;
  if (k < n_trials) {
    const FgrFrame fr = fgr_frame(stat, absolute);
    double p[3][3], q[3][3];
    for (int s = 0; s < 3; ++s) {
      const uint32_t pos = dgr_counter_pick(seed, 3 * (uint64_t)k + s, (uint32_t)n_mut);
      int32_t i, j;
      fgr_pair(__ldg(mut + pos), swapped, nn_st, nn_ts, i, j);
      dgr_frame_point(src, i, fr.ms, fr.scale, p[s]);
      dgr_frame_point(tgt, j, fr.mt, fr.scale, q[s]);
    }
    ok = 1;
    for (int e = 0; e < 3; ++e) {
      const int a = e, b = e == 2 ? 0 : e + 1;
      const double ls = dgr_dist3(p[a], p[b]), lt = dgr_dist3(q[a], q[b]);
      if (!(ls * tuple_scale < lt && lt < ls / tuple_scale)) ok = 0;
    }
  }
  flag[local] = ok;
  const int cnt = __syncthreads_count(ok);
  if (threadIdx.x == 0) blk[blockIdx.x] = cnt;
}

// exclusive offsets of this chunk's blocks, shifted by the acceptances of the earlier chunks
__global__ void __launch_bounds__(1024)
fgr_tuple_scan_kernel(int32_t* __restrict__ blk, const int32_t* __restrict__ n_mut_p, int64_t h0, int64_t Kc,
                      int32_t* __restrict__ tstate) {
  const int64_t n_mut = *n_mut_p;
  const int64_t n_trials = n_mut >= 3 ? 100 * n_mut : 0;
  const int acc = tstate[0];                            // read by every thread before thread 0 rewrites it below
  const int live = acc < Kc && h0 < n_trials;
  if (!live) {
    if (threadIdx.x == 0) tstate[1] = 0;
    return;
  }
  const int total = dgr_block_scan_inplace(blk, kFgrChunkBlocks);
  for (int b = threadIdx.x; b < kFgrChunkBlocks; b += blockDim.x) blk[b] += acc;
  if (threadIdx.x == 0) {
    tstate[0] = acc + total;
    tstate[1] = 1;
  }
}

struct FgrShared {
  DgrReduceShared<kNv, kFgrSolveThreads, kFgrCluster> red;
  double T[12];                                         // target -> source in normalised units, row-major [R | t]
};

template <int CS>
__global__ void __launch_bounds__(kFgrSolveThreads, 1)
fgr_solve_kernel(const float* __restrict__ src, const float* __restrict__ tgt, const int32_t* __restrict__ nn_st,
                 const int32_t* __restrict__ nn_ts, int swapped, const int32_t* __restrict__ mut,
                 const int32_t* __restrict__ n_mut_p, const int32_t* __restrict__ tsel,
                 const int32_t* __restrict__ tstate, int64_t Kc, int tuple_test, const double* __restrict__ stat,
                 int absolute, uint64_t seed, int iteration_number, int decrease_mu, double division_factor,
                 double max_corr_dist, double* __restrict__ corr, int32_t* __restrict__ corres_out,
                 double* __restrict__ result) {
  __shared__ FgrShared sh;
  unsigned rank = 0;
  if constexpr (CS > 1) rank = cg::this_cluster().block_rank();
  const int tid = threadIdx.x;
  const int64_t n_mut = *n_mut_p;
  int64_t n_corr, drawn;
  if (tuple_test) {
    const int64_t acc = n_mut >= 3 ? min((int64_t)tstate[0], Kc) : 0;
    n_corr = 3 * acc;
    drawn = n_mut < 3 ? 0 : ((int64_t)tstate[0] >= Kc ? (int64_t)tsel[Kc - 1] + 1 : 100 * n_mut);
  } else {
    n_corr = n_mut;
    drawn = 0;
  }
  const FgrFrame fr = fgr_frame(stat, absolute);
  // the normalised correspondences, once; a thread later reads exactly the entries it wrote here
  const int64_t G = (int64_t)CS * kFgrSolveThreads, g0 = (int64_t)rank * kFgrSolveThreads + tid;
  for (int64_t k = g0; k < n_corr; k += G) {
    const int64_t pos = tuple_test ? (int64_t)dgr_counter_pick(seed, 3 * (uint64_t)tsel[k / 3] + k % 3, (uint32_t)n_mut)
                                   : k;
    int32_t i, j;
    fgr_pair(mut[pos], swapped, nn_st, nn_ts, i, j);
    dgr_frame_point(src, i, fr.ms, fr.scale, corr + 6 * k);
    dgr_frame_point(tgt, j, fr.mt, fr.scale, corr + 6 * k + 3);
    if (corres_out != nullptr) { corres_out[2 * k] = i; corres_out[2 * k + 1] = j; }
  }
  if (tid < 12) sh.T[tid] = (tid % 5 == 0) ? 1.0 : 0.0;
  __syncthreads();
  double mu = absolute ? fr.s : 1.0;
  const int ran = n_corr >= 10;
  int parity = 0;
  for (int itr = 0; ran && itr < iteration_number; ++itr) {
    if (decrease_mu && itr % 4 == 0 && mu > max_corr_dist) mu /= division_factor;
    double T[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) T[k] = sh.T[k];
    double v[kNv];
#pragma unroll
    for (int k = 0; k < kNv; ++k) v[k] = 0.0;
    for (int64_t k = g0; k < n_corr; k += G) {
      const double* c = corr + 6 * k;
      const double p[3] = {c[0], c[1], c[2]};
      double q[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) q[r] = T[4 * r] * c[3] + T[4 * r + 1] * c[4] + T[4 * r + 2] * c[5] + T[4 * r + 3];
      const double rv[3] = {p[0] - q[0], p[1] - q[1], p[2] - q[2]};
      const double tmp = mu / (rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2] + mu);
      const double w = tmp * tmp;
      // d(p - (R q + t)) / d(alpha, beta, gamma, t) at the current q, one row per residual component
      const double J[3][6] = {{0.0, -q[2], q[1], -1.0, 0.0, 0.0},
                              {q[2], 0.0, -q[0], 0.0, -1.0, 0.0},
                              {-q[1], q[0], 0.0, 0.0, 0.0, -1.0}};
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        int m = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
#pragma unroll
          for (int b = a; b < 6; ++b) { v[m] += w * J[r][a] * J[r][b]; ++m; }
          v[21 + a] += w * J[r][a] * rv[r];
        }
      }
    }
    dgr_allreduce<CS>(sh.red, v, parity);
    if (tid == 0) {
      double x[6];
      if (!cholesky6_step(sh.red.tot, sh.red.tot + 21, x))
        for (int k = 0; k < 6; ++k) x[k] = 0.0;
      zyx_update_left(x, T, sh.T);                      // delta = [Rz(gamma) Ry(beta) Rx(alpha) | x[3..6)], on the left
    }
    __syncthreads();
  }
  if constexpr (CS > 1) cg::this_cluster().sync();      // nobody exits while peers may still write its slots
  if (rank != 0 || tid != 0) return;
  // target -> source in the input frame: [R | -R m_t + scale t + m_s]; the result is its inverse
  double R[3][3], t[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) R[r][c] = sh.T[4 * r + c];
    t[r] = -(R[r][0] * fr.mt[0] + R[r][1] * fr.mt[1] + R[r][2] * fr.mt[2]) + fr.scale * sh.T[4 * r + 3] + fr.ms[r];
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) result[4 * r + c] = R[c][r];
    result[4 * r + 3] = -(R[0][r] * t[0] + R[1][r] * t[1] + R[2][r] * t[2]);
  }
  result[12] = 0; result[13] = 0; result[14] = 0; result[15] = 1;
  result[16] = (double)n_mut;
  result[17] = (double)n_corr;
  result[18] = (double)drawn;
  result[19] = mu;
  result[20] = ran;
  result[21] = swapped;
  result[22] = 0;
  result[23] = 0;
}

}  // namespace

extern "C" {

int32_t dgr_fgr_ws_elems(int64_t n_src, int64_t n_tgt, int64_t maximum_tuple_count, int32_t tuple_test,
                         int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0 && n_tgt >= 0 && maximum_tuple_count >= 0, "bad arguments");
  *n_elems = fgr_layout(n_src, n_tgt, maximum_tuple_count, tuple_test != 0, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_fgr_feature_matching(const float* src, int64_t n_src, const float* tgt, int64_t n_tgt,
                                 const int32_t* nn_st, const int32_t* nn_ts, double division_factor,
                                 int32_t use_absolute_scale, int32_t decrease_mu,
                                 double maximum_correspondence_distance, int32_t iteration_number,
                                 double tuple_scale, int64_t maximum_tuple_count, int32_t tuple_test, uint64_t seed,
                                 uint64_t* ws, int32_t* corres_out, double* result, void* stream) {
  DGR_ARG_CHECK(src != nullptr && tgt != nullptr && nn_st != nullptr && nn_ts != nullptr && ws != nullptr &&
                result != nullptr, "null pointer");
  DGR_ARG_CHECK(n_src >= 1 && n_tgt >= 1, "both clouds need a point");
  const int64_t n_min = n_src < n_tgt ? n_src : n_tgt, n_first = n_src < n_tgt ? n_tgt : n_src;
  DGR_ARG_CHECK(n_first < (1ll << 31) && 100 * n_min < (1ll << 31), "point count out of range");
  DGR_ARG_CHECK(division_factor > 1.0, "division_factor must be > 1");
  DGR_ARG_CHECK(maximum_correspondence_distance > 0.0, "maximum_correspondence_distance must be positive");
  DGR_ARG_CHECK(iteration_number >= 0, "iteration_number must be >= 0");
  DGR_ARG_CHECK(tuple_scale > 0.0 && tuple_scale <= 1.0, "tuple_scale must lie in (0, 1]");
  DGR_ARG_CHECK(maximum_tuple_count >= 1 && maximum_tuple_count <= (1ll << 30), "maximum_tuple_count out of range");
  cudaStream_t st = (cudaStream_t)stream;
  const int tt = tuple_test != 0, absolute = use_absolute_scale != 0, swapped = n_tgt > n_src;
  FgrWs w;
  fgr_layout(n_src, n_tgt, maximum_tuple_count, tt, ws, &w);
  const int64_t Kc = fgr_kc(n_min, maximum_tuple_count);
  const unsigned n_mblk = dgr_blocks(n_first, kFgrThreads);
  int launches = 0;
  dgr_cloud_stats(src, n_src, tgt, n_tgt, w.stat, st);
  fgr_mutual_kernel<<<n_mblk, kFgrThreads, 0, st>>>(swapped ? nn_ts : nn_st, swapped ? nn_st : nn_ts, n_first, n_min,
                                                    w.mflag, w.mblk, w.tstate);
  dgr_scan_counts(w.mblk, n_mblk, st);
  dgr_select_first(w.mflag, w.mblk, n_first, n_min, 0, w.mut, nullptr, st);
  launches += 4;
  const int32_t* n_mut = w.mblk + n_mblk;
  if (tt && n_min >= 3) {
    for (int64_t h0 = 0; h0 < 100 * n_min; h0 += kFgrChunk) {
      fgr_tuple_kernel<<<kFgrChunkBlocks, kFgrThreads, 0, st>>>(src, tgt, nn_st, nn_ts, swapped, w.mut, n_mut, w.stat,
                                                                 absolute, seed, h0, tuple_scale, Kc, w.tstate,
                                                                 w.tflag, w.tblk);
      fgr_tuple_scan_kernel<<<1, 1024, 0, st>>>(w.tblk, n_mut, h0, Kc, w.tstate);
      dgr_select_first(w.tflag, w.tblk, kFgrChunk, Kc, h0, w.tsel, w.tstate + 1, st);
      launches += 3;
    }
  }
  const bool clustered = !tt && n_min >= kFgrClusterMin;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.gridDim = dim3(clustered ? kFgrCluster : 1);
  cfg.blockDim = dim3(kFgrSolveThreads);
  cfg.stream = st;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = clustered ? kFgrCluster : 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = clustered ? 1 : 0;
  if (clustered)
    DGR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, fgr_solve_kernel<kFgrCluster>, src, tgt, nn_st, nn_ts, swapped,
                                      (const int32_t*)w.mut, n_mut, (const int32_t*)w.tsel, (const int32_t*)w.tstate,
                                      Kc, tt, (const double*)w.stat, absolute, seed, (int)iteration_number,
                                      (int)(decrease_mu != 0), division_factor, maximum_correspondence_distance,
                                      w.corr, corres_out, result));
  else
    fgr_solve_kernel<1><<<1, kFgrSolveThreads, 0, st>>>(src, tgt, nn_st, nn_ts, swapped, w.mut, n_mut, w.tsel,
                                                         w.tstate, Kc, tt, w.stat, absolute, seed, iteration_number,
                                                         decrease_mu != 0, division_factor,
                                                         maximum_correspondence_distance, w.corr, corres_out, result);
  launches += 1;
  dgr_note_launches(launches);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
