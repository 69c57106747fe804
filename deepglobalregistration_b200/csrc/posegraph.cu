// Multiway registration: open3d's GetInformationMatrixFromPointClouds and GlobalOptimization with
// GlobalOptimizationLevenbergMarquardt, restated in oracle/pose_graph.py (which states every reading of open3d).
//   info_match_kernel   8 lanes per source point: the nearest target point q strictly within max_dist of T s
//                       (dgr_voxel_nearest8, the rule of dgr_icp); the ten sums count, sum q, sum q q^T as per-CTA
//                       partials (dgr_block_sum)
//   info_final_kernel   the partials added in a fixed order; the closed-form 6x6 information matrix and the count
//   pose_graph_kernel   one CTA for the whole optimisation (both LM passes, the pruning, the compensation): one
//                       thread per edge for residuals and Jacobian blocks, the 6x6 blocks of H summed per node and
//                       per node pair in edge order (incidence lists built on the host), a damped right-looking
//                       blocked Cholesky of the dense padded H in global memory (L2-resident), two blocked triangular
//                       solves, fixed-order block sums for the costs.  No atomics and no host read inside the loop:
//                       the same bits on every run, and the result comes back in one copy.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "kabsch.cuh"

namespace {

constexpr int kInfoThreads = 256;
constexpr int kInfoMaxBlocks = 2368;
constexpr int kInfoNv = 10;                             // count, sum q (3), sum q q^T (xx, xy, xz, yy, yz, zz)
constexpr int kPgThreads = 512;
constexpr int kPgWarps = kPgThreads / 32;
constexpr int kPgNb = 32;                               // Cholesky panel width
constexpr int kPgStats = DGR_POSE_GRAPH_STATS;

// ---------------------------------------------------------------------------------------
// information matrix
// ---------------------------------------------------------------------------------------
struct Pose12 {
  double m[12];                                         // row-major [R | t]
};

__global__ void __launch_bounds__(kInfoThreads)
info_match_kernel(const float* __restrict__ src, int64_t n_src, const float* __restrict__ tgt,
                  const dgr_keyspec_t* __restrict__ spec_p, const uint64_t* __restrict__ keys,
                  const int32_t* __restrict__ vals, uint64_t mask, int32_t batch, double cell, int reach,
                  double max_dist, Pose12 T, double* __restrict__ part) {
  const dgr_keyspec_t s = *spec_p;
  double v[kInfoNv];
#pragma unroll
  for (int k = 0; k < kInfoNv; ++k) v[k] = 0.0;
  const int sub = threadIdx.x & 7;
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) >> 3;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3; i0 < ((n_src + groups - 1) / groups) * groups;
       i0 += groups) {
    const bool have = i0 < n_src;                       // whole warps stay in the loop for the shuffles
    const int64_t i = have ? i0 : 0;
    const double x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
    const double* M = T.m;
    const double p[3] = {M[0] * x + M[1] * y + M[2] * z + M[3], M[4] * x + M[5] * y + M[6] * z + M[7],
                         M[8] * x + M[9] * y + M[10] * z + M[11]};
    double best = max_dist * max_dist;
    int best_j;
    dgr_voxel_nearest8(p, have, sub, tgt, s, keys, vals, mask, batch, cell, reach, best, best_j);
    if (have && best_j >= 0 && sub == 0) {              // one lane of the group adds the match
      const int64_t j = best_j;
      const double q[3] = {tgt[3 * j], tgt[3 * j + 1], tgt[3 * j + 2]};
      v[0] += 1.0;
      v[1] += q[0]; v[2] += q[1]; v[3] += q[2];
      v[4] += q[0] * q[0]; v[5] += q[0] * q[1]; v[6] += q[0] * q[2];
      v[7] += q[1] * q[1]; v[8] += q[1] * q[2]; v[9] += q[2] * q[2];
    }
  }
  __shared__ double red[kInfoThreads / 32][kInfoNv];
  const double tot = dgr_block_sum<kInfoThreads>(v, red);
  if (threadIdx.x < kInfoNv) part[(int64_t)blockIdx.x * kInfoNv + threadIdx.x] = tot;
}

// warp k sums partial k over the CTAs (lane-strided, then a fixed butterfly); thread 0 writes
// Lambda = [[tr(Q) I - Q, [S]x], [[S]x^T, n I]] (S = sum q, Q = sum q q^T) and n
__global__ void __launch_bounds__(32 * kInfoNv)
info_final_kernel(const double* __restrict__ part, int n_blocks, double* __restrict__ out) {
  __shared__ double tot[kInfoNv];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double v = 0.0;
  for (int b = lane; b < n_blocks; b += 32) v += part[(int64_t)b * kInfoNv + warp];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  if (lane == 0) tot[warp] = v;
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double n = tot[0], S[3] = {tot[1], tot[2], tot[3]};
  const double Q[3][3] = {{tot[4], tot[5], tot[6]}, {tot[5], tot[7], tot[8]}, {tot[6], tot[8], tot[9]}};
  const double tr = Q[0][0] + Q[1][1] + Q[2][2];
  const double Sx[3][3] = {{0.0, -S[2], S[1]}, {S[2], 0.0, -S[0]}, {-S[1], S[0], 0.0}};
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      double e;
      if (r < 3 && c < 3) e = (r == c ? tr : 0.0) - Q[r][c];
      else if (r < 3) e = Sx[r][c - 3];
      else if (c < 3) e = Sx[c][r - 3];
      else e = r == c ? n : 0.0;
      out[6 * r + c] = e;
    }
  out[36] = n;
}

inline int info_blocks(int64_t n_src) {
  unsigned blocks = dgr_blocks(n_src * 8, kInfoThreads);    // 8 lanes per source point
  return blocks > (unsigned)kInfoMaxBlocks ? kInfoMaxBlocks : (int)blocks;
}

// ---------------------------------------------------------------------------------------
// pose graph
// ---------------------------------------------------------------------------------------
struct PgOpt {
  int N, E, P, npad, ref;
  double mu_scale;        // preference_loop_closure * max_correspondence_distance^2
  double prune;
  int max_iteration, max_iteration_lm;
  double min_rel_inc, min_rel_res_inc, min_right, min_res, upper, lower;
};

struct PgWs {
  // inputs: one host-to-device copy of the region [P0, out)
  double* P0;          // [N][12] initial poses, row-major [R | t]
  double* X;           // [E][12] edge transformations (source into target)
  double* Lam;         // [E][36] information matrices
  double* l0;          // [E] initial line process (the confidence of an uncertain edge, 1 otherwise)
  int32_t* ends;       // [E][2] (source, target)
  int32_t* unc;        // [E] uncertain flags
  int32_t* inc_off;    // [N + 1]
  int32_t* inc;        // [2E] incident edges of each node, ascending
  int32_t* pair_off;   // [P + 1]
  int32_t* pair_e;     // [E] edges of each node pair, ascending
  int32_t* pmap;       // [N][N] pair index of nodes (a, c), a > c; -1 when no edge joins them
  // work
  double* Pc;          // [N][12] current poses
  double* Pn;          // [N][12] trial poses
  double* Xi;          // [E][12] X^-1
  double* r;           // [E][6] residuals at Pc
  double* rn;          // [E][6] residuals at Pn
  double* l;           // [E] line process
  int32_t* act;        // [E] edge in the current pass
  double* A;           // [E][36] l J^T Lambda J
  double* g;           // [E][6] l J^T Lambda r
  double* Hd;          // [N][36] diagonal blocks of H
  double* Hp;          // [P][36] off-diagonal blocks (a, c), a > c
  double* b;           // [npad] right-hand side -J^T Lambda r (entries from 6 N on are never written or read)
  double* y;           // [npad] solve vector; the step delta after the solves
  double* L;           // [npad][npad] H + lambda I, factored in place (lower triangle)
  double* out;         // [16 N + 2 E + kPgStats] result
};

inline int pg_npad(int64_t N) { return (int)(((6 * N + kPgNb - 1) / kPgNb) * kPgNb); }

int64_t pg_layout(int64_t N, int64_t E, int64_t P, void* base, PgWs* w) {
  const int64_t npad = pg_npad(N);
  DgrCarver c(base);
  PgWs r;
  r.P0 = c.take<double>(12 * N);
  r.X = c.take<double>(12 * E);
  r.Lam = c.take<double>(36 * E);
  r.l0 = c.take<double>(E);
  r.ends = c.take<int32_t>(2 * E);
  r.unc = c.take<int32_t>(E);
  r.inc_off = c.take<int32_t>(N + 1);
  r.inc = c.take<int32_t>(2 * E);
  r.pair_off = c.take<int32_t>(P + 1);
  r.pair_e = c.take<int32_t>(E);
  r.pmap = c.take<int32_t>(N * N);
  r.Pc = c.take<double>(12 * N);
  r.Pn = c.take<double>(12 * N);
  r.Xi = c.take<double>(12 * E);
  r.r = c.take<double>(6 * E);
  r.rn = c.take<double>(6 * E);
  r.l = c.take<double>(E);
  r.act = c.take<int32_t>(E);
  r.A = c.take<double>(36 * E);
  r.g = c.take<double>(6 * E);
  r.Hd = c.take<double>(36 * N);
  r.Hp = c.take<double>(36 * P);
  r.b = c.take<double>(npad);
  r.y = c.take<double>(npad);
  r.L = c.take<double>(npad * npad);
  r.out = c.take<double>(16 * N + 2 * E + kPgStats);
  if (w != nullptr) *w = r;
  return c.words;
}

// C = A B for row-major [R | t] poses
__device__ __forceinline__ void pg_mul(const double* A, const double* B, double* C) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c)
      C[4 * r + c] = A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c] + A[4 * r + 2] * B[8 + c] + (c == 3 ? A[4 * r + 3] : 0.0);
}

__device__ __forceinline__ void pg_inv(const double* A, double* B) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) B[4 * r + c] = A[4 * c + r];
    B[4 * r + 3] = -(A[r] * A[3] + A[4 + r] * A[7] + A[8 + r] * A[11]);
  }
}

// open3d's linearised 6-vector (1/2 (A21 - A12), 1/2 (A02 - A20), 1/2 (A10 - A01), A03, A13, A23)
__device__ __forceinline__ void pg_vec6(const double* A, double* v) {
  v[0] = 0.5 * (A[9] - A[6]);
  v[1] = 0.5 * (A[2] - A[8]);
  v[2] = 0.5 * (A[4] - A[1]);
  v[3] = A[3];
  v[4] = A[7];
  v[5] = A[11];
}

// M = X^-1 P_t^-1 and the residual v(M P_s) of edge e
__device__ __forceinline__ void pg_edge(const PgWs& w, const double* __restrict__ P, int e, double* M, double* rv) {
  const int s = w.ends[2 * e], t = w.ends[2 * e + 1];
  double Pt[12], Ti[12], A[12];
  for (int k = 0; k < 12; ++k) Pt[k] = P[12 * t + k];
  pg_inv(Pt, Ti);
  pg_mul(w.Xi + 12 * e, Ti, M);
  pg_mul(M, P + 12 * s, A);
  pg_vec6(A, rv);
}

__device__ __forceinline__ double pg_quad(const double* __restrict__ Lam, const double* rv) {
  double q = 0.0;
  for (int a = 0; a < 6; ++a) {
    double s = 0.0;
    for (int c = 0; c < 6; ++c) s += Lam[6 * a + c] * rv[c];
    q += rv[a] * s;
  }
  return q;
}

// l = (mu / (mu + q))^2; 0 / 0 reads as 1
__device__ __forceinline__ double pg_line(double mu, double q) {
  const double d = mu + q;
  if (d == 0.0) return 1.0;
  const double t = mu / d;
  return t * t;
}

__device__ __forceinline__ double pg_cost(double q, double l, double mu, int uncertain) {
  if (!uncertain) return q;
  const double s = sqrt(l) - 1.0;
  return l * q + mu * s * s;
}

// |x|^2 of open3d's TransformMatrix4dToVector6d (ZYX Euler angles, translation) of one pose
__device__ __forceinline__ double pg_pose_vec_sq(const double* T) {
  const double sy = sqrt(T[0] * T[0] + T[4] * T[4]);
  double a, b, c;
  if (!(sy < 1e-6)) {
    a = atan2(T[9], T[10]);
    b = atan2(-T[8], sy);
    c = atan2(T[4], T[0]);
  } else {
    a = atan2(-T[6], T[5]);
    b = atan2(-T[8], sy);
    c = 0.0;
  }
  return a * a + b * b + c * c + T[3] * T[3] + T[7] * T[7] + T[11] * T[11];
}

struct PgShared {
  double part[kPgWarps][8];
  double tot[8];
  double D[kPgNb][kPgNb + 1];                           // diagonal block of the panel step
  double ys[kPgNb];
  int fail;
};

// fixed-order sums of K per-thread values, broadcast to every thread
template <int K>
__device__ __forceinline__ void pg_sum(PgShared& sh, const double (&v)[K], double (&out)[K]) {
  const double s = dgr_block_sum<kPgThreads>(v, sh.part);
  if (threadIdx.x < K) sh.tot[threadIdx.x] = s;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) out[k] = sh.tot[k];
  __syncthreads();
}

__device__ __forceinline__ double pg_max(PgShared& sh, double v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, d));
  if (lane == 0) sh.part[warp][0] = v;
  __syncthreads();
  double m = sh.part[0][0];
  for (int k = 1; k < kPgWarps; ++k) m = fmax(m, sh.part[k][0]);
  __syncthreads();
  return m;
}

// residuals of the active edges at poses P into rv; -> sum of the cost terms with line process l
__device__ __noinline__ double pg_residuals(PgShared& sh, const PgWs& w, const PgOpt& o, const double* P, double* rv, double mu) {
  double c[1] = {0.0};
  for (int e = threadIdx.x; e < o.E; e += kPgThreads) {
    if (!w.act[e]) continue;
    double M[12], r6[6];
    pg_edge(w, P, e, M, r6);
    for (int k = 0; k < 6; ++k) rv[6 * e + k] = r6[k];
    c[0] += pg_cost(pg_quad(w.Lam + 36 * e, r6), w.l[e], mu, w.unc[e]);
  }
  double t[1];
  pg_sum(sh, c, t);
  return t[0];
}

// line process at the residuals r, then per edge A = l J^T Lambda J, g = l J^T Lambda r, then the blocks of H and b
// (each a sum over edges in edge order); -> max |b|
__device__ __noinline__ double pg_system(PgShared& sh, const PgWs& w, const PgOpt& o, double mu) {
  for (int e = threadIdx.x; e < o.E; e += kPgThreads) {
    if (!w.act[e]) continue;
    const double* Lam = w.Lam + 36 * e;
    double M[12], r6[6];
    pg_edge(w, w.Pc, e, M, r6);
    const double* rv = w.r + 6 * e;
    const double l = w.unc[e] ? pg_line(mu, pg_quad(Lam, rv)) : 1.0;
    w.l[e] = l;
    // J[:, i] = v(M G_i P_s): rotation generators [e_i]x, translation generators e_k in column 3
    const int s = w.ends[2 * e];
    const double* Ps = w.Pc + 12 * s;
    double J[6][6];
    for (int i = 0; i < 3; ++i) {
      double W[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
      const int a = (i + 1) % 3, bb = (i + 2) % 3;
      W[bb][a] = 1.0;
      W[a][bb] = -1.0;
      double MW[3][3];
      for (int p = 0; p < 3; ++p)
        for (int q = 0; q < 3; ++q) MW[p][q] = M[4 * p] * W[0][q] + M[4 * p + 1] * W[1][q] + M[4 * p + 2] * W[2][q];
      double B[12];
      for (int p = 0; p < 3; ++p)
        for (int q = 0; q < 4; ++q) B[4 * p + q] = MW[p][0] * Ps[q] + MW[p][1] * Ps[4 + q] + MW[p][2] * Ps[8 + q];
      double v6[6];
      pg_vec6(B, v6);
      for (int k = 0; k < 6; ++k) J[k][i] = v6[k];
    }
    for (int k = 0; k < 3; ++k) {
      J[0][3 + k] = 0.0; J[1][3 + k] = 0.0; J[2][3 + k] = 0.0;
      for (int p = 0; p < 3; ++p) J[3 + p][3 + k] = M[4 * p + k];
    }
    // row p of J^T Lambda, then row p of A and entry p of g
    for (int p = 0; p < 6; ++p) {
      double JL[6];
      for (int c = 0; c < 6; ++c) {
        double acc = 0.0;
        for (int m = 0; m < 6; ++m) acc += J[m][p] * Lam[6 * m + c];
        JL[c] = acc;
      }
      double gp = 0.0;
      for (int m = 0; m < 6; ++m) gp += JL[m] * rv[m];
      w.g[6 * e + p] = l * gp;
      for (int q = 0; q < 6; ++q) {
        double acc = 0.0;
        for (int m = 0; m < 6; ++m) acc += JL[m] * J[m][q];
        w.A[36 * e + 6 * p + q] = l * acc;
      }
    }
  }
  __syncthreads();
  // diagonal blocks: + A of every incident edge; b: -g at the source, +g at the target
  for (int k = threadIdx.x; k < o.N * 42; k += kPgThreads) {
    const int node = k / 42, c = k % 42;
    double acc = 0.0;
    for (int q = w.inc_off[node]; q < w.inc_off[node + 1]; ++q) {
      const int e = w.inc[q];
      if (!w.act[e]) continue;
      if (c < 36) acc += w.A[36 * e + c];
      else acc += (w.ends[2 * e] == node ? -1.0 : 1.0) * w.g[6 * e + c - 36];
    }
    if (c < 36) w.Hd[36 * node + c] = acc;
    else w.b[6 * node + c - 36] = acc;
  }
  // off-diagonal blocks: - A of every edge joining the pair
  for (int k = threadIdx.x; k < o.P * 36; k += kPgThreads) {
    const int p = k / 36, c = k % 36;
    double acc = 0.0;
    for (int q = w.pair_off[p]; q < w.pair_off[p + 1]; ++q) {
      const int e = w.pair_e[q];
      if (w.act[e]) acc -= w.A[36 * e + c];
    }
    w.Hp[36 * p + c] = acc;
  }
  __syncthreads();
  double m = 0.0;
  for (int i = threadIdx.x; i < 6 * o.N; i += kPgThreads) m = fmax(m, fabs(w.b[i]));
  return pg_max(sh, m);
}

// L = H + lambda I (lower triangle; the padding rows are the identity), factored in place: right-looking, panels of
// kPgNb columns.  -> false on a pivot that is not positive and finite
__device__ __noinline__ bool pg_factor(PgShared& sh, const PgWs& w, const PgOpt& o, double lambda) {
  const int n = o.npad, n6 = 6 * o.N, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* L = w.L;
  for (int64_t q = tid; q < (int64_t)n * n; q += kPgThreads) {
    const int i = (int)(q / n), j = (int)(q % n);
    if (j > i) continue;
    double v;
    if (i >= n6) {
      v = i == j ? 1.0 : 0.0;
    } else {
      const int a = i / 6, c = j / 6;
      if (a == c) {
        v = w.Hd[36 * a + 6 * (i % 6) + j % 6] + (i == j ? lambda : 0.0);
      } else {
        const int p = w.pmap[a * o.N + c];
        v = p < 0 ? 0.0 : w.Hp[36 * p + 6 * (i % 6) + j % 6];
      }
    }
    L[q] = v;
  }
  if (tid == 0) sh.fail = 0;
  __syncthreads();
  for (int k0 = 0; k0 < n; k0 += kPgNb) {
    const int k1 = k0 + kPgNb;
    // 1. the diagonal block, unblocked, on warp 0
    if (warp == 0) {
      for (int r = 0; r < kPgNb; ++r) sh.D[r][lane] = lane <= r ? L[(int64_t)(k0 + r) * n + k0 + lane] : 0.0;
      __syncwarp();
      for (int j = 0; j < kPgNb; ++j) {
        if (lane == 0) {
          const double d = sh.D[j][j];
          const bool ok = d > 0.0 && isfinite(d);
          if (!ok) sh.fail = 1;
          sh.D[j][j] = ok ? sqrt(d) : 1.0;
        }
        __syncwarp();
        if (lane > j) sh.D[lane][j] /= sh.D[j][j];
        __syncwarp();
        if (lane > j) {
          const double lij = sh.D[lane][j];
          for (int c = j + 1; c <= lane; ++c) sh.D[lane][c] -= lij * sh.D[c][j];
        }
        __syncwarp();
      }
      for (int r = 0; r < kPgNb; ++r)
        if (lane <= r) L[(int64_t)(k0 + r) * n + k0 + lane] = sh.D[r][lane];
    }
    __syncthreads();
    // 2. the panel below it: row i solves x L_kk^T = L[i, k0:k1)
    for (int i = k1 + tid; i < n; i += kPgThreads) {
      double x[kPgNb];
      double* row = L + (int64_t)i * n + k0;
#pragma unroll
      for (int j = 0; j < kPgNb; ++j) x[j] = row[j];
#pragma unroll
      for (int j = 0; j < kPgNb; ++j) {
        double s = x[j];
#pragma unroll
        for (int m = 0; m < j; ++m) s -= x[m] * sh.D[j][m];
        x[j] = s / sh.D[j][j];
      }
#pragma unroll
      for (int j = 0; j < kPgNb; ++j) row[j] = x[j];
    }
    __syncthreads();
    // 3. the trailing lower triangle: a warp per 32 x 32 tile, a lane per column
    const int nt = (n - k1) / kPgNb;
    for (int t = warp; t < nt * (nt + 1) / 2; t += kPgWarps) {
      int ti = 0;
      while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
      const int tj = t - ti * (ti + 1) / 2;
      const int j = k1 + kPgNb * tj + lane;
      double lj[kPgNb];
      const double* rj = L + (int64_t)j * n + k0;
#pragma unroll
      for (int m = 0; m < kPgNb; ++m) lj[m] = rj[m];
      for (int rr = 0; rr < kPgNb; ++rr) {
        const int i = k1 + kPgNb * ti + rr;
        if (i < j) continue;
        const double* ri = L + (int64_t)i * n + k0;
        double s = 0.0;
#pragma unroll
        for (int m = 0; m < kPgNb; ++m) s += ri[m] * lj[m];
        L[(int64_t)i * n + j] -= s;
      }
    }
    __syncthreads();
  }
  return sh.fail == 0;
}

// warp-wide fixed-order sum
__device__ __forceinline__ double pg_warp_sum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// y = b, then L y' = y and L^T delta = y' in place (blocked by panels)
__device__ __noinline__ void pg_solve(PgShared& sh, const PgWs& w, const PgOpt& o) {
  const int n = o.npad, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* L = w.L;
  double* y = w.y;
  // the padding rows solve to exactly 0: the back solve multiplies them by the zero entries L[pad][real], and a stale
  // workspace value there (NaN bit patterns included) would otherwise reach the real unknowns
  for (int i = tid; i < n; i += kPgThreads) y[i] = i < 6 * o.N ? w.b[i] : 0.0;
  __syncthreads();
  for (int k0 = 0; k0 < n; k0 += kPgNb) {
    if (warp == 0) {
      double mine = y[k0 + lane];
      for (int j = 0; j < kPgNb; ++j) {
        const double yj = __shfl_sync(0xffffffffu, mine, j);
        const double lj = L[(int64_t)(k0 + j) * n + k0 + j];
        const double s = pg_warp_sum(lane < j ? L[(int64_t)(k0 + j) * n + k0 + lane] * mine : 0.0);
        if (lane == j) mine = (yj - s) / lj;
      }
      y[k0 + lane] = mine;
      sh.ys[lane] = mine;
    }
    __syncthreads();
    for (int i = k0 + kPgNb + tid; i < n; i += kPgThreads) {
      const double* ri = L + (int64_t)i * n + k0;
      double s = 0.0;
      for (int m = 0; m < kPgNb; ++m) s += ri[m] * sh.ys[m];
      y[i] -= s;
    }
    __syncthreads();
  }
  for (int k0 = n - kPgNb; k0 >= 0; k0 -= kPgNb) {
    if (warp == 0) {
      double mine = y[k0 + lane];
      for (int j = kPgNb - 1; j >= 0; --j) {
        const double yj = __shfl_sync(0xffffffffu, mine, j);
        const double lj = L[(int64_t)(k0 + j) * n + k0 + j];
        const double s = pg_warp_sum(lane > j ? L[(int64_t)(k0 + lane) * n + k0 + j] * mine : 0.0);
        if (lane == j) mine = (yj - s) / lj;
      }
      y[k0 + lane] = mine;
      sh.ys[lane] = mine;
    }
    __syncthreads();
    for (int c = tid; c < k0; c += kPgThreads) {
      double s = 0.0;
      for (int m = 0; m < kPgNb; ++m) s += L[(int64_t)(k0 + m) * n + c] * sh.ys[m];
      y[c] -= s;
    }
    __syncthreads();
  }
}

struct PgPass {
  int iterations, failed, factorisations;
  double mu, cost0, cost;
};

// one GlobalOptimizationLevenbergMarquardt run over the active edges, from the poses in w.Pc
__device__ __noinline__ PgPass pg_pass(PgShared& sh, const PgWs& w, const PgOpt& o) {
  const int tid = threadIdx.x, n6 = 6 * o.N;
  PgPass res = {0, 0, 0, 0.0, 0.0, 0.0};
  {
    double v[2] = {0.0, 0.0}, t[2];
    for (int e = tid; e < o.E; e += kPgThreads)
      if (w.act[e]) { v[0] += w.Lam[36 * e + 35]; v[1] += 1.0; }
    pg_sum(sh, v, t);
    res.mu = o.mu_scale * (t[1] > 0.0 ? t[0] / t[1] : 0.0);
  }
  const double mu = res.mu;
  double E = pg_residuals(sh, w, o, w.Pc, w.r, mu);    // with the line process the pass starts from
  res.cost0 = E;
  double maxb = pg_system(sh, w, o, mu);
  double maxdiag = 0.0;
  for (int i = tid; i < n6; i += kPgThreads) maxdiag = fmax(maxdiag, w.Hd[36 * (i / 6) + 7 * (i % 6)]);
  maxdiag = pg_max(sh, maxdiag);
  double lambda = 1e-5 * maxdiag, ni = 2.0;
  bool stop = maxb < o.min_right;
  for (int iter = 0; iter < o.max_iteration && !stop; ++iter) {
    res.iterations = iter + 1;
    int lm = 0;
    double rho = 0.0;
    do {
      ++res.factorisations;
      if (!pg_factor(sh, w, o, lambda)) {
        res.failed = 1;
        stop = true;
        break;
      }
      pg_solve(sh, w, o);
      double v[3] = {0.0, 0.0, 0.0}, t[3];
      for (int i = tid; i < n6; i += kPgThreads) {
        const double d = w.y[i];
        v[0] += d * d;
        v[2] += d * (lambda * d + w.b[i]);
      }
      for (int k = tid; k < o.N; k += kPgThreads) v[1] += pg_pose_vec_sq(w.Pc + 12 * k);
      pg_sum(sh, v, t);
      if (sqrt(t[0]) < o.min_rel_inc * (sqrt(t[1]) + o.min_rel_inc)) stop = true;
      if (!stop) {
        for (int k = tid; k < o.N; k += kPgThreads) zyx_update_left(w.y + 6 * k, w.Pc + 12 * k, w.Pn + 12 * k);
        __syncthreads();
        const double En = pg_residuals(sh, w, o, w.Pn, w.rn, mu);
        rho = (E - En) / (t[2] + 1e-3);
        if (rho > 0.0) {
          if (fabs(E - En) < o.min_rel_res_inc * E) stop = true;
          const double q = 2.0 * rho - 1.0;
          const double alpha = fmin(1.0 - q * q * q, o.upper);
          lambda *= fmax(o.lower, alpha);
          ni = 2.0;
          E = En;
          for (int k = tid; k < 12 * o.N; k += kPgThreads) w.Pc[k] = w.Pn[k];
          for (int k = tid; k < 6 * o.E; k += kPgThreads) w.r[k] = w.rn[k];
          __syncthreads();
          maxb = pg_system(sh, w, o, mu);
          if (maxb < o.min_right) stop = true;
          if (stop) break;
        } else {
          lambda *= ni;
          ni *= 2.0;
        }
      }
      ++lm;
      if (lm >= o.max_iteration_lm) stop = true;
    } while (!(rho > 0.0 || stop));
    if (E < o.min_res) stop = true;
  }
  res.cost = E;
  return res;
}

__global__ void __launch_bounds__(kPgThreads, 1)
pose_graph_kernel(PgWs w, PgOpt o) {
  __shared__ PgShared sh;
  const int tid = threadIdx.x;
  for (int e = tid; e < o.E; e += kPgThreads) {
    pg_inv(w.X + 12 * e, w.Xi + 12 * e);
    w.l[e] = w.l0[e];
    w.act[e] = 1;
  }
  for (int k = tid; k < 12 * o.N; k += kPgThreads) w.Pc[k] = w.P0[k];
  __syncthreads();
  const PgPass p1 = pg_pass(sh, w, o);
  int pruned = 0;
  PgPass p2 = {0, 0, 0, 0.0, p1.cost, p1.cost};
  if (!p1.failed) {
    double v[1] = {0.0}, t[1];
    for (int e = tid; e < o.E; e += kPgThreads)
      if (w.unc[e] && !(w.l[e] >= o.prune)) { w.act[e] = 0; v[0] += 1.0; }
    pg_sum(sh, v, t);                                   // also the barrier before the second pass
    pruned = (int)t[0];
    p2 = pg_pass(sh, w, o);
  }
  double* out = w.out;
  // compensation: P_k <- P0_ref P_ref^-1 P_k, the reference node keeping its input pose bit for bit
  double C[12];
  if (o.ref >= 0) {
    double Ri[12];
    pg_inv(w.Pc + 12 * o.ref, Ri);
    pg_mul(w.P0 + 12 * o.ref, Ri, C);
  }
  for (int k = tid; k < o.N; k += kPgThreads) {
    double T[12];
    if (o.ref < 0) for (int q = 0; q < 12; ++q) T[q] = w.Pc[12 * k + q];
    else if (k == o.ref) for (int q = 0; q < 12; ++q) T[q] = w.P0[12 * k + q];
    else pg_mul(C, w.Pc + 12 * k, T);
    for (int q = 0; q < 12; ++q) out[16 * k + q] = T[q];
    out[16 * k + 12] = 0.0; out[16 * k + 13] = 0.0; out[16 * k + 14] = 0.0; out[16 * k + 15] = 1.0;
  }
  for (int e = tid; e < o.E; e += kPgThreads) {
    out[16 * o.N + e] = w.act[e];
    out[16 * o.N + o.E + e] = w.l[e];
  }
  if (tid == 0) {
    double* st = out + 16 * o.N + 2 * o.E;
    for (int k = 0; k < kPgStats; ++k) st[k] = 0.0;
    st[0] = p1.iterations;
    st[1] = p2.iterations;
    st[2] = p2.cost;
    st[3] = pruned;
    st[4] = p1.failed || p2.failed ? 1.0 : 0.0;
    st[5] = p1.mu;
    st[6] = p2.mu;
    st[7] = p1.cost0;
    st[8] = p1.cost;
    st[9] = p1.factorisations + p2.factorisations;
  }
}

bool finite_all(const double* p, int64_t n) {
  for (int64_t k = 0; k < n; ++k)
    if (!std::isfinite(p[k])) return false;
  return true;
}

// node pairs (a, c), a > c, joined by an edge, in ascending (a, c) order
int64_t count_pairs(const int32_t* ends, int64_t E, int64_t N, std::vector<int32_t>* pmap) {
  std::vector<int32_t> m((size_t)(N * N), -1);
  for (int64_t e = 0; e < E; ++e) {
    const int a = std::max(ends[2 * e], ends[2 * e + 1]), c = std::min(ends[2 * e], ends[2 * e + 1]);
    m[(size_t)(a * N + c)] = 0;
  }
  int64_t P = 0;
  for (int64_t q = 0; q < N * N; ++q)
    if (m[(size_t)q] == 0) m[(size_t)q] = (int32_t)P++;
  if (pmap != nullptr) *pmap = std::move(m);
  return P;
}

}  // namespace

// the information matrix of kInfoNv (= 10) sums per CTA in part[n_blocks][10], written to out[37]; odometry.cu's
// information pass shares it
void dgr_info_final(const double* part, int n_blocks, double* out, cudaStream_t st) {
  info_final_kernel<<<1, 32 * kInfoNv, 0, st>>>(part, n_blocks, out);
}

extern "C" {

int32_t dgr_information_matrix_ws_elems(int64_t n_src, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0, "bad arguments");
  *n_elems = (int64_t)info_blocks(n_src) * kInfoNv;
  return DGR_OK;
}

int32_t dgr_information_matrix(const float* src, int64_t n_src, const float* tgt, const dgr_keyspec_t* spec,
                               const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch, double cell,
                               double max_dist, const double* T, double* ws, double* out, void* stream) {
  DGR_ARG_CHECK(T != nullptr && ws != nullptr && out != nullptr && spec != nullptr && keys != nullptr &&
                vals != nullptr, "null pointer");
  DGR_ARG_CHECK(n_src >= 0 && n_src < (1ll << 31), "point count out of range");
  DGR_ARG_CHECK(n_src == 0 || (src != nullptr && tgt != nullptr), "null pointer");
  DGR_TRY(dgr_check_hash_search(cap, cell, max_dist, 4));
  DGR_ARG_CHECK(finite_all(T, 16), "transformation must be finite");
  cudaStream_t st = (cudaStream_t)stream;
  Pose12 P;
  for (int k = 0; k < 12; ++k) P.m[k] = T[k];
  const int blocks = info_blocks(n_src);
  info_match_kernel<<<blocks, kInfoThreads, 0, st>>>(src, n_src, tgt, spec, keys, vals, (uint64_t)cap - 1, batch, cell,
                                                     (int)ceil(max_dist / cell), max_dist, P, ws);
  dgr_info_final(ws, blocks, out, st);
  dgr_note_launches(2);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_pose_graph_ws_elems(int64_t n_nodes, int64_t n_edges, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr, "null pointer");
  DGR_ARG_CHECK(n_nodes >= 1 && n_nodes <= DGR_POSE_GRAPH_MAX_NODES, "node count out of range");
  DGR_ARG_CHECK(n_edges >= 0 && n_edges <= DGR_POSE_GRAPH_MAX_EDGES, "edge count out of range");
  *n_elems = pg_layout(n_nodes, n_edges, n_edges, nullptr, nullptr);   // at most one node pair per edge
  return DGR_OK;
}

int32_t dgr_pose_graph_optimize(const double* poses, int64_t n_nodes, const int32_t* ends, const double* T,
                                const double* info, const int32_t* uncertain, const double* confidence,
                                int64_t n_edges, double max_correspondence_distance, double edge_prune_threshold,
                                double preference_loop_closure, int32_t reference_node, int32_t max_iteration,
                                double min_relative_increment, double min_relative_residual_increment,
                                double min_right_term, double min_residual, int32_t max_iteration_lm,
                                double upper_scale_factor, double lower_scale_factor, uint64_t* ws, double* poses_out,
                                int32_t* kept_out, double* l_out, double* stats, void* stream) {
  const int64_t N = n_nodes, E = n_edges;
  DGR_ARG_CHECK(N >= 1 && N <= DGR_POSE_GRAPH_MAX_NODES, "node count out of range");
  DGR_ARG_CHECK(E >= 0 && E <= DGR_POSE_GRAPH_MAX_EDGES, "edge count out of range");
  DGR_ARG_CHECK(poses != nullptr && ws != nullptr && poses_out != nullptr && stats != nullptr, "null pointer");
  DGR_ARG_CHECK(E == 0 || (ends != nullptr && T != nullptr && info != nullptr && uncertain != nullptr &&
                           confidence != nullptr && kept_out != nullptr && l_out != nullptr), "null pointer");
  for (int64_t e = 0; e < E; ++e) {
    DGR_ARG_CHECK(ends[2 * e] >= 0 && ends[2 * e] < N && ends[2 * e + 1] >= 0 && ends[2 * e + 1] < N,
                  "edge node id out of range");
    DGR_ARG_CHECK(ends[2 * e] != ends[2 * e + 1], "edge joins a node to itself");
  }
  DGR_ARG_CHECK(finite_all(poses, 16 * N), "node poses must be finite");
  DGR_ARG_CHECK(E == 0 || finite_all(T, 16 * E), "edge transformations must be finite");
  DGR_ARG_CHECK(E == 0 || finite_all(info, 36 * E), "information matrices must be finite");
  DGR_ARG_CHECK(E == 0 || finite_all(confidence, E), "confidences must be finite");
  DGR_ARG_CHECK(reference_node >= -1 && reference_node < N, "reference_node must lie in [-1, n_nodes)");
  DGR_ARG_CHECK(max_correspondence_distance > 0.0 && std::isfinite(max_correspondence_distance),
                "max_correspondence_distance must be positive");
  DGR_ARG_CHECK(std::isfinite(edge_prune_threshold), "edge_prune_threshold must be finite");
  DGR_ARG_CHECK(preference_loop_closure >= 0.0 && std::isfinite(preference_loop_closure),
                "preference_loop_closure must be >= 0");
  DGR_ARG_CHECK(max_iteration >= 0 && max_iteration_lm >= 1, "iteration limits out of range");
  DGR_ARG_CHECK(std::isfinite(min_relative_increment) && std::isfinite(min_relative_residual_increment) &&
                std::isfinite(min_right_term) && std::isfinite(min_residual) && std::isfinite(upper_scale_factor) &&
                std::isfinite(lower_scale_factor), "convergence criteria must be finite");
  cudaStream_t st = (cudaStream_t)stream;
  // the incidence lists, on the host
  std::vector<int32_t> pmap;
  const int64_t P = count_pairs(ends, E, N, &pmap);
  PgWs w, h;
  pg_layout(N, E, P, ws, &w);
  const int64_t n_in = reinterpret_cast<uint64_t*>(w.Pc) - ws;     // the input regions come first
  std::vector<uint64_t> host((size_t)n_in, 0);
  pg_layout(N, E, P, host.data(), &h);                 // only its input regions are written
  for (int64_t k = 0; k < N; ++k)
    for (int q = 0; q < 12; ++q) h.P0[12 * k + q] = poses[16 * k + q];
  for (int64_t e = 0; e < E; ++e) {
    for (int q = 0; q < 12; ++q) h.X[12 * e + q] = T[16 * e + q];
    for (int q = 0; q < 36; ++q) h.Lam[36 * e + q] = info[36 * e + q];
    h.unc[e] = uncertain[e] != 0;
    h.l0[e] = h.unc[e] ? confidence[e] : 1.0;
    h.ends[2 * e] = ends[2 * e];
    h.ends[2 * e + 1] = ends[2 * e + 1];
  }
  std::vector<int32_t> deg((size_t)N, 0), pcnt((size_t)P, 0);
  for (int64_t e = 0; e < E; ++e) {
    ++deg[ends[2 * e]];
    ++deg[ends[2 * e + 1]];
    const int a = std::max(ends[2 * e], ends[2 * e + 1]), c = std::min(ends[2 * e], ends[2 * e + 1]);
    ++pcnt[pmap[(size_t)(a * N + c)]];
  }
  h.inc_off[0] = 0;
  for (int64_t k = 0; k < N; ++k) h.inc_off[k + 1] = h.inc_off[k] + deg[k];
  h.pair_off[0] = 0;
  for (int64_t p = 0; p < P; ++p) h.pair_off[p + 1] = h.pair_off[p] + pcnt[p];
  std::vector<int32_t> fill_n((size_t)N, 0), fill_p((size_t)P, 0);
  for (int64_t e = 0; e < E; ++e) {                    // edges in ascending order into every list
    for (int side = 0; side < 2; ++side) {
      const int node = ends[2 * e + side];
      h.inc[h.inc_off[node] + fill_n[node]++] = (int32_t)e;
    }
    const int a = std::max(ends[2 * e], ends[2 * e + 1]), c = std::min(ends[2 * e], ends[2 * e + 1]);
    const int p = pmap[(size_t)(a * N + c)];
    h.pair_e[h.pair_off[p] + fill_p[p]++] = (int32_t)e;
  }
  for (int64_t q = 0; q < N * N; ++q) h.pmap[q] = pmap[(size_t)q];
  DGR_CUDA_CHECK(cudaMemcpyAsync(ws, host.data(), n_in * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  PgOpt o;
  o.N = (int)N; o.E = (int)E; o.P = (int)P; o.npad = pg_npad(N); o.ref = reference_node;
  o.mu_scale = preference_loop_closure * max_correspondence_distance * max_correspondence_distance;
  o.prune = edge_prune_threshold;
  o.max_iteration = max_iteration; o.max_iteration_lm = max_iteration_lm;
  o.min_rel_inc = min_relative_increment; o.min_rel_res_inc = min_relative_residual_increment;
  o.min_right = min_right_term; o.min_res = min_residual;
  o.upper = upper_scale_factor; o.lower = lower_scale_factor;
  pose_graph_kernel<<<1, kPgThreads, 0, st>>>(w, o);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  const int64_t n_out = 16 * N + 2 * E + kPgStats;
  std::vector<double> res((size_t)n_out);
  DGR_CUDA_CHECK(cudaMemcpyAsync(res.data(), w.out, n_out * sizeof(double), cudaMemcpyDeviceToHost, st));
  DGR_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int64_t q = 0; q < 16 * N; ++q) poses_out[q] = res[(size_t)q];
  for (int64_t e = 0; e < E; ++e) {
    kept_out[e] = res[(size_t)(16 * N + e)] != 0.0;
    l_out[e] = res[(size_t)(16 * N + E + e)];
  }
  for (int k = 0; k < kPgStats; ++k) stats[k] = res[(size_t)(16 * N + 2 * E + k)];
  return DGR_OK;
}

}  // extern "C"
