// Normal estimation, covariances, colour gradients and ICP: open3d 0.10's EstimateNormals(KDTreeSearchParamHybrid(
// radius, max_nn)), EstimatePerPointCovariances, InitializePointCloudForColoredICP and RegistrationICP with
// TransformationEstimationPointToPoint / PointToPlane / ForColoredICP / ForGeneralizedICP and the robust kernels of
// open3d >= 0.12, restated in oracle/normals.py, oracle/icp.py, oracle/icp_plane.py, oracle/colored_icp.py and
// oracle/gicp.py (which pin every boundary convention).  All search one cloud's voxel hash (a
// dgr_unique_first table with at most one point per cell): the (2 reach + 1)^3 cells around a point,
// reach = ceil(radius / cell) <= 4, 8 lanes per point as in dgr_voxel_nearest8.  No atomics: every sum has a fixed
// order, so a call gives the same bits on every run.
//   nbr_probe_kernel<S>      8 lanes per point, one probe pass: count and the 9 fp64 sums S adds over the rows with
//                            |p_j - p_i|^2 < radius^2 (the offsets' cumulants for normals and covariances, the
//                            gradient rows for colour gradients); a point with <= max_nn of them gets its result
//   nbr_select_kernel<S>     a warp per point with more than max_nn: the in-radius keys again (dgr_gather_in_radius);
//                            the sums of the max_nn ranked first
//   icp_match_kernel<E>      nearest target row within max_dist (dgr_voxel_nearest8); the estimator's sums, the
//                            count and sum d^2 as per-block partials
//   icp_update_kernel<E>     the partials reduced in block order, open3d's stopping rule, the estimator's step
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kabsch.cuh"

namespace {

constexpr int kNormThreads = 256;
constexpr int kSelWarps = 4;                            // nbr_select_kernel: warps (points) per block
constexpr int kMaxReach = 4;                            // normals, colour gradients and ICP
constexpr int kMaxNN = 64;
constexpr int kIcpThreads = 256;
constexpr int kIcpMaxBlocks = 2368;
constexpr int kIcpStride = 32;                          // doubles per block partial
constexpr int kIcpState = 32;                           // doubles of IcpState (static_assert below)

// m[0..3) += e, m[3..9) += e e^T (xx, xy, xz, yy, yz, zz)
__device__ __forceinline__ void add_cumulants(double m[9], const double e[3]) {
  m[0] += e[0]; m[1] += e[1]; m[2] += e[2];
  m[3] += e[0] * e[0]; m[4] += e[0] * e[1]; m[5] += e[0] * e[2];
  m[6] += e[1] * e[1]; m[7] += e[1] * e[2]; m[8] += e[2] * e[2];
}

// open3d's ComputeNormal on the cumulant sums of n neighbours: C = E[e e^T] - mu mu^T, the eigenvector of the
// smallest eigenvalue (one-sided Jacobi, kabsch.cuh; the first on a tie); (0, 0, 1) for n < 3 or C == 0.
// Sign: the largest-magnitude component made positive (the first on a tie) - a fixed rule, not open3d's - then,
// with previous normals, flipped when it points against the previous one (open3d's rule).
__device__ void store_normal(const double m[9], int n, const float* __restrict__ prev, int64_t i,
                             float* __restrict__ normals) {
  double nv[3] = {0.0, 0.0, 1.0};
  if (n >= 3) {
    const double inv = 1.0 / (double)n;
    const double mu[3] = {m[0] * inv, m[1] * inv, m[2] * inv};
    const double cxx = m[3] * inv - mu[0] * mu[0], cxy = m[4] * inv - mu[0] * mu[1], cxz = m[5] * inv - mu[0] * mu[2];
    const double cyy = m[6] * inv - mu[1] * mu[1], cyz = m[7] * inv - mu[1] * mu[2], czz = m[8] * inv - mu[2] * mu[2];
    if (cxx != 0.0 || cxy != 0.0 || cxz != 0.0 || cyy != 0.0 || cyz != 0.0 || czz != 0.0) {
      const double C[3][3] = {{cxx, cxy, cxz}, {cxy, cyy, cyz}, {cxz, cyz, czz}};
      double A[3][3], V[3][3], sig[3];
      jacobi_svd3(C, A, V, sig);
      int k = 0;
      if (sig[1] < sig[k]) k = 1;
      if (sig[2] < sig[k]) k = 2;
      for (int a = 0; a < 3; ++a) nv[a] = V[a][k];
      int big = 0;
      if (fabs(nv[1]) > fabs(nv[big])) big = 1;
      if (fabs(nv[2]) > fabs(nv[big])) big = 2;
      if (nv[big] < 0.0)
        for (int a = 0; a < 3; ++a) nv[a] = -nv[a];
    }
  }
  if (prev != nullptr) {
    const double d = nv[0] * (double)prev[3 * i] + nv[1] * (double)prev[3 * i + 1] + nv[2] * (double)prev[3 * i + 2];
    if (d < 0.0)
      for (int a = 0; a < 3; ++a) nv[a] = -nv[a];
  }
  for (int a = 0; a < 3; ++a) normals[3 * i + a] = (float)nv[a];
}

// The per-point sums of a neighbourhood pass: 9 fp64 sums over the kept rows j of point i (offset e = p_j - p_i),
// then one result per point.  point(i) loads what add() needs of point i; store() gets the sums and the kept count.
//   NormalSums    the cumulants of e (add_cumulants); store_normal
//   GradientSums  open3d's colour-gradient rows u = e - (e.n_i) n_i, b = I_j - I_i: sum u u^T (xx, xy, xz, yy, yz,
//                 zz) and sum u b; the point's own row adds exact zeros.  store_gradient
struct NormalSums {
  const float* prev;
  float* normals;
  struct Point {};
  __device__ __forceinline__ Point point(int64_t) const { return {}; }
  __device__ __forceinline__ void add(const Point&, double m[9], const double e[3], int32_t) const {
    add_cumulants(m, e);
  }
  __device__ __forceinline__ void store(const double m[9], int n, int64_t i) const {
    store_normal(m, n, prev, i, normals);
  }
};

// open3d's EstimatePerPointCovariances: C = E[e e^T] - mu mu^T over the n kept offsets (NormalSums' cumulants), the
// identity for n < 3; cov[i] = (xx, xy, xz, yy, yz, zz) in fp64
struct CovarianceSums {
  double* cov;
  struct Point {};
  __device__ __forceinline__ Point point(int64_t) const { return {}; }
  __device__ __forceinline__ void add(const Point&, double m[9], const double e[3], int32_t) const {
    add_cumulants(m, e);
  }
  __device__ __forceinline__ void store(const double m[9], int n, int64_t i) const {
    double c[6] = {1.0, 0.0, 0.0, 1.0, 0.0, 1.0};
    if (n >= 3) {
      const double inv = 1.0 / (double)n;
      const double mu[3] = {m[0] * inv, m[1] * inv, m[2] * inv};
      c[0] = m[3] * inv - mu[0] * mu[0]; c[1] = m[4] * inv - mu[0] * mu[1]; c[2] = m[5] * inv - mu[0] * mu[2];
      c[3] = m[6] * inv - mu[1] * mu[1]; c[4] = m[7] * inv - mu[1] * mu[2]; c[5] = m[8] * inv - mu[2] * mu[2];
    }
    for (int a = 0; a < 6; ++a) cov[6 * i + a] = c[a];
  }
};

// InitializePointCloudForGeneralizedICP: C = R diag(eps, 1, 1) R^T with R = GetRotationFromE1ToX(n), evaluated
// literally in fp64: v = e1 x n, c = e1.n, R = I + [v]x + [v]x^2 / (1 + c), or diag(-1, -1, 1) when c < -0.99
__global__ void cov_from_normals_kernel(const float* __restrict__ normals, int64_t n, double eps,
                                        double* __restrict__ cov) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = normals[3 * i], y = normals[3 * i + 1], z = normals[3 * i + 2];
  double R[3][3] = {{-1.0, 0.0, 0.0}, {0.0, -1.0, 0.0}, {0.0, 0.0, 1.0}};
  if (!(x < -0.99)) {
    const double v[3] = {0.0, -z, y};
    const double S[3][3] = {{0.0, -v[2], v[1]}, {v[2], 0.0, -v[0]}, {-v[1], v[0], 0.0}};
    const double f = 1.0 / (1.0 + x);
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) {
        const double s2 = S[a][0] * S[0][b] + S[a][1] * S[1][b] + S[a][2] * S[2][b];
        R[a][b] = (a == b ? 1.0 : 0.0) + S[a][b] + s2 * f;
      }
  }
  const double d[3] = {eps, 1.0, 1.0};
  double c[6];
  int k = 0;
  for (int a = 0; a < 3; ++a)
    for (int b = a; b < 3; ++b) c[k++] = R[a][0] * d[0] * R[b][0] + R[a][1] * d[1] * R[b][1] + R[a][2] * d[2] * R[b][2];
  for (int q = 0; q < 6; ++q) cov[6 * i + q] = c[q];
}

// open3d's InitializePointCloudForColoredICP at point i from the sums of nn neighbours (i included): g = 0 for
// nn < 4, else the solution of (sum u u^T + (nn - 1)^2 n n^T) g = sum u b by a 3x3 Cholesky in fp64 (g = 0 on a
// non-positive pivot, open3d's result when its solve fails), rounded to float once
__device__ void store_gradient(const double m[9], int nn, const double nv[3], int64_t i, float* __restrict__ grad) {
  double g[3] = {0.0, 0.0, 0.0};
  if (nn >= 4) {
    const double k = (double)(nn - 1) * (double)(nn - 1);
    const double a00 = m[0] + k * nv[0] * nv[0], a01 = m[1] + k * nv[0] * nv[1], a02 = m[2] + k * nv[0] * nv[2];
    const double a11 = m[3] + k * nv[1] * nv[1], a12 = m[4] + k * nv[1] * nv[2], a22 = m[5] + k * nv[2] * nv[2];
    if (a00 > 0.0) {
      const double l00 = sqrt(a00), l10 = a01 / l00, l20 = a02 / l00;
      const double d1 = a11 - l10 * l10;
      if (d1 > 0.0) {
        const double l11 = sqrt(d1), l21 = (a12 - l20 * l10) / l11;
        const double d2 = a22 - l20 * l20 - l21 * l21;
        if (d2 > 0.0) {
          const double l22 = sqrt(d2);
          const double y0 = m[6] / l00, y1 = (m[7] - l10 * y0) / l11, y2 = (m[8] - l20 * y0 - l21 * y1) / l22;
          g[2] = y2 / l22;
          g[1] = (y1 - l21 * g[2]) / l11;
          g[0] = (y0 - l10 * g[1] - l20 * g[2]) / l00;
        }
      }
    }
  }
  for (int a = 0; a < 3; ++a) grad[3 * i + a] = (float)g[a];
}

struct GradientSums {
  const float* nrm;
  const float* intensity;
  float* grad;
  struct Point { double n[3], I; };
  __device__ __forceinline__ Point point(int64_t i) const {
    return {{(double)nrm[3 * i], (double)nrm[3 * i + 1], (double)nrm[3 * i + 2]}, (double)intensity[i]};
  }
  __device__ __forceinline__ void add(const Point& q, double m[9], const double e[3], int32_t j) const {
    const double en = e[0] * q.n[0] + e[1] * q.n[1] + e[2] * q.n[2];
    const double u[3] = {e[0] - en * q.n[0], e[1] - en * q.n[1], e[2] - en * q.n[2]};
    const double b = (double)__ldg(intensity + j) - q.I;
    m[0] += u[0] * u[0]; m[1] += u[0] * u[1]; m[2] += u[0] * u[2];
    m[3] += u[1] * u[1]; m[4] += u[1] * u[2]; m[5] += u[2] * u[2];
    m[6] += u[0] * b; m[7] += u[1] * b; m[8] += u[2] * b;
  }
  __device__ __forceinline__ void store(const double m[9], int n, int64_t i) const {
    store_gradient(m, n, point(i).n, i, grad);
  }
};

template <class S>
__global__ void __launch_bounds__(kNormThreads)
nbr_probe_kernel(const float* __restrict__ xyz, int64_t n, const dgr_keyspec_t* __restrict__ spec_p,
                 const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int32_t batch,
                 double cell, int reach, double r2, int max_nn, const S sums, int32_t* __restrict__ counts) {
  const dgr_keyspec_t s = *spec_p;
  const int64_t i0 = ((int64_t)blockIdx.x * kNormThreads + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const bool have = i0 < n;                             // whole warps stay for the shuffles
  const int64_t i = have ? i0 : 0;
  const double p[3] = {(double)xyz[3 * i], (double)xyz[3 * i + 1], (double)xyz[3 * i + 2]};
  const typename S::Point q = sums.point(i);
  const int side = 2 * reach + 1, n_cells = side * side * side;
  int c3[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c3[a] = (int)floor(p[a] / cell);
  int cnt = 0;
  double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int c = sub; c < n_cells && have; c += 8) {
    const int32_t j = dgr_probe_cell(c, side, reach, c3, batch, s, keys, vals, mask);
    if (j < 0) continue;
    double e[3];
    if (dgr_offset_d2(xyz, j, p, e) < r2) {
      ++cnt;
      sums.add(q, m, e, j);
    }
  }
#pragma unroll
  for (int d = 1; d < 8; d <<= 1) {                     // fixed butterfly within the group of 8
    cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] += __shfl_xor_sync(0xffffffffu, m[k], d);
  }
  if (!have || sub != 0) return;
  counts[i] = cnt;
  if (cnt <= max_nn) sums.store(m, cnt, i);
}

template <class S>
__global__ void __launch_bounds__(kSelWarps * 32)
nbr_select_kernel(const float* __restrict__ xyz, int64_t n, const dgr_keyspec_t* __restrict__ spec_p,
                  const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int32_t batch,
                  double cell, int reach, double r2, double gap_limit, int slots, int max_nn, const S sums,
                  const int32_t* __restrict__ counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kSelWarps + warp;
  if (i >= n || counts[i] <= max_nn) return;            // uniform per warp
  double* kd = reinterpret_cast<double*>(smem_raw) + (size_t)warp * slots;
  int32_t* kj = reinterpret_cast<int32_t*>(reinterpret_cast<double*>(smem_raw) + (size_t)kSelWarps * slots) +
                (size_t)warp * slots;
  const dgr_keyspec_t s = *spec_p;
  const double p[3] = {(double)xyz[3 * i], (double)xyz[3 * i + 1], (double)xyz[3 * i + 2]};
  const int cnt = dgr_gather_in_radius(xyz, p, cell, reach, r2, gap_limit, batch, s, keys, vals, mask, kd, kj);
  // candidate k is kept when fewer than max_nn keys rank before it
  const typename S::Point q = sums.point(i);
  double mm[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = lane; k < cnt; k += 32) {
    const int32_t jk = kj[k];
    if (dgr_key_rank(kd, kj, cnt, kd[k], jk) < max_nn) {
      double e[3];
      dgr_offset_d2(xyz, jk, p, e);
      sums.add(q, mm, e, jk);
    }
  }
#pragma unroll
  for (int d = 1; d < 32; d <<= 1)
#pragma unroll
    for (int k = 0; k < 9; ++k) mm[k] += __shfl_xor_sync(0xffffffffu, mm[k], d);
  if (lane == 0) sums.store(mm, max_nn, i);
}

// ---------------------------------------------------------------------------------------
// ICP: all max_iter + 1 (match, update) launch pairs are enqueued up front and turn into no-ops once the
// device-side `done` flag is set, so a call makes no host round trip
// ---------------------------------------------------------------------------------------
struct IcpState {
  double T[12];          // current pose, row-major [R | t]
  double prev_fitness, prev_rmse, fitness, rmse, n_corr;
  int iteration, done;
};

__global__ void icp_init_kernel(const double* __restrict__ T_init, IcpState* st) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    for (int k = 0; k < 12; ++k) st->T[k] = T_init[k];
    st->prev_fitness = st->prev_rmse = st->fitness = st->rmse = st->n_corr = 0.0;
    st->iteration = 0;
    st->done = 0;
  }
}

// What the estimators read besides the matched pair: target normals (point-to-plane, colored), for colored ICP the
// target colour gradients and intensities, the source intensities and sqrt(lambda), sqrt(1 - lambda), for
// generalized ICP both clouds' covariances, and the robust loss (DGR_LOSS_*) and its scale k of a weighted estimator
struct IcpInputs {
  const float* tnorm;
  const float* tgrad;
  const float* tint;
  const float* sint;
  double sqrt_geo, sqrt_photo;
  const double* scov;
  const double* tcov;
  int loss;
  double loss_k;
};

// open3d's RobustKernel::Weight(r) of the DGR_LOSS_* losses, scale k; L1 gives 0 at r = 0 (open3d: infinity)
__device__ __forceinline__ double loss_weight(int loss, double k, double r) {
  const double a = fabs(r);
  switch (loss) {
    case DGR_LOSS_L1: return a > 0.0 ? 1.0 / a : 0.0;
    case DGR_LOSS_HUBER: return a <= k ? 1.0 : k / a;
    case DGR_LOSS_CAUCHY: { const double u = r / k; return 1.0 / (1.0 + u * u); }
    case DGR_LOSS_GM: { const double d = k + r * r; return k / (d * d); }
    case DGR_LOSS_TUKEY: { const double u = fmin(1.0, a / k), e = 1.0 - u * u; return e * e; }
    default: return 1.0;
  }
}

// open3d's TransformationEstimationPointToPoint: sums n, sum d^2, sum p (3), sum q (3), sum q p^T (9) over the
// correspondences (p = current transformed source point, q its target point); the step is the Kabsch rotation of
// the centred cross-covariance, composed on the left (the identity without correspondences)
struct PointToPoint {
  using Update = PointToPoint;
  static constexpr int kNv = 17, kCount = 0, kD2 = 1;
  __device__ __forceinline__ static void accumulate(const double p[3], const double q[3], const IcpInputs&,
                                                    const double*, int64_t, int64_t, double d2, int sub,
                                                    double* acc) {
    add_sum(acc, sub, 0, 1.0);
    add_sum(acc, sub, 1, d2);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      add_sum(acc, sub, 2 + a, p[a]);
      add_sum(acc, sub, 5 + a, q[a]);
#pragma unroll
      for (int b = 0; b < 3; ++b) add_sum(acc, sub, 8 + 3 * a + b, q[a] * p[b]);
    }
  }
  __device__ __forceinline__ static void step(const double* tot, double* T) {
    const double n = tot[kCount];
    double R[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}, t[3] = {0, 0, 0};
    if (n > 0) {
      double mp[3], mq[3], S[3][3];
      for (int a = 0; a < 3; ++a) { mp[a] = tot[2 + a] / n; mq[a] = tot[5 + a] / n; }
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) S[a][b] = tot[8 + 3 * a + b] / n - mq[a] * mp[b];
      kabsch_rotation(S, R);
      for (int a = 0; a < 3; ++a) t[a] = mq[a] - (R[a][0] * mp[0] + R[a][1] * mp[1] + R[a][2] * mp[2]);
    }
    double Tn[12];
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 4; ++b) {
        double v = R[a][0] * T[b] + R[a][1] * T[4 + b] + R[a][2] * T[8 + b];
        if (b == 3) v += t[a];
        Tn[4 * a + b] = v;
      }
    }
    for (int q = 0; q < 12; ++q) T[q] = Tn[q];
  }
};

// open3d's TransformationEstimationPointToPlane: with the target normal n, r = (s - q).n and J = [s x n, n]; sums
// J^T J (upper triangle, 21), J^T r (6), n, sum d^2; the step solves J^T J x = -J^T r by Cholesky (a non-positive
// pivot - no match, a single plane - gives the identity) and composes [Rz(x2) Ry(x1) Rx(x0) | x3..5] on the left.
// kW: the row weighted by loss_weight(r) (open3d >= 0.12's kernel argument).
template <bool kW>
struct PointToPlaneT {
  using Update = PointToPlaneT<false>;
  static constexpr int kNv = 29, kCount = 27, kD2 = 28;
  __device__ __forceinline__ static void accumulate(const double p[3], const double q[3], const IcpInputs& in,
                                                    const double*, int64_t, int64_t j, double d2, int sub,
                                                    double* acc) {
    const float* __restrict__ tnorm = in.tnorm;
    const double nv[3] = {tnorm[3 * j], tnorm[3 * j + 1], tnorm[3 * j + 2]};
    const double r = (p[0] - q[0]) * nv[0] + (p[1] - q[1]) * nv[1] + (p[2] - q[2]) * nv[2];
    const double J[6] = {p[1] * nv[2] - p[2] * nv[1], p[2] * nv[0] - p[0] * nv[2], p[0] * nv[1] - p[1] * nv[0],
                         nv[0], nv[1], nv[2]};
    add_row<kW>(acc, sub, J, r, kW ? loss_weight(in.loss, in.loss_k, r) : 1.0);
    add_sum(acc, sub, 27, 1.0);
    add_sum(acc, sub, 28, d2);
  }
  __device__ __forceinline__ static void step(const double* tot, double* T) {
    double x[6], T0[12];
    if (!cholesky6_step(tot, tot + 21, x))
      for (int q = 0; q < 6; ++q) x[q] = 0.0;
    for (int q = 0; q < 12; ++q) T0[q] = T[q];
    zyx_update_left(x, T0, T);
  }
};
using PointToPlane = PointToPlaneT<false>;

// open3d's TransformationEstimationForColoredICP(lambda): two rows per correspondence (source point s = p, target
// point q, normal n, colour gradient d, intensities I_s, I_t), both added into PointToPlane's 29 sums and step:
//   geometric    r = sqrt(lambda) (s - q).n,  J = sqrt(lambda) [s x n, n];
//   photometric  with s' = s - ((s - q).n) n and m = -(I - n n^T) d = (d.n) n - d:
//                r = sqrt(1 - lambda) (I_s - (d.(s' - q) + I_t)),  J = sqrt(1 - lambda) [s x m, m].
// At lambda = 1 the photometric row is exactly zero and the sums are PointToPlane's.  kW: each row weighted by
// loss_weight of its own (scaled) residual, as open3d >= 0.12 does.
template <bool kW>
struct ColoredT {
  using Update = PointToPlane;
  __device__ __forceinline__ static void accumulate(const double p[3], const double q[3], const IcpInputs& in,
                                                    const double*, int64_t i, int64_t j, double d2, int sub,
                                                    double* acc) {
    const double nv[3] = {in.tnorm[3 * j], in.tnorm[3 * j + 1], in.tnorm[3 * j + 2]};
    const double dv[3] = {in.tgrad[3 * j], in.tgrad[3 * j + 1], in.tgrad[3 * j + 2]};
    const double rg = (p[0] - q[0]) * nv[0] + (p[1] - q[1]) * nv[1] + (p[2] - q[2]) * nv[2];
    const double dn = dv[0] * nv[0] + dv[1] * nv[1] + dv[2] * nv[2];
    const double mv[3] = {dn * nv[0] - dv[0], dn * nv[1] - dv[1], dn * nv[2] - dv[2]};
    const double w[3] = {p[0] - rg * nv[0] - q[0], p[1] - rg * nv[1] - q[1], p[2] - rg * nv[2] - q[2]};
    const double rp = (double)in.sint[i] - ((dv[0] * w[0] + dv[1] * w[1] + dv[2] * w[2]) + (double)in.tint[j]);
#pragma unroll
    for (int row = 0; row < 2; ++row) {
      const double* v = row == 0 ? nv : mv;
      const double sc = row == 0 ? in.sqrt_geo : in.sqrt_photo;
      const double r = sc * (row == 0 ? rg : rp);
      const double J[6] = {sc * (p[1] * v[2] - p[2] * v[1]), sc * (p[2] * v[0] - p[0] * v[2]),
                           sc * (p[0] * v[1] - p[1] * v[0]), sc * v[0], sc * v[1], sc * v[2]};
      add_row<kW>(acc, sub, J, r, kW ? loss_weight(in.loss, in.loss_k, r) : 1.0);
    }
    add_sum(acc, sub, 27, 1.0);
    add_sum(acc, sub, 28, d2);
  }
};

// open3d's TransformationEstimationForGeneralizedICP (Segal, Haehnel & Thrun 2009): with the source covariance
// rotated by the current pose, C_s' = R C_s R^T, and M = C_s' + C_t, three rows per correspondence k = 0..2 with
// v = W[k], W = M^(-1/2) (the principal root, from the eigenvectors jacobi_svd3 gives for a positive-definite M):
// r = v.(s - q), J = [s x v, v], into PointToPlane's 29 sums and step.  A correspondence whose M fails a 3x3
// Cholesky (a non-positive pivot) adds no row; it still counts towards fitness and RMSE.  kW: each row weighted by
// loss_weight(r).
template <bool kW>
struct GeneralizedT {
  using Update = PointToPlane;
  __device__ __forceinline__ static void accumulate(const double p[3], const double q[3], const IcpInputs& in,
                                                    const double T[12], int64_t i, int64_t j, double d2, int sub,
                                                    double* acc) {
    const double* cs = in.scov + 6 * i;
    const double* ct = in.tcov + 6 * j;
    const double C[3][3] = {{cs[0], cs[1], cs[2]}, {cs[1], cs[3], cs[4]}, {cs[2], cs[4], cs[5]}};
    double RC[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) RC[a][b] = T[4 * a] * C[0][b] + T[4 * a + 1] * C[1][b] + T[4 * a + 2] * C[2][b];
    double M[3][3];
    M[0][0] = RC[0][0] * T[0] + RC[0][1] * T[1] + RC[0][2] * T[2] + ct[0];
    M[0][1] = RC[0][0] * T[4] + RC[0][1] * T[5] + RC[0][2] * T[6] + ct[1];
    M[0][2] = RC[0][0] * T[8] + RC[0][1] * T[9] + RC[0][2] * T[10] + ct[2];
    M[1][1] = RC[1][0] * T[4] + RC[1][1] * T[5] + RC[1][2] * T[6] + ct[3];
    M[1][2] = RC[1][0] * T[8] + RC[1][1] * T[9] + RC[1][2] * T[10] + ct[4];
    M[2][2] = RC[2][0] * T[8] + RC[2][1] * T[9] + RC[2][2] * T[10] + ct[5];
    M[1][0] = M[0][1]; M[2][0] = M[0][2]; M[2][1] = M[1][2];
    add_sum(acc, sub, 27, 1.0);
    add_sum(acc, sub, 28, d2);
    // M's Cholesky pivots in order; W needs a positive-definite M
    const double d0 = M[0][0];
    if (!(d0 > 0.0)) return;
    const double l10 = M[1][0] / sqrt(d0), l20 = M[2][0] / sqrt(d0);
    const double d1 = M[1][1] - l10 * l10;
    if (!(d1 > 0.0)) return;
    const double l21 = (M[2][1] - l20 * l10) / sqrt(d1);
    if (!(M[2][2] - l20 * l20 - l21 * l21 > 0.0)) return;
    double A[3][3], V[3][3], sig[3];
    jacobi_svd3(M, A, V, sig);
    const double is[3] = {1.0 / sqrt(sig[0]), 1.0 / sqrt(sig[1]), 1.0 / sqrt(sig[2])};
    const double e[3] = {p[0] - q[0], p[1] - q[1], p[2] - q[2]};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double v[3];
#pragma unroll
      for (int b = 0; b < 3; ++b)
        v[b] = V[k][0] * is[0] * V[b][0] + V[k][1] * is[1] * V[b][1] + V[k][2] * is[2] * V[b][2];
      const double r = v[0] * e[0] + v[1] * e[1] + v[2] * e[2];
      const double J[6] = {p[1] * v[2] - p[2] * v[1], p[2] * v[0] - p[0] * v[2], p[0] * v[1] - p[1] * v[0],
                           v[0], v[1], v[2]};
      add_row<kW>(acc, sub, J, r, kW ? loss_weight(in.loss, in.loss_k, r) : 1.0);
    }
  }
};

// Every estimator E names the estimator whose sums layout (kNv, kCount, kD2) and step icp_update_kernel runs
// (E::Update): its own, or PointToPlane's for those that add rows into the same 29 sums.
// kNv = E::Update::kNv sums in (kNv + 7) / 8 accumulators per lane.  Per-block partials: part[block][k], summed lanes
// by butterfly and warps in order.
template <class E>
__global__ void __launch_bounds__(kIcpThreads)
icp_match_kernel(const float* __restrict__ src, int64_t n_src, const float* __restrict__ tgt, const IcpInputs in,
                 const dgr_keyspec_t* __restrict__ spec_p,
                 const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int32_t batch,
                 double voxel, double max_dist, const IcpState* __restrict__ st, double* __restrict__ part) {
  constexpr int kNv = E::Update::kNv, kSlots = (kNv + 7) / 8;
  if (st->done) return;
  const dgr_keyspec_t s = *spec_p;
  double T[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) T[k] = st->T[k];
  double acc[kSlots];
#pragma unroll
  for (int a = 0; a < kSlots; ++a) acc[a] = 0.0;
  const int reach = (int)ceil(max_dist / voxel);
  const int sub = threadIdx.x & 7;
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) >> 3;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3; i0 < ((n_src + groups - 1) / groups) * groups;
       i0 += groups) {
    const bool have = i0 < n_src;                       // whole warps stay in the loop for the shuffles
    const int64_t i = have ? i0 : 0;
    const double x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
    const double p[3] = {T[0] * x + T[1] * y + T[2] * z + T[3], T[4] * x + T[5] * y + T[6] * z + T[7],
                         T[8] * x + T[9] * y + T[10] * z + T[11]};
    double best = max_dist * max_dist;
    int best_j;
    dgr_voxel_nearest8(p, have, sub, tgt, s, keys, vals, mask, batch, voxel, reach, best, best_j);
    if (have && best_j >= 0) {                          // every lane of the group has the match
      const int64_t j = best_j;
      const double q[3] = {tgt[3 * j], tgt[3 * j + 1], tgt[3 * j + 2]};
      E::accumulate(p, q, in, T, i, j, best, sub, acc);
    }
  }
  __shared__ double red[kIcpThreads / 32][kIcpStride];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < kSlots; ++a) {
    double v = acc[a];
    v += __shfl_xor_sync(0xffffffffu, v, 8);            // the 4 groups of the warp, same sub
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    if (lane < 8) red[warp][8 * a + lane] = v;
  }
  __syncthreads();
  if (threadIdx.x < kNv) {
    double v = 0.0;
    for (int w = 0; w < kIcpThreads / 32; ++w) v += red[w][threadIdx.x];
    part[(int64_t)blockIdx.x * kIcpStride + threadIdx.x] = v;
  }
}

// one block of E::kNv warps: warp k sums partial k over the blocks (lane-strided, then butterfly)
template <class E>
__global__ void __launch_bounds__(E::kNv * 32)
icp_update_kernel(IcpState* st, const double* __restrict__ part, int n_blocks, int64_t n_src, int max_iter,
                  double rel_fitness, double rel_rmse, double* __restrict__ result) {
  __shared__ double tot[kIcpStride];
  const bool live = !st->done;                          // uniform per launch
  if (live) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double v = 0.0;
    for (int b = lane; b < n_blocks; b += 32) v += part[(int64_t)b * kIcpStride + warp];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (lane == 0) tot[warp] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  if (live) {
    const double n = tot[E::kCount];
    double fitness, rmse;
    const bool stop = icp_stop_rule(*st, n, tot[E::kD2], n_src, max_iter, rel_fitness, rel_rmse, fitness, rmse);
    const int k = st->iteration;
    st->fitness = fitness;
    st->rmse = rmse;
    st->n_corr = n;
    if (stop) {
      st->done = 1;
    } else {
      E::step(tot, st->T);
      st->prev_fitness = fitness;
      st->prev_rmse = rmse;
      st->iteration = k + 1;
    }
  }
  for (int q = 0; q < 12; ++q) result[q] = st->T[q];
  result[12] = 0.0; result[13] = 0.0; result[14] = 0.0; result[15] = 1.0;
  result[16] = st->fitness;
  result[17] = st->rmse;
  result[18] = (double)st->iteration;
  result[19] = st->n_corr;
}

inline int icp_blocks(int64_t n_src) {
  unsigned blocks = dgr_blocks(n_src * 8, kIcpThreads);     // 8 lanes per source point
  return blocks > (unsigned)kIcpMaxBlocks ? kIcpMaxBlocks : (int)blocks;
}

// workspace size in 8-byte words; carves `base` into the state and the per-block partials when it is not null
int64_t icp_layout(int64_t n_src, double* base, IcpState** state, double** part) {
  static_assert(sizeof(IcpState) <= kIcpState * sizeof(double), "state workspace too small");
  DgrCarver c(base);
  IcpState* s = reinterpret_cast<IcpState*>(c.take<double>(kIcpState));
  double* p = c.take<double>((int64_t)icp_blocks(n_src) * kIcpStride);
  if (state != nullptr) { *state = s; *part = p; }
  return c.words;
}

// the two passes of a neighbourhood search over the cloud's own hash (normals, colour gradients), checked first
template <class S>
int32_t nbr_launch(const float* xyz, int64_t n, const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals,
                   int64_t cap, int32_t batch, double cell, double radius, int32_t max_nn, const S& sums,
                   int32_t* counts, void* stream) {
  DGR_ARG_CHECK(n >= 0 && n < (1ll << 31), "point count out of range");
  DGR_ARG_CHECK(n == 0 || (xyz != nullptr && spec != nullptr && keys != nullptr && vals != nullptr &&
                           counts != nullptr), "null pointer");
  DGR_TRY(dgr_check_hash_search(cap, cell, radius, kMaxReach));
  DGR_ARG_CHECK(max_nn >= 1 && max_nn <= kMaxNN, "max_nn must lie in [1, 64]");
  if (n == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int reach = (int)ceil(radius / cell);
  const double r2 = radius * radius, gap_limit = dgr_gap_limit(radius, cell);
  const int slots = dgr_live_cells(reach, gap_limit);
  nbr_probe_kernel<S><<<dgr_blocks(n * 8, kNormThreads), kNormThreads, 0, st>>>(
      xyz, n, spec, keys, vals, (uint64_t)cap - 1, batch, cell, reach, r2, max_nn, sums, counts);
  const size_t smem = (size_t)kSelWarps * slots * (sizeof(double) + sizeof(int32_t));   // <= 35 KB (reach 4)
  nbr_select_kernel<S><<<dgr_blocks(n, kSelWarps), kSelWarps * 32, smem, st>>>(
      xyz, n, spec, keys, vals, (uint64_t)cap - 1, batch, cell, reach, r2, gap_limit, slots, max_nn, sums, counts);
  dgr_note_launches(2);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

// enqueue init and max_iter + 1 (match, update) pairs of estimator E; the arguments are checked by the caller
template <class E>
void icp_run(const float* src, int64_t n_src, const float* tgt, const IcpInputs& in, const dgr_keyspec_t* spec,
             const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch, double voxel, double max_dist,
             const double* T_init, int32_t max_iter, double rel_fitness, double rel_rmse, double* ws, double* result,
             cudaStream_t st) {
  IcpState* state;
  double* part;
  icp_layout(n_src, ws, &state, &part);
  const int blocks = icp_blocks(n_src);
  icp_init_kernel<<<1, 32, 0, st>>>(T_init, state);
  for (int k = 0; k <= max_iter; ++k) {
    icp_match_kernel<E><<<blocks, kIcpThreads, 0, st>>>(src, n_src, tgt, in, spec, keys, vals, (uint64_t)cap - 1,
                                                        batch, voxel, max_dist, state, part);
    icp_update_kernel<typename E::Update><<<1, E::Update::kNv * 32, 0, st>>>(state, part, blocks, n_src, max_iter,
                                                                     rel_fitness, rel_rmse, result);
  }
  dgr_note_launches(1 + 2 * (max_iter + 1));
}

// estimator E<false> for the L2 loss (today's unweighted code), E<true> with the loss weight otherwise
template <template <bool> class E>
void icp_run_loss(const float* src, int64_t n_src, const float* tgt, const IcpInputs& in, const dgr_keyspec_t* spec,
                  const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch, double voxel, double max_dist,
                  const double* T_init, int32_t max_iter, double rel_fitness, double rel_rmse, double* ws,
                  double* result, cudaStream_t st) {
  if (in.loss == DGR_LOSS_L2)
    icp_run<E<false>>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                      rel_fitness, rel_rmse, ws, result, st);
  else
    icp_run<E<true>>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                     rel_fitness, rel_rmse, ws, result, st);
}

// a DGR_LOSS_* id, and for the losses with a scale a finite k > 0
int32_t check_loss(int32_t loss, double loss_k) {
  DGR_ARG_CHECK(loss >= DGR_LOSS_L2 && loss <= DGR_LOSS_TUKEY, "unknown loss");
  DGR_ARG_CHECK(loss == DGR_LOSS_L2 || loss == DGR_LOSS_L1 || (loss_k > 0.0 && loss_k < INFINITY),
                "loss_k must be finite and positive");
  return DGR_OK;
}

// the checks every ICP entry point makes before it enqueues
int32_t check_icp(int64_t cap, double voxel, double max_dist, int32_t max_iter, int64_t n_src, const double* T_init,
                  const double* ws, const double* result, const dgr_keyspec_t* spec) {
  DGR_TRY(dgr_check_hash_search(cap, voxel, max_dist, kMaxReach));
  DGR_ARG_CHECK(max_iter >= 0, "bad ICP parameters");
  DGR_ARG_CHECK(n_src >= 0 && n_src < (1ll << 31), "point count out of range");
  DGR_ARG_CHECK(T_init != nullptr && ws != nullptr && result != nullptr && spec != nullptr, "null pointer");
  return DGR_OK;
}

}  // namespace

extern "C" {

int32_t dgr_estimate_normals(const float* xyz, int64_t n, const dgr_keyspec_t* spec, const uint64_t* keys,
                             const int32_t* vals, int64_t cap, int32_t batch, double cell, double radius,
                             int32_t max_nn, const float* prev, float* normals, int32_t* counts, void* stream) {
  DGR_ARG_CHECK(n == 0 || normals != nullptr, "null pointer");
  return nbr_launch(xyz, n, spec, keys, vals, cap, batch, cell, radius, max_nn, NormalSums{prev, normals}, counts,
                    stream);
}

int32_t dgr_color_gradient(const float* xyz, const float* normals, const float* intensity, int64_t n,
                           const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals, int64_t cap,
                           int32_t batch, double cell, double radius, int32_t max_nn, float* grad, int32_t* counts,
                           void* stream) {
  DGR_ARG_CHECK(n == 0 || (normals != nullptr && intensity != nullptr && grad != nullptr), "null pointer");
  return nbr_launch(xyz, n, spec, keys, vals, cap, batch, cell, radius, max_nn,
                    GradientSums{normals, intensity, grad}, counts, stream);
}

int32_t dgr_estimate_covariances(const float* xyz, int64_t n, const dgr_keyspec_t* spec, const uint64_t* keys,
                                 const int32_t* vals, int64_t cap, int32_t batch, double cell, double radius,
                                 int32_t max_nn, double* cov, int32_t* counts, void* stream) {
  DGR_ARG_CHECK(n == 0 || cov != nullptr, "null pointer");
  return nbr_launch(xyz, n, spec, keys, vals, cap, batch, cell, radius, max_nn, CovarianceSums{cov}, counts, stream);
}

int32_t dgr_covariances_from_normals(const float* normals, int64_t n, double epsilon, double* cov, void* stream) {
  DGR_ARG_CHECK(n >= 0 && n < (1ll << 31), "point count out of range");
  DGR_ARG_CHECK(epsilon > 0.0 && epsilon < INFINITY, "epsilon must be finite and positive");
  DGR_ARG_CHECK(n == 0 || (normals != nullptr && cov != nullptr), "null pointer");
  if (n == 0) return DGR_OK;
  cov_from_normals_kernel<<<dgr_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(normals, n, epsilon, cov);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_icp_ws_elems(int64_t n_src, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_src >= 0, "bad arguments");
  *n_elems = icp_layout(n_src, nullptr, nullptr, nullptr);
  return DGR_OK;
}

int32_t dgr_icp(const float* src, int64_t n_src, const float* tgt, const float* tgt_normals, const dgr_keyspec_t* spec,
                const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch, double voxel, double max_dist,
                const double* T_init, int32_t max_iter, double rel_fitness, double rel_rmse, double* ws,
                double* result, void* stream) {
  DGR_TRY(check_icp(cap, voxel, max_dist, max_iter, n_src, T_init, ws, result, spec));
  cudaStream_t st = (cudaStream_t)stream;
  const IcpInputs in{tgt_normals, nullptr, nullptr, nullptr, 1.0, 0.0, nullptr, nullptr, DGR_LOSS_L2, 0.0};
  if (tgt_normals != nullptr)
    icp_run<PointToPlane>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                          rel_fitness, rel_rmse, ws, result, st);
  else
    icp_run<PointToPoint>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                          rel_fitness, rel_rmse, ws, result, st);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_icp_loss(const float* src, int64_t n_src, const float* tgt, const float* tgt_normals,
                     const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals, int64_t cap, int32_t batch,
                     double voxel, double max_dist, int32_t loss, double loss_k, const double* T_init,
                     int32_t max_iter, double rel_fitness, double rel_rmse, double* ws, double* result,
                     void* stream) {
  DGR_TRY(check_icp(cap, voxel, max_dist, max_iter, n_src, T_init, ws, result, spec));
  DGR_TRY(check_loss(loss, loss_k));
  DGR_ARG_CHECK(tgt_normals != nullptr, "null pointer: point-to-plane ICP needs target normals");
  const IcpInputs in{tgt_normals, nullptr, nullptr, nullptr, 1.0, 0.0, nullptr, nullptr, loss, loss_k};
  icp_run_loss<PointToPlaneT>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                              rel_fitness, rel_rmse, ws, result, (cudaStream_t)stream);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_colored_icp_loss(const float* src, const float* src_intensity, int64_t n_src, const float* tgt,
                             const float* tgt_normals, const float* tgt_intensity, const float* tgt_grad,
                             const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals, int64_t cap,
                             int32_t batch, double voxel, double max_dist, double lambda_geometric, int32_t loss,
                             double loss_k, const double* T_init, int32_t max_iter, double rel_fitness,
                             double rel_rmse, double* ws, double* result, void* stream) {
  DGR_TRY(check_icp(cap, voxel, max_dist, max_iter, n_src, T_init, ws, result, spec));
  DGR_TRY(check_loss(loss, loss_k));
  DGR_ARG_CHECK(lambda_geometric >= 0.0 && lambda_geometric <= 1.0, "lambda_geometric must lie in [0, 1]");
  DGR_ARG_CHECK(keys != nullptr && vals != nullptr && tgt != nullptr && tgt_normals != nullptr &&
                tgt_intensity != nullptr && tgt_grad != nullptr &&
                (n_src == 0 || (src != nullptr && src_intensity != nullptr)), "null pointer");
  const IcpInputs in{tgt_normals, tgt_grad, tgt_intensity, src_intensity, sqrt(lambda_geometric),
                     sqrt(1.0 - lambda_geometric), nullptr, nullptr, loss, loss_k};
  icp_run_loss<ColoredT>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                         rel_fitness, rel_rmse, ws, result, (cudaStream_t)stream);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_colored_icp(const float* src, const float* src_intensity, int64_t n_src, const float* tgt,
                        const float* tgt_normals, const float* tgt_intensity, const float* tgt_grad,
                        const dgr_keyspec_t* spec, const uint64_t* keys, const int32_t* vals, int64_t cap,
                        int32_t batch, double voxel, double max_dist, double lambda_geometric, const double* T_init,
                        int32_t max_iter, double rel_fitness, double rel_rmse, double* ws, double* result,
                        void* stream) {
  return dgr_colored_icp_loss(src, src_intensity, n_src, tgt, tgt_normals, tgt_intensity, tgt_grad, spec, keys, vals,
                              cap, batch, voxel, max_dist, lambda_geometric, DGR_LOSS_L2, 0.0, T_init, max_iter,
                              rel_fitness, rel_rmse, ws, result, stream);
}

int32_t dgr_generalized_icp(const float* src, const double* src_cov, int64_t n_src, const float* tgt,
                            const double* tgt_cov, const dgr_keyspec_t* spec, const uint64_t* keys,
                            const int32_t* vals, int64_t cap, int32_t batch, double voxel, double max_dist,
                            int32_t loss, double loss_k, const double* T_init, int32_t max_iter, double rel_fitness,
                            double rel_rmse, double* ws, double* result, void* stream) {
  DGR_TRY(check_icp(cap, voxel, max_dist, max_iter, n_src, T_init, ws, result, spec));
  DGR_TRY(check_loss(loss, loss_k));
  DGR_ARG_CHECK(src_cov != nullptr && tgt_cov != nullptr, "null pointer: generalized ICP needs both covariances");
  DGR_ARG_CHECK(keys != nullptr && vals != nullptr && tgt != nullptr && (n_src == 0 || src != nullptr),
                "null pointer");
  const IcpInputs in{nullptr, nullptr, nullptr, nullptr, 1.0, 0.0, src_cov, tgt_cov, loss, loss_k};
  icp_run_loss<GeneralizedT>(src, n_src, tgt, in, spec, keys, vals, cap, batch, voxel, max_dist, T_init, max_iter,
                             rel_fitness, rel_rmse, ws, result, (cudaStream_t)stream);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

}  // extern "C"
