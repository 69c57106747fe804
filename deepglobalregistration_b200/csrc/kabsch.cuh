// Small fp64 solvers shared by registration.cu (weighted Procrustes), ransac.cu (4-point hypotheses), fgr.cu and
// pointnetlk.cu (Gauss-Newton / Lucas-Kanade steps), icp.cu (normals, ICP steps), goicp.cu (trimmed ICP),
// super4pcs.cu (congruent-set fits) and odometry.cu (RGB-D odometry steps).
#pragma once

// ---------------------------------------------------------------------------------------
// 3x3 SVD (one-sided Jacobi, fp64) -> proper rotation U diag(1,1,det(U)det(V)) V^T
// ---------------------------------------------------------------------------------------
__device__ inline double det3(const double m[3][3]) {
  return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) -
         m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
         m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}

// One-sided Jacobi sweeps on S: on return A = S V has orthogonal columns, V is orthogonal and sig[j] = |A[:, j]|
// (the singular values, unsorted).  For a symmetric positive semi-definite S the columns of V are its eigenvectors
// and sig its eigenvalues.
__device__ __forceinline__ void jacobi_svd3(const double S[3][3], double A[3][3], double V[3][3], double sig[3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      A[i][j] = S[i][j];
      V[i][j] = (i == j) ? 1.0 : 0.0;
    }
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int k = 0; k < 3; ++k) {
          alpha += A[k][p] * A[k][p];
          beta += A[k][q] * A[k][q];
          gamma += A[k][p] * A[k][q];
        }
        if (fabs(gamma) <= 1e-300 || fabs(gamma) <= 1e-17 * sqrt(alpha * beta)) continue;
        rotated = true;
        double zeta = (beta - alpha) / (2.0 * gamma);
        double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int k = 0; k < 3; ++k) {
          double ap = A[k][p], aq = A[k][q];
          A[k][p] = c * ap - s * aq;
          A[k][q] = s * ap + c * aq;
          double vp = V[k][p], vq = V[k][q];
          V[k][p] = c * vp - s * vq;
          V[k][q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  for (int j = 0; j < 3; ++j) sig[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
}

__device__ inline void kabsch_rotation(const double S[3][3], double R[3][3]) {
  double A[3][3], V[3][3], sig[3];
  jacobi_svd3(S, A, V, sig);
  int ord[3] = {0, 1, 2};   // descending singular values
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (sig[ord[b]] > sig[ord[a]]) { int tmp = ord[a]; ord[a] = ord[b]; ord[b] = tmp; }
  if (sig[ord[0]] <= 1e-300) {   // zero covariance (all points coincide): LAPACK returns U = V = I
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[i][j] = (i == j) ? 1.0 : 0.0;
    return;
  }
  double U[3][3], W[3][3];
  const double tiny = 1e-300 + 1e-14 * sig[ord[0]];
  for (int j = 0; j < 3; ++j) {
    int o = ord[j];
    for (int k = 0; k < 3; ++k) {
      W[k][j] = V[k][o];
      U[k][j] = sig[o] > tiny ? A[k][o] / sig[o] : 0.0;
    }
  }
  if (sig[ord[1]] <= tiny) {   // rank <= 1: complete with any unit vector orthogonal to u0
    double ax = fabs(U[0][0]), ay = fabs(U[1][0]), az = fabs(U[2][0]);
    double e[3] = {0, 0, 0};
    e[(ax <= ay && ax <= az) ? 0 : (ay <= az ? 1 : 2)] = 1.0;
    double d = e[0] * U[0][0] + e[1] * U[1][0] + e[2] * U[2][0];
    double v[3] = {e[0] - d * U[0][0], e[1] - d * U[1][0], e[2] - d * U[2][0]};
    double nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if (nv < 1e-300) { v[0] = 1; v[1] = 0; v[2] = 0; nv = 1; }
    for (int k = 0; k < 3; ++k) U[k][1] = v[k] / nv;
  }
  if (sig[ord[2]] <= tiny) {   // rank <= 2: u2 = u0 x u1 (sign is absorbed by the det fix)
    U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
    U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
    U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
  }
  const double sgn = (det3(U) * det3(W) < 0) ? -1.0 : 1.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      R[i][j] = U[i][0] * W[j][0] + U[i][1] * W[j][1] + sgn * U[i][2] * W[j][2];
}

// ---------------------------------------------------------------------------------------
// 6-DoF Gauss-Newton step (FGR, point-to-plane ICP)
// ---------------------------------------------------------------------------------------
// x = -(A^-1 g) by Cholesky of the symmetric A (upper triangle a[21], row-major); false on a non-positive pivot
__device__ inline bool cholesky6_step(const double* a, const double* g, double x[6]) {
  double L[6][6];
  int k = 0;
  double A[6][6];
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) { A[r][c] = a[k]; A[c][r] = a[k]; ++k; }
  for (int j = 0; j < 6; ++j) {
    double d = A[j][j];
    for (int m = 0; m < j; ++m) d -= L[j][m] * L[j][m];
    if (!(d > 0.0)) return false;
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < 6; ++i) {
      double e = A[i][j];
      for (int m = 0; m < j; ++m) e -= L[i][m] * L[j][m];
      L[i][j] = e / L[j][j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double e = -g[i];
    for (int m = 0; m < i; ++m) e -= L[i][m] * y[m];
    y[i] = e / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double e = y[i];
    for (int m = i + 1; m < 6; ++m) e -= L[m][i] * x[m];
    x[i] = e / L[i][i];
  }
  return true;
}

// Tn = [Rz(x[2]) Ry(x[1]) Rx(x[0]) | x[3..6)] T, poses row-major [R | t] (open3d's TransformVector6dToMatrix4d)
__device__ __forceinline__ void zyx_update_left(const double x[6], const double T[12], double* Tn) {
  const double ca = cos(x[0]), sa = sin(x[0]), cb = cos(x[1]), sb = sin(x[1]), cc = cos(x[2]), sc = sin(x[2]);
  const double Rz[3][3] = {{cc, -sc, 0.0}, {sc, cc, 0.0}, {0.0, 0.0, 1.0}};
  const double Ry[3][3] = {{cb, 0.0, sb}, {0.0, 1.0, 0.0}, {-sb, 0.0, cb}};
  const double Rx[3][3] = {{1.0, 0.0, 0.0}, {0.0, ca, -sa}, {0.0, sa, ca}};
  double Rzy[3][3], D[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Rzy[r][c] = Rz[r][0] * Ry[0][c] + Rz[r][1] * Ry[1][c] + Rz[r][2] * Ry[2][c];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) D[r][c] = Rzy[r][0] * Rx[0][c] + Rzy[r][1] * Rx[1][c] + Rzy[r][2] * Rx[2][c];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c)
      Tn[4 * r + c] = D[r][0] * T[c] + D[r][1] * T[4 + c] + D[r][2] * T[8 + c] + (c == 3 ? x[3 + r] : 0.0);
}

// ---------------------------------------------------------------------------------------
// The 29 fixed-order Gauss-Newton sums (icp.cu's estimators, odometry.cu): a point's group of 8 lanes shares its rows
// ---------------------------------------------------------------------------------------
// Lane `sub` of a point's group of 8 owns the sums k = 8 a + sub, in its accumulator a
__device__ __forceinline__ void add_sum(double* acc, int sub, int k, double v) {
  if ((k & 7) == sub) acc[k >> 3] += v;
}

// One residual row r, J into the 29 sums J^T J (upper triangle, 21) and J^T r (6); weighted (kW): w J J^T and w J r.
// The unweighted instantiation is the plain products, not a multiply by 1.
template <bool kW>
__device__ __forceinline__ void add_row(double* acc, int sub, const double J[6], double r, double w) {
  int k = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const double wa = kW ? w * J[a] : J[a];
#pragma unroll
    for (int b = a; b < 6; ++b) add_sum(acc, sub, k++, wa * J[b]);
  }
#pragma unroll
  for (int a = 0; a < 6; ++a) add_sum(acc, sub, 21 + a, (kW ? w * J[a] : J[a]) * r);
}

// ---------------------------------------------------------------------------------------
// open3d's RegistrationICP stopping rule (both estimation methods): fitness and inlier RMSE of the correspondences
// found at step k = st.iteration (n of them, squared Euclidean distances summing to sum_d2); the loop stops when both changed by
// less than the tolerances since step k - 1, or at k = max_iter
// ---------------------------------------------------------------------------------------
template <class State>
__device__ __forceinline__ bool icp_stop_rule(const State& st, double n, const double& sum_d2, int64_t n_src, int max_iter,
                                              double rel_fitness, double rel_rmse, double& fitness, double& rmse) {
  fitness = n_src > 0 ? n / (double)n_src : 0.0;
  rmse = n > 0 ? sqrt(sum_d2 / n) : 0.0;
  const int k = st.iteration;
  bool stop = false;
  if (k > 0 && fabs(st.prev_fitness - fitness) < rel_fitness && fabs(st.prev_rmse - rmse) < rel_rmse) stop = true;
  if (k >= max_iter) stop = true;
  return stop;
}
