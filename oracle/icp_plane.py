"""ORACLE (test infrastructure only) - point-to-plane ICP: open3d 0.10's ``registration_icp(source, target,
max_correspondence_distance, init, TransformationEstimationPointToPlane())`` with the default
ICPConvergenceCriteria, the GPU's dgr_icp with target normals (csrc/icp.cu).  Target normals come from the caller
(oracle/normals.py, or the GPU's own, to test this stage alone).

PARITY UNPINNED: open3d is not installable offline, so this restates its published RegistrationICP loop in float64
and pins the conventions the GPU follows:

* correspondences: the nearest target point strictly within max_correspondence_distance of the current
  transformed source point (the same search as the point-to-point oracle, oracle/icp.py);
* fitness = correspondences / source points and the inlier RMSE from the EUCLIDEAN nearest distances, as open3d
  computes them for both estimation methods (not the point-to-plane residuals);
* update: r = (s - q).n, J = [s x n, n] per correspondence, J^T J x = -J^T r solved by Cholesky in the loop order of
  the GPU's cholesky6_step; a non-positive pivot (a singular system: no correspondence, a single plane) makes the
  update the identity.  open3d solves with LDLT, which handles rank-deficient systems differently;
* pose: T <- [Rz(x2) Ry(x1) Rx(x0) | x3..5] T, the source transformed by the accumulated T at every step;
* stop at step k when k > 0 and both the fitness and the RMSE changed by less than the tolerances, or at
  k = max_iter (the point-to-point rule); ``iterations`` = updates applied.
"""
import numpy as np
from scipy.spatial import cKDTree


def cholesky_step(A, g):
  """x = -(A^-1 g) for the symmetric 6x6 A, or None on a non-positive pivot."""
  L = np.zeros((6, 6))
  for j in range(6):
    d = A[j, j] - sum(L[j, m] * L[j, m] for m in range(j))
    if not d > 0.0:
      return None
    L[j, j] = np.sqrt(d)
    for i in range(j + 1, 6):
      L[i, j] = (A[i, j] - sum(L[i, m] * L[j, m] for m in range(j))) / L[j, j]
  y = np.zeros(6)
  for i in range(6):
    y[i] = (-g[i] - sum(L[i, m] * y[m] for m in range(i))) / L[i, i]
  x = np.zeros(6)
  for i in range(5, -1, -1):
    x[i] = (y[i] - sum(L[m, i] * x[m] for m in range(i + 1, 6))) / L[i, i]
  return x


def zyx_update(x):
  """4x4 [Rz(x2) Ry(x1) Rx(x0) | x3..5] (open3d's TransformVector6dToMatrix4d)."""
  ca, sa, cb, sb, cc, sc = np.cos(x[0]), np.sin(x[0]), np.cos(x[1]), np.sin(x[1]), np.cos(x[2]), np.sin(x[2])
  Rz = np.array([[cc, -sc, 0.0], [sc, cc, 0.0], [0.0, 0.0, 1.0]])
  Ry = np.array([[cb, 0.0, sb], [0.0, 1.0, 0.0], [-sb, 0.0, cb]])
  Rx = np.array([[1.0, 0.0, 0.0], [0.0, ca, -sa], [0.0, sa, ca]])
  U = np.eye(4)
  U[:3, :3] = Rz @ Ry @ Rx
  U[:3, 3] = x[3:]
  return U


def icp_point_to_plane(src, tgt, tgt_normals, max_dist, T_init=None, max_iter=30, rel_fitness=1e-6, rel_rmse=1e-6):
  """-> (4x4 pose, dict(fitness, inlier_rmse, iterations, n_corr, solves_failed))."""
  src, tgt = np.asarray(src, np.float64).reshape(-1, 3), np.asarray(tgt, np.float64).reshape(-1, 3)
  nrm = np.asarray(tgt_normals, np.float64).reshape(-1, 3)
  T = np.eye(4) if T_init is None else np.array(T_init, np.float64)
  tree = cKDTree(tgt) if len(tgt) else None
  failed = 0
  pf = pr = 0.0
  k = 0
  while True:
    s = src @ T[:3, :3].T + T[:3, 3]
    if tree is not None and len(s):
      d, j = tree.query(s, k=1, distance_upper_bound=max_dist)
      m = np.isfinite(d)
    else:
      d, j, m = np.zeros(len(s)), np.zeros(len(s), np.int64), np.zeros(len(s), bool)
    n = int(m.sum())
    fit = n / len(s) if len(s) else 0.0
    rmse = float(np.sqrt((d[m] ** 2).sum() / n)) if n else 0.0
    if (k > 0 and abs(pf - fit) < rel_fitness and abs(pr - rmse) < rel_rmse) or k >= max_iter:
      break
    sm, q, nq = s[m], tgt[j[m]], nrm[j[m]]
    r = ((sm - q) * nq).sum(1)
    J = np.concatenate([np.cross(sm, nq), nq], axis=1)
    x = cholesky_step(J.T @ J, J.T @ r)
    if x is None:
      failed += 1
      x = np.zeros(6)
    T = zyx_update(x) @ T
    pf, pr = fit, rmse
    k += 1
  return T, dict(fitness=fit, inlier_rmse=rmse, iterations=k, n_corr=n, solves_failed=failed)
