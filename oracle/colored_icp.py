"""ORACLE (test infrastructure only) - colored ICP: open3d 0.10's ``registration_colored_icp(source, target,
max_distance, init, criteria, lambda_geometric)`` (ColoredICP.cpp; unchanged in >= 0.12 apart from the robust kernel),
the GPU's dgr_color_gradient and dgr_colored_icp (csrc/icp.cu).  Target normals and gradients come from the caller
(oracle/normals.py and color_gradient below, or the GPU's own, to test one stage alone).

PARITY UNPINNED: open3d is not installable offline, so this restates its published algorithm in float64 and pins the
conventions the GPU follows:

* intensity of a point: (r + g + b) / 3 of its colour in [0, 1];
* target colour gradient (InitializePointCloudForColoredICP, KDTreeSearchParamHybrid(2 max_distance, 30) on the
  target): the neighbours of oracle/normals.py (strict radius, the max_nn smallest by (d^2, row), the point itself
  included).  With nn < 4 of them the gradient is 0.  Otherwise every neighbour j other than i gives the row
  u = e - (e.n_i) n_i (e = p_j - p_i) with b = I_j - I_i, and one more row (nn - 1) n_i with b = 0; the gradient
  solves the normal equations (sum u u^T + (nn - 1)^2 n n^T) g = sum u b.  DEPARTURE: open3d calls
  SolveLinearSystemPSD (an LDLT-based solve); here it is a 3x3 Cholesky in fp64 in the loop order of the GPU's
  store_gradient, and a non-positive pivot leaves g = 0, which is open3d's result when its solve fails;
* estimator (TransformationEstimationForColoredICP(lambda_geometric = 0.968)), per correspondence of the current
  transformed source point s and its nearest target point q with normal n, gradient d and intensities I_s, I_t:
    geometric    r = sqrt(lambda) (s - q).n,  J = sqrt(lambda) [s x n, n];
    photometric  s' = s - ((s - q).n) n, m = -(I - n n^T) d:
                 r = sqrt(1 - lambda) (I_s - (d.(s' - q) + I_t)),  J = sqrt(1 - lambda) [s x m, m]
  (r and J of the photometric row share one sign convention, so the step is the Gauss-Newton step of the summed
  squares); J^T J x = -J^T r by the Cholesky of oracle/icp_plane.py (a non-positive pivot gives the identity step,
  which is also open3d's result on a failed solve; open3d solves with LDLT, as for point-to-plane);
* correspondences, fitness, the Euclidean inlier RMSE, the pose update T <- [Rz(x2) Ry(x1) Rx(x0) | x3..5] T and the
  relative-fitness / relative-RMSE / max_iteration stopping rule are oracle/icp_plane.py's: open3d's RegistrationICP
  uses them for every estimator.
"""
import numpy as np
from scipy.spatial import cKDTree

from .icp_plane import cholesky_step, zyx_update
from .normals import neighbours

LAMBDA_GEOMETRIC = 0.968


def intensity(colors):
  """(r + g + b) / 3 of colours [n, 3] in [0, 1]."""
  c = np.asarray(colors, np.float64).reshape(-1, 3)
  return (c[:, 0] + c[:, 1] + c[:, 2]) / 3.0


def solve3(A, b):
  """(g, smallest pivot / largest diagonal entry) of the symmetric positive 3x3 A g = b by Cholesky in the GPU's
  order; (0, pivot ratio) on a non-positive pivot."""
  a00, a01, a02, a11, a12, a22 = A[0, 0], A[0, 1], A[0, 2], A[1, 1], A[1, 2], A[2, 2]
  scale = max(a00, a11, a22, 1e-300)
  if not a00 > 0.0:
    return np.zeros(3), a00 / scale
  l00 = np.sqrt(a00)
  l10, l20 = a01 / l00, a02 / l00
  d1 = a11 - l10 * l10
  if not d1 > 0.0:
    return np.zeros(3), d1 / scale
  l11 = np.sqrt(d1)
  l21 = (a12 - l20 * l10) / l11
  d2 = a22 - l20 * l20 - l21 * l21
  if not d2 > 0.0:
    return np.zeros(3), d2 / scale
  l22 = np.sqrt(d2)
  y0 = b[0] / l00
  y1 = (b[1] - l10 * y0) / l11
  y2 = (b[2] - l20 * y0 - l21 * y1) / l22
  g2 = y2 / l22
  g1 = (y1 - l21 * g2) / l11
  g0 = (y0 - l10 * g1 - l20 * g2) / l00
  return np.array([g0, g1, g2]), min(a00, d1, d2) / scale


def color_gradient(xyz, normals, inten, radius, max_nn=30):
  """-> (gradients float64 [n, 3], counts within the radius int [n], pivot ratio [n]: the smallest Cholesky pivot
  over the largest diagonal entry of the system, 0 where nn < 4)."""
  xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
  nrm = np.asarray(normals, np.float64).reshape(-1, 3)
  inten = np.asarray(inten, np.float64).reshape(-1)
  nbrs, counts = neighbours(xyz, radius, max_nn)
  grad = np.zeros((len(xyz), 3))
  pivot = np.zeros(len(xyz))
  for i, nb in enumerate(nbrs):
    nn = len(nb)
    if nn < 4:
      continue
    nb = nb[nb != i]
    n = nrm[i]
    e = xyz[nb] - xyz[i]
    u = e - (e @ n)[:, None] * n
    b = inten[nb] - inten[i]
    A = u.T @ u + float(nn - 1) ** 2 * np.outer(n, n)
    grad[i], pivot[i] = solve3(A, u.T @ b)
  return grad, counts, pivot


def colored_icp(src, src_intensity, tgt, tgt_normals, tgt_intensity, tgt_grad, max_dist, T_init=None,
                lambda_geometric=LAMBDA_GEOMETRIC, max_iter=30, rel_fitness=1e-6, rel_rmse=1e-6):
  """-> (4x4 pose, dict(fitness, inlier_rmse, iterations, n_corr, solves_failed))."""
  src, tgt = np.asarray(src, np.float64).reshape(-1, 3), np.asarray(tgt, np.float64).reshape(-1, 3)
  I_s = np.asarray(src_intensity, np.float64).reshape(-1)
  I_t = np.asarray(tgt_intensity, np.float64).reshape(-1)
  nrm = np.asarray(tgt_normals, np.float64).reshape(-1, 3)
  grd = np.asarray(tgt_grad, np.float64).reshape(-1, 3)
  sg, sp = np.sqrt(lambda_geometric), np.sqrt(1.0 - lambda_geometric)
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
    sm, q, nq, dq = s[m], tgt[j[m]], nrm[j[m]], grd[j[m]]
    rg = ((sm - q) * nq).sum(1)
    proj = sm - rg[:, None] * nq
    rp = I_s[m] - (((proj - q) * dq).sum(1) + I_t[j[m]])
    mv = (dq * nq).sum(1)[:, None] * nq - dq
    J = np.concatenate([sg * np.concatenate([np.cross(sm, nq), nq], axis=1),
                        sp * np.concatenate([np.cross(sm, mv), mv], axis=1)])
    r = np.concatenate([sg * rg, sp * rp])
    x = cholesky_step(J.T @ J, J.T @ r)
    if x is None:
      failed += 1
      x = np.zeros(6)
    T = zyx_update(x) @ T
    pf, pr = fit, rmse
    k += 1
  return T, dict(fitness=fit, inlier_rmse=rmse, iterations=k, n_corr=n, solves_failed=failed)
