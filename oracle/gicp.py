"""ORACLE (test infrastructure only) - generalized ICP and the robust losses: open3d >= 0.13's
``registration_generalized_icp(source, target, max_correspondence_distance, init,
TransformationEstimationForGeneralizedICP(epsilon, kernel), criteria)``, ``EstimatePerPointCovariances`` and the
robust kernels of open3d >= 0.12 (``L2Loss``, ``L1Loss``, ``HuberLoss``, ``CauchyLoss``, ``GMLoss``, ``TukeyLoss``)
on the point-to-plane, colored and generalized estimators; the GPU's dgr_estimate_covariances,
dgr_covariances_from_normals, dgr_generalized_icp, dgr_icp_loss and dgr_colored_icp_loss (csrc/icp.cu).

PARITY UNPINNED: open3d is not installable offline, so this restates its published code in float64 and pins the
conventions the GPU follows:

* loss weights, RobustKernel::Weight(r) at residual r and scale k: L2 1; L1 1 / |r|; Huber 1 for |r| <= k, else
  k / |r|; Cauchy 1 / (1 + (r / k)^2); GM k / (k + r^2)^2; Tukey (1 - min(1, |r| / k)^2)^2.  DEPARTURE: L1 at r = 0
  has weight 0 here; open3d's 1 / |r| is infinite there and turns the system into NaN;
* a weighted estimator adds w J J^T and w J r per row, each row weighted on its own residual.  Colored ICP has two
  rows, each weighted on its sqrt(lambda)-scaled residual (open3d >= 0.12's ColoredICP.cpp);
* covariances (EstimatePerPointCovariances with KDTreeSearchParamHybrid(radius, max_nn)): the neighbour sets of
  oracle/normals.py (strict radius, the max_nn smallest by (d^2, row), the point itself included), the population
  covariance C = E[e e^T] - mu mu^T over the offsets e = p_j - p_i; fewer than 3 neighbours give the identity;
* covariances from normals (InitializePointCloudForGeneralizedICP): C = R diag(epsilon, 1, 1) R^T with
  R = GetRotationFromE1ToX(n), read as the Rodrigues form I + [v]x + [v]x^2 / (1 + c), v = e1 x n, c = e1 . n, and a
  fixed diag(-1, -1, 1) when c < -0.99.  For a unit n with c >= -0.99 this is I - (1 - epsilon) n n^T; in the
  c < -0.99 branch C is diag(epsilon, 1, 1) whatever n is;
* precedence: a cloud's own covariances if it has them, else covariances from its normals; open3d estimates normals
  with KDTreeSearchParamKNN(20) when a cloud has neither, a search the voxel hash cannot run, so that is an error in
  the stand-in;
* generalized ICP, per correspondence of the current transformed source point s and its target point q:
  C_s' = R C_s R^T with R the rotation of the accumulated pose (open3d >= 0.13 transforms the covariances with the
  points), M = C_s' + C_t, W = M^(-1/2) (the principal root), three rows k = 0..2 with v = W[k]: r = v . (s - q),
  J = [s x v, v].  DEPARTURE: a correspondence whose M fails a 3x3 Cholesky (a non-positive pivot, in the GPU's
  order) adds no row; it still counts towards fitness and RMSE.  open3d would produce NaN there;
* correspondences, fitness, the Euclidean inlier RMSE, the Cholesky step (oracle/icp_plane.cholesky_step), the pose
  update and the stopping rule are oracle/icp_plane.py's: open3d's RegistrationICP uses them for every estimator.

``icp_point_to_plane`` and ``colored_icp`` here take ``kernel=None`` and are oracle/icp_plane.py's and
oracle/colored_icp.py's own functions when it is None.  A kernel is ``(name, k)`` with name in LOSSES.
"""
import numpy as np
from scipy.spatial import cKDTree

from . import colored_icp as _colored
from . import icp_plane as _plane
from .icp_plane import cholesky_step, zyx_update
from .normals import neighbours

LOSSES = ('L2', 'L1', 'Huber', 'Cauchy', 'GM', 'Tukey')        # index = the library's DGR_LOSS_* id
SCALED = ('Huber', 'Cauchy', 'GM', 'Tukey')                     # the losses that take k


def loss_weight(kernel, r):
  """RobustKernel::Weight of kernel = (name, k) (or None: 1) at residuals r (array)."""
  r = np.asarray(r, np.float64)
  if kernel is None:
    return np.ones_like(r)
  name, k = kernel[0], float(kernel[1])
  a = np.abs(r)
  if name == 'L2':
    return np.ones_like(r)
  if name == 'L1':
    with np.errstate(divide='ignore'):
      return np.where(a > 0.0, 1.0 / np.where(a > 0.0, a, 1.0), 0.0)
  if name == 'Huber':
    with np.errstate(divide='ignore'):
      return np.where(a <= k, 1.0, k / np.where(a > 0.0, a, 1.0))
  if name == 'Cauchy':
    return 1.0 / (1.0 + (r / k) ** 2)
  if name == 'GM':
    return k / (k + r * r) ** 2
  if name == 'Tukey':
    e = 1.0 - np.minimum(1.0, a / k) ** 2
    return e * e
  raise ValueError(f'unknown loss {name!r}')


def sym6(C):
  """[n, 3, 3] -> [n, 6] (xx, xy, xz, yy, yz, zz), the library's layout."""
  C = np.asarray(C, np.float64)
  return np.stack([C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]], axis=1)


def full33(c6):
  """[n, 6] (xx, xy, xz, yy, yz, zz) -> [n, 3, 3]."""
  c = np.asarray(c6, np.float64).reshape(-1, 6)
  return np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], axis=1)


def estimate_covariances(xyz, radius, max_nn):
  """-> (covariances float64 [n, 3, 3], counts within the radius int [n])."""
  xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
  nbrs, counts = neighbours(xyz, radius, max_nn)
  cov = np.tile(np.eye(3), (len(xyz), 1, 1))
  for i, nb in enumerate(nbrs):
    if len(nb) >= 3:
      e = xyz[nb] - xyz[i]
      mu = e.sum(0) / len(nb)
      cov[i] = (e.T @ e) / len(nb) - np.outer(mu, mu)
  return cov, counts


def rotation_e1_to_x(x):
  """open3d's GetRotationFromE1ToX as read here: I + [v]x + [v]x^2 / (1 + c), v = e1 x x, c = e1 . x; diag(-1, -1, 1)
  when c < -0.99."""
  x = np.asarray(x, np.float64)
  c = x[0]
  if c < -0.99:
    return np.diag([-1.0, -1.0, 1.0])
  v = np.cross([1.0, 0.0, 0.0], x)
  S = np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
  return np.eye(3) + S + (S @ S) / (1.0 + c)


def covariances_from_normals(normals, epsilon):
  """The literal R diag(epsilon, 1, 1) R^T per normal -> float64 [n, 3, 3]."""
  nrm = np.asarray(normals, np.float64).reshape(-1, 3)
  D = np.diag([float(epsilon), 1.0, 1.0])
  out = np.empty((len(nrm), 3, 3))
  for i, n in enumerate(nrm):
    R = rotation_e1_to_x(n)
    out[i] = R @ D @ R.T
  return out


def covariances_from_normals_closed(normals, epsilon):
  """I - (1 - epsilon) n n^T per normal: the literal form's value for a unit n with e1 . n >= -0.99."""
  nrm = np.asarray(normals, np.float64).reshape(-1, 3)
  return np.eye(3)[None] - (1.0 - float(epsilon)) * nrm[:, :, None] * nrm[:, None, :]


def _weighted_system(J, r, w):
  Jw = J * w[:, None]
  return Jw.T @ J, Jw.T @ r


def _icp_loop(src, tgt, max_dist, T_init, max_iter, rel_fitness, rel_rmse, system):
  """open3d's RegistrationICP loop (oracle/icp_plane.py's) with the estimator's (J^T J, J^T r) from
  system(s_m, source rows, target rows, T) -> (A, g, rows skipped)."""
  src, tgt = np.asarray(src, np.float64).reshape(-1, 3), np.asarray(tgt, np.float64).reshape(-1, 3)
  T = np.eye(4) if T_init is None else np.array(T_init, np.float64)
  tree = cKDTree(tgt) if len(tgt) else None
  failed = skipped = 0
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
    A, g, sk = system(s[m], np.nonzero(m)[0], j[m], T)
    skipped += sk
    x = cholesky_step(A, g)
    if x is None:
      failed += 1
      x = np.zeros(6)
    T = zyx_update(x) @ T
    pf, pr = fit, rmse
    k += 1
  return T, dict(fitness=fit, inlier_rmse=rmse, iterations=k, n_corr=n, solves_failed=failed, rows_skipped=skipped)


def icp_point_to_plane(src, tgt, tgt_normals, max_dist, T_init=None, kernel=None, max_iter=30, rel_fitness=1e-6,
                       rel_rmse=1e-6):
  """oracle/icp_plane.icp_point_to_plane, each row weighted by loss_weight(kernel, r)."""
  if kernel is None:
    return _plane.icp_point_to_plane(src, tgt, tgt_normals, max_dist, T_init, max_iter, rel_fitness, rel_rmse)
  tg = np.asarray(tgt, np.float64).reshape(-1, 3)
  nrm = np.asarray(tgt_normals, np.float64).reshape(-1, 3)

  def system(sm, _, jm, __):
    q, nq = tg[jm], nrm[jm]
    r = ((sm - q) * nq).sum(1)
    J = np.concatenate([np.cross(sm, nq), nq], axis=1)
    return (*_weighted_system(J, r, loss_weight(kernel, r)), 0)

  return _icp_loop(src, tgt, max_dist, T_init, max_iter, rel_fitness, rel_rmse, system)


def colored_icp(src, src_intensity, tgt, tgt_normals, tgt_intensity, tgt_grad, max_dist, T_init=None,
                lambda_geometric=_colored.LAMBDA_GEOMETRIC, kernel=None, max_iter=30, rel_fitness=1e-6,
                rel_rmse=1e-6):
  """oracle/colored_icp.colored_icp, each of the two rows weighted on its own scaled residual."""
  if kernel is None:
    return _colored.colored_icp(src, src_intensity, tgt, tgt_normals, tgt_intensity, tgt_grad, max_dist, T_init,
                                lambda_geometric, max_iter, rel_fitness, rel_rmse)
  tg = np.asarray(tgt, np.float64).reshape(-1, 3)
  I_s = np.asarray(src_intensity, np.float64).reshape(-1)
  I_t = np.asarray(tgt_intensity, np.float64).reshape(-1)
  nrm = np.asarray(tgt_normals, np.float64).reshape(-1, 3)
  grd = np.asarray(tgt_grad, np.float64).reshape(-1, 3)
  sg, sp = np.sqrt(lambda_geometric), np.sqrt(1.0 - lambda_geometric)

  def system(sm, im, jm, _):
    q, nq, dq = tg[jm], nrm[jm], grd[jm]
    rg = ((sm - q) * nq).sum(1)
    proj = sm - rg[:, None] * nq
    rp = I_s[im] - (((proj - q) * dq).sum(1) + I_t[jm])
    mv = (dq * nq).sum(1)[:, None] * nq - dq
    J = np.concatenate([sg * np.concatenate([np.cross(sm, nq), nq], axis=1),
                        sp * np.concatenate([np.cross(sm, mv), mv], axis=1)])
    r = np.concatenate([sg * rg, sp * rp])
    return (*_weighted_system(J, r, loss_weight(kernel, r)), 0)

  return _icp_loop(src, tgt, max_dist, T_init, max_iter, rel_fitness, rel_rmse, system)


def cholesky3_ok(M):
  """[n] bool: every pivot of the 3x3 Cholesky of M [n, 3, 3] is positive (the GPU's order)."""
  d0 = M[:, 0, 0]
  with np.errstate(invalid='ignore', divide='ignore'):
    l10, l20 = M[:, 1, 0] / np.sqrt(d0), M[:, 2, 0] / np.sqrt(d0)
    d1 = M[:, 1, 1] - l10 * l10
    l21 = (M[:, 2, 1] - l20 * l10) / np.sqrt(d1)
    d2 = M[:, 2, 2] - l20 * l20 - l21 * l21
  return (d0 > 0.0) & (d1 > 0.0) & (d2 > 0.0)


def inverse_sqrt(M):
  """The principal M^(-1/2) of symmetric positive-definite M [n, 3, 3]."""
  w, V = np.linalg.eigh(M)
  return np.einsum('nij,nj,nkj->nik', V, 1.0 / np.sqrt(w), V)


def generalized_icp(src, src_cov, tgt, tgt_cov, max_dist, T_init=None, kernel=None, max_iter=30, rel_fitness=1e-6,
                    rel_rmse=1e-6):
  """Generalized ICP of src onto tgt with their covariances ([n, 3, 3] or [n, 6]).  -> (4x4 pose, dict(fitness,
  inlier_rmse, iterations, n_corr, solves_failed, rows_skipped)); rows_skipped counts the correspondences (over all
  updates) whose M failed the Cholesky test."""
  Cs_all = np.asarray(src_cov, np.float64)
  Ct_all = np.asarray(tgt_cov, np.float64)
  Cs_all = full33(Cs_all) if Cs_all.shape[-1] == 6 else Cs_all.reshape(-1, 3, 3)
  Ct_all = full33(Ct_all) if Ct_all.shape[-1] == 6 else Ct_all.reshape(-1, 3, 3)
  tg = np.asarray(tgt, np.float64).reshape(-1, 3)

  def system(sm, im, jm, T):
    R = T[:3, :3]
    M = np.einsum('ab,nbc,dc->nad', R, Cs_all[im], R) + Ct_all[jm]
    ok = cholesky3_ok(M)
    sm, q, M = sm[ok], tg[jm][ok], M[ok]
    W = inverse_sqrt(M) if len(M) else np.zeros((0, 3, 3))
    e = sm - q
    J = np.concatenate([np.concatenate([np.cross(sm, W[:, k]), W[:, k]], axis=1) for k in range(3)])
    r = np.concatenate([(W[:, k] * e).sum(1) for k in range(3)])
    return (*_weighted_system(J, r, loss_weight(kernel, r)), int((~ok).sum()))

  return _icp_loop(src, tgt, max_dist, T_init, max_iter, rel_fitness, rel_rmse, system)
