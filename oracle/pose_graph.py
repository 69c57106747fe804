"""ORACLE (test infrastructure only) - multiway registration as open3d runs it:
``pipelines.registration.get_information_matrix_from_point_clouds`` and ``global_optimization`` with
``GlobalOptimizationLevenbergMarquardt`` (Choi, Zhou & Koltun, *Robust reconstruction of indoor scenes*, CVPR 2015,
§4-5), restated in float64 numpy.

PARITY UNPINNED: open3d is not installed here and not vendored, so every reading below is a restatement from memory of
open3d's published GlobalOptimization.cpp / Registration.cpp, recorded as an assumption:

Information matrix.  Each source point s is moved by T; its nearest target point q strictly within
max_correspondence_distance (squared distance < radius^2, the lower target row on a tie - the rule of oracle/icp.py's
search as dgr_icp applies it) contributes G^T G with G = [[0, z, -y, 1, 0, 0], [-z, 0, x, 0, 1, 0], [y, -x, 0, 0, 0,
1]], q = (x, y, z) in target coordinates (rotation first).  So Lambda[5, 5] is the correspondence count.  This module
sums the explicit three-row G products; the kernel uses the closed form of the ten sums, so the two check each other.

Pose graph.  Node k has pose P_k (fragment k into the world).  Edge e = (s, t, X_e, Lambda_e, uncertain_e) has residual
r_e = v(X_e^-1 P_t^-1 P_s), v(A) = (1/2 (A21 - A12), 1/2 (A02 - A20), 1/2 (A10 - A01), A03, A13, A23).  Its Jacobian
with respect to a left update P_s <- Exp(d) P_s is J_s[:, i] = v(X^-1 P_t^-1 G_i P_s) (G_i the generators of
Exp(d) = [Rz(d2) Ry(d1) Rx(d0) | d3..5] at 0, open3d's TransformVector6dToMatrix4d), and J_t = -J_s.
  * objective E = sum_certain r^T Lambda r + sum_uncertain [l r^T Lambda r + mu (sqrt(l) - 1)^2];
  * line process l = (mu / (mu + r^T Lambda r))^2 on uncertain edges (0 / 0 reads as 1), 1 on certain ones;
  * mu = preference_loop_closure * max_correspondence_distance^2 * mean(Lambda_e[5, 5]) over the edges of the pass
    (0 without edges);
  * normal equations H = sum l J^T Lambda J, b = -sum l J^T Lambda r; step delta = (H + lambda I)^-1 b, poses
    P_k <- Exp(delta_k) P_k;
  * LM schedule: the cost of a pass starts with the line process each edge carries in (an uncertain edge's
    confidence in the first pass - open3d's default confidence 1.0 is its line process initialisation - and its
    first-pass l in the second); l is then recomputed at every accepted state; a trial cost uses the l of the current
    state.  lambda_0 = 1e-5 max diag(H), ni = 2.  Per outer iteration, up to max_iteration_lm trials: stop when
    |delta| < min_relative_increment (|x| + min_relative_increment) (x = every pose as ZYX Euler angles and
    translation, open3d's TransformMatrix4dToVector6d); rho = (E - E_new) / (delta . (lambda delta + b) + 1e-3); on
    rho > 0 accept, stop when |E - E_new| < min_relative_residual_increment E, lambda *= max(lower_scale_factor,
    min(1 - (2 rho - 1)^3, upper_scale_factor)), ni = 2, rebuild l, H, b and stop when max|b| < min_right_term; on
    rho <= 0 lambda *= ni, ni *= 2.  After the trials stop when E < min_residual.  max|b| < min_right_term before the
    first iteration ends the pass at once.  open3d's right-term test reads max(b); this reads max|b|;
  * GlobalOptimization: a pass over every edge, the uncertain edges with l < edge_prune_threshold removed, a pass over
    the rest from the first pass's poses (mu recomputed over the kept edges), then with reference_node >= 0 every pose
    P_k <- P0_ref P_ref^-1 P_k and the reference node set to its input pose exactly;
  * a factorisation that meets a pivot that is not positive ends the optimisation with status 1, the poses those of
    the last accepted step;
  * defaults (open3d's, as remembered): GlobalOptimizationOption(max_correspondence_distance=0.075,
    edge_prune_threshold=0.25, preference_loop_closure=1.0, reference_node=-1) - -1 means no compensation;
    GlobalOptimizationConvergenceCriteria(max_iteration=100, min_relative_increment=1e-6,
    min_relative_residual_increment=1e-6, min_right_term=1e-6, min_residual=1e-6, max_iteration_lm=20,
    upper_scale_factor=2/3, lower_scale_factor=1/3).
"""
import math

import numpy as np
from scipy.spatial import cKDTree

OPTION_DEFAULTS = dict(max_correspondence_distance=0.075, edge_prune_threshold=0.25, preference_loop_closure=1.0,
                       reference_node=-1)
CRITERIA_DEFAULTS = dict(max_iteration=100, min_relative_increment=1e-6, min_relative_residual_increment=1e-6,
                         min_right_term=1e-6, min_residual=1e-6, max_iteration_lm=20, upper_scale_factor=2 / 3,
                         lower_scale_factor=1 / 3)


# --------------------------------------------------------------------------- #
# information matrix
# --------------------------------------------------------------------------- #
def nearest_within(p, tgt, max_dist, k=8):
  """Row of the nearest target point strictly within max_dist of every row of p (lower row on a tie), -1 when none;
  squared distances in float64."""
  tgt = np.asarray(tgt, np.float64)
  if len(tgt) == 0 or len(p) == 0:
    return np.full(len(p), -1, np.int64)
  k = min(k, len(tgt))
  _, idx = cKDTree(tgt).query(p, k=k, distance_upper_bound=max_dist * (1 + 1e-9))
  idx = np.asarray(idx).reshape(len(p), k)
  valid = idx < len(tgt)
  safe = np.where(valid, idx, 0)
  d2 = ((p[:, None, :] - tgt[safe]) ** 2).sum(-1)
  d2 = np.where(valid & (d2 < max_dist * max_dist), d2, np.inf)
  key = np.lexsort((np.where(np.isfinite(d2), safe, np.iinfo(np.int64).max), d2), axis=-1)[:, 0]
  best = safe[np.arange(len(p)), key]
  return np.where(np.isfinite(d2[np.arange(len(p)), key]), best, -1)


def correspondences(src, tgt, T, max_dist):
  """Target points q matched by T s (float32 clouds read in float64, as the kernel reads them)."""
  src = np.asarray(src, np.float32).astype(np.float64).reshape(-1, 3)
  tgt = np.asarray(tgt, np.float32).astype(np.float64).reshape(-1, 3)
  T = np.asarray(T, np.float64).reshape(4, 4)
  p = src @ T[:3, :3].T + T[:3, 3]
  j = nearest_within(p, tgt, max_dist)
  return tgt[j[j >= 0]]


def g_rows(q):
  """[n, 3, 6] the three G-rows of every target point."""
  x, y, z = q[:, 0], q[:, 1], q[:, 2]
  o, l = np.zeros_like(x), np.ones_like(x)
  return np.stack([np.stack([o, z, -y, l, o, o], -1), np.stack([-z, o, x, o, l, o], -1),
                   np.stack([y, -x, o, o, o, l], -1)], 1)


def information_matrix(src, tgt, T, max_dist):
  """(Lambda [6, 6], count) from the explicit sum of G^T G."""
  q = correspondences(src, tgt, T, max_dist)
  G = g_rows(q)
  return np.einsum('nri,nrj->ij', G, G), len(q)


def information_closed_form(q):
  """Lambda from the ten sums of the matched target points q: [[tr(Q) I - Q, [S]x], [[S]x^T, n I]]."""
  q = np.asarray(q, np.float64).reshape(-1, 3)
  S, Q = q.sum(0), q.T @ q
  Sx = np.array([[0, -S[2], S[1]], [S[2], 0, -S[0]], [-S[1], S[0], 0]])
  L = np.zeros((6, 6))
  L[:3, :3] = np.trace(Q) * np.eye(3) - Q
  L[:3, 3:] = Sx
  L[3:, :3] = Sx.T
  L[3:, 3:] = len(q) * np.eye(3)
  return L


# --------------------------------------------------------------------------- #
# pose graph
# --------------------------------------------------------------------------- #
def vec6(A):
  return np.array([0.5 * (A[2, 1] - A[1, 2]), 0.5 * (A[0, 2] - A[2, 0]), 0.5 * (A[1, 0] - A[0, 1]),
                   A[0, 3], A[1, 3], A[2, 3]])


def exp6(x):
  """open3d's TransformVector6dToMatrix4d: [Rz(x2) Ry(x1) Rx(x0) | x3..5]."""
  ca, sa, cb, sb, cc, sc = math.cos(x[0]), math.sin(x[0]), math.cos(x[1]), math.sin(x[1]), math.cos(x[2]), \
      math.sin(x[2])
  Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1.0]])
  Ry = np.array([[cb, 0, sb], [0, 1.0, 0], [-sb, 0, cb]])
  Rx = np.array([[1.0, 0, 0], [0, ca, -sa], [0, sa, ca]])
  T = np.eye(4)
  T[:3, :3] = Rz @ Ry @ Rx
  T[:3, 3] = x[3:6]
  return T


def pose_vector(T):
  """open3d's TransformMatrix4dToVector6d: ZYX Euler angles, then the translation."""
  R = T[:3, :3]
  sy = math.sqrt(R[0, 0] ** 2 + R[1, 0] ** 2)
  if not sy < 1e-6:
    a, b, c = math.atan2(R[2, 1], R[2, 2]), math.atan2(-R[2, 0], sy), math.atan2(R[1, 0], R[0, 0])
  else:
    a, b, c = math.atan2(-R[1, 2], R[1, 1]), math.atan2(-R[2, 0], sy), 0.0
  return np.array([a, b, c, T[0, 3], T[1, 3], T[2, 3]])


def inv(T):
  out = np.eye(4)
  out[:3, :3] = T[:3, :3].T
  out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
  return out


GENERATORS = []
for _i in range(6):
  _G = np.zeros((4, 4))
  if _i < 3:
    _a, _b = (_i + 1) % 3, (_i + 2) % 3
    _G[_b, _a], _G[_a, _b] = 1.0, -1.0
  else:
    _G[_i - 3, 3] = 1.0
  GENERATORS.append(_G)


def residual(P, ends, Xinv, e):
  s, t = ends[e]
  return vec6(Xinv[e] @ inv(P[t]) @ P[s])


def jacobian_source(P, ends, Xinv, e):
  s, t = ends[e]
  M = Xinv[e] @ inv(P[t])
  return np.stack([vec6(M @ G @ P[s]) for G in GENERATORS], 1)


def line_process(mu, q):
  d = mu + q
  return 1.0 if d == 0.0 else (mu / d) ** 2


def edge_cost(q, l, mu, uncertain):
  return l * q + mu * (math.sqrt(l) - 1.0) ** 2 if uncertain else q


def _pass(P, ends, Xinv, info, unc, l, act, o, c):
  """One LM pass over the active edges; P, l updated in place.  -> stats dict."""
  N = len(P)
  idx = np.flatnonzero(act)
  mu = o['preference_loop_closure'] * o['max_correspondence_distance'] ** 2 * (
      float(np.mean(info[idx, 5, 5])) if len(idx) else 0.0)

  def residuals(Q):
    return {e: residual(Q, ends, Xinv, e) for e in idx}

  def cost(r):
    return float(sum(edge_cost(float(r[e] @ info[e] @ r[e]), l[e], mu, unc[e]) for e in idx))

  def system(r):
    H, b = np.zeros((6 * N, 6 * N)), np.zeros(6 * N)
    for e in idx:
      q = float(r[e] @ info[e] @ r[e])
      l[e] = line_process(mu, q) if unc[e] else 1.0
      J = jacobian_source(P, ends, Xinv, e)
      A = l[e] * J.T @ info[e] @ J
      g = l[e] * J.T @ info[e] @ r[e]
      s, t = ends[e]
      H[6 * s:6 * s + 6, 6 * s:6 * s + 6] += A
      H[6 * t:6 * t + 6, 6 * t:6 * t + 6] += A
      H[6 * s:6 * s + 6, 6 * t:6 * t + 6] -= A
      H[6 * t:6 * t + 6, 6 * s:6 * s + 6] -= A
      b[6 * s:6 * s + 6] -= g
      b[6 * t:6 * t + 6] += g
    return H, b

  r = residuals(P)
  E = cost(r)
  out = dict(mu=mu, cost0=E, iterations=0, failed=0, factorisations=0)
  H, b = system(r)
  lam, ni = 1e-5 * (float(np.max(np.diag(H))) if N else 0.0), 2.0
  stop = float(np.max(np.abs(b))) < c['min_right_term']
  for it in range(c['max_iteration']):
    if stop:
      break
    out['iterations'] = it + 1
    lm, rho = 0, 0.0
    while True:
      out['factorisations'] += 1
      try:
        Lc = np.linalg.cholesky(H + lam * np.eye(6 * N))
      except np.linalg.LinAlgError:
        out['failed'], stop = 1, True
        break
      delta = np.linalg.solve(Lc.T, np.linalg.solve(Lc, b))
      xn = math.sqrt(sum(float(pose_vector(T) @ pose_vector(T)) for T in P))
      if np.linalg.norm(delta) < c['min_relative_increment'] * (xn + c['min_relative_increment']):
        stop = True
      if not stop:
        Pn = np.stack([exp6(delta[6 * k:6 * k + 6]) @ P[k] for k in range(N)])
        rn = residuals(Pn)
        En = cost(rn)
        rho = (E - En) / (float(delta @ (lam * delta + b)) + 1e-3)
        if rho > 0:
          if abs(E - En) < c['min_relative_residual_increment'] * E:
            stop = True
          alpha = min(1.0 - (2.0 * rho - 1.0) ** 3, c['upper_scale_factor'])
          lam *= max(c['lower_scale_factor'], alpha)
          ni = 2.0
          E = En
          P[:] = Pn
          r = rn
          H, b = system(r)
          if float(np.max(np.abs(b))) < c['min_right_term']:
            stop = True
          if stop:
            break
        else:
          lam *= ni
          ni *= 2.0
      lm += 1
      if lm >= c['max_iteration_lm']:
        stop = True
      if rho > 0 or stop:
        break
    if E < c['min_residual']:
      stop = True
  out['cost'] = E
  return out


def global_optimization(poses, ends, T, info, uncertain, confidence=None, option=None, criteria=None):
  """-> (poses [N, 4, 4], kept [E] bool, l [E], stats) as dgr_pose_graph_optimize returns them."""
  o = dict(OPTION_DEFAULTS, **(option or {}))
  c = dict(CRITERIA_DEFAULTS, **(criteria or {}))
  P0 = np.asarray(poses, np.float64).reshape(-1, 4, 4).copy()
  P = P0.copy()
  ends = np.asarray(ends, np.int64).reshape(-1, 2)
  E = len(ends)
  X = np.asarray(T, np.float64).reshape(E, 4, 4)
  Xinv = np.stack([inv(x) for x in X]) if E else np.zeros((0, 4, 4))
  info = np.asarray(info, np.float64).reshape(E, 6, 6)
  unc = np.asarray(uncertain, bool).reshape(E)
  conf = np.ones(E) if confidence is None else np.asarray(confidence, np.float64).reshape(E)
  l = np.where(unc, conf, 1.0)
  act = np.ones(E, bool)
  p1 = _pass(P, ends, Xinv, info, unc, l, act, o, c)
  pruned = 0
  p2 = dict(mu=0.0, iterations=0, failed=0, factorisations=0, cost=p1['cost'])
  if not p1['failed']:
    drop = unc & ~(l >= o['edge_prune_threshold'])
    act &= ~drop
    pruned = int(drop.sum())
    p2 = _pass(P, ends, Xinv, info, unc, l, act, o, c)
  ref = o['reference_node']
  if ref >= 0:
    C = P0[ref] @ inv(P[ref])
    P = np.stack([P0[k] if k == ref else C @ P[k] for k in range(len(P))])
  stats = dict(iterations=p1['iterations'], iterations_pruned=p2['iterations'], cost=p2['cost'], pruned=pruned,
               status=int(p1['failed'] or p2['failed']), mu=p1['mu'], mu_pruned=p2['mu'], cost_start=p1['cost0'],
               cost_first_pass=p1['cost'], factorisations=p1['factorisations'] + p2['factorisations'])
  return P, act.copy(), l, stats
