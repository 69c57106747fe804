"""ORACLE (test infrastructure only) - fp64 yardsticks for the pose solvers: weighted Procrustes and the robust SE(3)
refinement of `dgr_se3_register` (csrc/registration.cu), and the 3x3 Kabsch / 6x6 Cholesky steps of csrc/kabsch.cuh
that ICP, RANSAC, FGR, Go-ICP, Super4PCS and PointNetLK share.

Every reference is computed from the float32 rows actually handed to the kernel, never from the model that generated
them.  The acceptance criterion has the form of oracle/precision.py:

    e(kernel) <= KAPPA * max(e(fp32 oracle), floor)

with e32 the error of an honest fp32 computation of the same thing (oracle.registration) against the fp64 reference.

Unique minimiser (`floor` <= UNIQUE_FLOOR): e = max(|R - R64|_max, |t - t64| / (|t64| + spread)).  The floor is the
first-order sensitivity of the Kabsch rotation to rounding S = sum wn (y - my)(x - mx)^T to float32:

    floor = 2^-24 |S|_2 / min_{i<j} (s~i + s~j),     s~ = (s1, s2, sign(det U det V) s3)

(a perturbation of S turns R about the axis of the pair (i, j) by its antisymmetric part over s~i + s~j).  The
translation t = my - R mx adds |dR| |mx| and the rounding of the centroids, both relative to |t64| + spread.

Non-unique minimiser (rank <= 1, or s~2 + s~3 = 0 for a reflection with s2 = s3): R itself is not compared.  The
objective f(R) = tr(R^T S) must be within KAPPA * max(e32_f, F_FLOOR) of its optimum s1 + s2 + s~3 (relative to s1),
with |R^T R - I|_max <= 4 * 2^-24 and det R = +1.
"""
import math
from fractions import Fraction

import numpy as np
import torch

from . import registration as oreg

KAPPA = 8.0
U32 = 2.0 ** -24
U64 = 2.0 ** -53
UNIQUE_FLOOR = 1e-4          # above this the rotation is too ill-posed to compare entrywise: objective criterion
F_FLOOR = 6 * U32            # |opt - f(R)| / s1 for R optimal to a float32 rounding of S (2 |dS|_nuclear <= 6 u s1)
ORTHO_TOL = 4 * U32
F32_EPS = oreg.F32_EPS


def _f64(a):
  if isinstance(a, torch.Tensor):
    a = a.detach().cpu().numpy()
  return np.asarray(a, np.float64)


def _rows32(a):
  """The float32 values of a, as float64 (what a kernel reads from a float32 tensor)."""
  if isinstance(a, torch.Tensor):
    a = a.detach().cpu().numpy()
  return np.asarray(a, np.float32).astype(np.float64)


# --------------------------------------------------------------------------- #
# Kabsch from a cross-covariance
# --------------------------------------------------------------------------- #
def kabsch64(S):
  """-> (R, sig, s): the Kabsch rotation U diag(1, 1, s) V^T of S = U diag(sig) V^T, s = sign(det U det V)."""
  S = _f64(S)
  U, sig, Vt = np.linalg.svd(S)
  s = -1.0 if np.linalg.det(U) * np.linalg.det(Vt) < 0 else 1.0
  return U @ np.diag([1.0, 1.0, s]) @ Vt, sig, s


def sensitivity_floor(S):
  """2^-24 |S|_2 / min_{i<j} (s~i + s~j): the rotation error that rounding S to float32 alone may cause (inf when the
  minimiser is not unique)."""
  _, sig, s = kabsch64(S)
  st = np.array([sig[0], sig[1], s * sig[2]])
  den = min(st[0] + st[1], st[0] + st[2], st[1] + st[2])
  if sig[0] == 0.0:
    return math.inf
  return U32 * sig[0] / den if den > 0 else math.inf


def objective(R, S):
  """f(R) = tr(R^T S)."""
  return float(np.trace(_f64(R).T @ _f64(S)))


# --------------------------------------------------------------------------- #
# numpy restatement of csrc/kabsch.cuh (jacobi_svd3 + kabsch_rotation)
# --------------------------------------------------------------------------- #
def jacobi_svd3(S, max_sweeps=60):
  """One-sided Jacobi on S in kabsch.cuh's sweep order and skip rule -> (A = S V, V, sig unsorted)."""
  A = [[float(S[i][j]) for j in range(3)] for i in range(3)]
  V = [[1.0 if i == j else 0.0 for j in range(3)] for i in range(3)]
  for _ in range(max_sweeps):
    rotated = False
    for p in range(2):
      for q in range(p + 1, 3):
        alpha = sum(A[k][p] * A[k][p] for k in range(3))
        beta = sum(A[k][q] * A[k][q] for k in range(3))
        gamma = sum(A[k][p] * A[k][q] for k in range(3))
        if abs(gamma) <= 1e-300 or abs(gamma) <= 1e-17 * math.sqrt(alpha * beta):
          continue
        rotated = True
        zeta = (beta - alpha) / (2.0 * gamma)
        t = (1.0 if zeta >= 0 else -1.0) / (abs(zeta) + math.sqrt(1.0 + zeta * zeta))
        c = 1.0 / math.sqrt(1.0 + t * t)
        s = c * t
        for k in range(3):
          ap, aq = A[k][p], A[k][q]
          A[k][p], A[k][q] = c * ap - s * aq, s * ap + c * aq
          vp, vq = V[k][p], V[k][q]
          V[k][p], V[k][q] = c * vp - s * vq, s * vp + c * vq
    if not rotated:
      break
  sig = [math.sqrt(A[0][j] ** 2 + A[1][j] ** 2 + A[2][j] ** 2) for j in range(3)]
  return np.array(A), np.array(V), np.array(sig)


def kabsch_rotation(S, max_sweeps=60):
  """kabsch.cuh's kabsch_rotation: descending order, the identity for a zero S, rank <= 1 / <= 2 completion, the
  det(U) det(W) fix."""
  A, V, sig = jacobi_svd3(S, max_sweeps)
  ord_ = [0, 1, 2]
  for a in range(2):
    for b in range(a + 1, 3):
      if sig[ord_[b]] > sig[ord_[a]]:
        ord_[a], ord_[b] = ord_[b], ord_[a]
  if sig[ord_[0]] <= 1e-300:
    return np.eye(3)
  tiny = 1e-300 + 1e-14 * sig[ord_[0]]
  U = np.zeros((3, 3))
  W = np.zeros((3, 3))
  for j in range(3):
    o = ord_[j]
    W[:, j] = V[:, o]
    U[:, j] = A[:, o] / sig[o] if sig[o] > tiny else 0.0
  if sig[ord_[1]] <= tiny:
    ax, ay, az = np.abs(U[:, 0])
    e = np.zeros(3)
    e[0 if (ax <= ay and ax <= az) else (1 if ay <= az else 2)] = 1.0
    v = e - (e @ U[:, 0]) * U[:, 0]
    nv = np.linalg.norm(v)
    if nv < 1e-300:
      v, nv = np.array([1.0, 0.0, 0.0]), 1.0
    U[:, 1] = v / nv
  if sig[ord_[2]] <= tiny:
    U[:, 2] = np.cross(U[:, 0], U[:, 1])
  sgn = -1.0 if np.linalg.det(U) * np.linalg.det(W) < 0 else 1.0
  return U[:, :2] @ W[:, :2].T + sgn * np.outer(U[:, 2], W[:, 2])


# --------------------------------------------------------------------------- #
# weighted Procrustes
# --------------------------------------------------------------------------- #
def _moments32(X, Y, w, eps=F32_EPS):
  """The fp32 centroids and S of oracle.registration.weighted_procrustes (torch fp32 on the CPU)."""
  X, Y, w = (torch.as_tensor(np.asarray(a, np.float32)) for a in (X, Y, w))
  w = w.reshape(-1, 1)
  wn = w / (w.abs().sum() + eps)
  mx = (wn * X).sum(0)
  my = (wn * Y).sum(0)
  S = (Y - my).t() @ (wn * (X - mx))
  return mx.double().numpy(), my.double().numpy(), S.double().numpy()


def procrustes64(X, Y, w, eps=F32_EPS):
  """fp64 weighted Procrustes of the float32 rows X, Y [n, 3] and weights w [n] (the reference's normalisation
  wn = w / (sum |w| + eps)).  -> dict(R, t, S, sig, s, opt, floor, spread, mx, my)."""
  X, Y, w = _rows32(X), _rows32(Y), _rows32(w).reshape(-1)
  wn = w / (np.abs(w).sum() + eps)
  mx, my = wn @ X, wn @ Y
  S = (Y - my).T @ (wn[:, None] * (X - mx))
  R, sig, s = kabsch64(S)
  t = my - R @ mx
  spread = float(np.sqrt(np.abs(wn) @ ((X - mx) ** 2).sum(1))) if len(X) else 0.0
  return dict(R=R, t=t, S=S, sig=sig, s=s, opt=float(sig[0] + sig[1] + s * sig[2]), floor=sensitivity_floor(S),
              spread=spread, mx=mx, my=my)


def pose_floor(ref):
  """The criterion's floor for (R, t): the rotation floor, and its effect on t = my - R mx plus the float32
  rounding of the centroids, relative to |t64| + spread."""
  f = ref['floor']
  den = np.linalg.norm(ref['t']) + ref['spread'] + 1e-300
  ft = (f * np.linalg.norm(ref['mx']) + U32 * (np.linalg.norm(ref['mx']) + np.linalg.norm(ref['my']))) / den
  return max(f, ft)


def pose_err(R, t, ref):
  """max(|R - R64|_max, |t - t64| / (|t64| + spread))."""
  er = float(np.abs(_f64(R) - ref['R']).max())
  et = float(np.linalg.norm(_f64(t).reshape(3) - ref['t']) / (np.linalg.norm(ref['t']) + ref['spread'] + 1e-300))
  return max(er, et)


def objective_err(R, ref):
  """(opt - f(R)) / s1 against the fp64 S (0 for a zero S)."""
  s1 = ref['sig'][0]
  return abs(ref['opt'] - objective(R, ref['S'])) / s1 if s1 > 0 else 0.0


def is_rotation(R, tol=ORTHO_TOL):
  R = _f64(R)
  return bool(np.abs(R.T @ R - np.eye(3)).max() <= tol and abs(np.linalg.det(R) - 1.0) <= tol)


def check(R, t, R32, t32, ref, kappa=KAPPA):
  """Apply the criterion to a result (R, t) next to the fp32 oracle's (R32, t32).  -> dict(ok, unique, e, e32, bound,
  ratio) where ratio = e / max(e32, floor) is the quantity KAPPA bounds."""
  unique = ref['floor'] <= UNIQUE_FLOOR
  if unique:
    e, e32, fl = pose_err(R, t, ref), pose_err(R32, t32, ref), pose_floor(ref)
  else:
    e, e32, fl = objective_err(R, ref), objective_err(R32, ref), F_FLOOR
  bound = kappa * max(e32, fl)
  ok = bool(e <= bound) and is_rotation(R)
  return dict(ok=ok, unique=unique, e=e, e32=e32, bound=bound, ratio=e / max(e32, fl))


def oracle32(X, Y, w, eps=F32_EPS):
  """The honest fp32 oracle (oracle.registration.weighted_procrustes) as float64 arrays; eps = 0 for plain
  unweighted pairs (ICP)."""
  R, t = oreg.weighted_procrustes(np.asarray(X, np.float32), np.asarray(Y, np.float32),
                                  np.asarray(w, np.float32).reshape(-1, 1), eps=eps)
  return R.double().numpy(), t.double().numpy()


def restated(X, Y, w, max_sweeps=60, round_S=None):
  """kabsch.cuh as restated above on fp32 moments (the kernel's arithmetic up to summation order).  round_S: a
  function applied to S first (the negative controls)."""
  mx, my, S = _moments32(X, Y, w)
  if round_S is not None:
    S = round_S(S)
  R = kabsch_rotation(S, max_sweeps)
  R = R.astype(np.float32).astype(np.float64)
  t = (my.astype(np.float32) - (R.astype(np.float32) @ mx.astype(np.float32))).astype(np.float64)
  return R, t


def bf16_round(a):
  """Round to bfloat16 (8 significant bits), nearest even."""
  return torch.as_tensor(np.asarray(a, np.float32)).bfloat16().double().numpy()


# --------------------------------------------------------------------------- #
# the refinement
# --------------------------------------------------------------------------- #
def refine64(X, Y, w, q, k, lr=0.1, gamma=0.999):
  """oracle.se3_refine's Adam loop in fp64 for exactly k steps (no break rule) from the fp64 Procrustes pose.
  -> (R, t, loss) with loss evaluated at the pose of step k - 1, as the kernel and the reference report it."""
  X, Y, w = (torch.from_numpy(_rows32(a)) for a in (X, Y, w))
  w = w.reshape(-1, 1)
  p = procrustes64(X.numpy(), Y.numpy(), w.numpy())
  R0 = torch.from_numpy(p['R'])
  rot6d = torch.cat([R0[:, 0], R0[:, 1]]).clone().requires_grad_(True)
  trans = torch.from_numpy(p['t']).reshape(1, 3).clone().requires_grad_(True)
  opt = torch.optim.Adam([rot6d, trans], lr=lr)
  loss_val = float('nan')
  for _ in range(k):
    loss = oreg.robust_loss(X @ oreg.rot6d_to_matrix(rot6d).t() + trans, Y, w, q)
    loss_val = loss.item()
    opt.zero_grad()
    loss.backward()
    opt.step()
    for g in opt.param_groups:
      g['lr'] *= gamma
  with torch.no_grad():
    R = oreg.rot6d_to_matrix(rot6d.detach())
  return R.numpy(), trans.detach().numpy().reshape(3), loss_val


# --------------------------------------------------------------------------- #
# ICP steps on known pairs
# --------------------------------------------------------------------------- #
def kabsch_pairs64(P, Q):
  """Two-pass centred fp64 Kabsch of the pairs (P[i], Q[i]) (Q ~ R P + t).  -> dict as procrustes64 (unit weights,
  no eps)."""
  P, Q = _f64(P), _f64(Q)
  mp, mq = P.mean(0), Q.mean(0)
  S = (Q - mq).T @ (P - mp) / len(P)
  R, sig, s = kabsch64(S)
  spread = float(np.sqrt(((P - mp) ** 2).sum(1).mean()))
  return dict(R=R, t=mq - R @ mp, S=S, sig=sig, s=s, opt=float(sig[0] + sig[1] + s * sig[2]),
              floor=sensitivity_floor(S), spread=spread, mx=mp, my=mq)


def plane_system(P, Q, N):
  """Exact (Fraction) J^T J [6, 6] and J^T r [6] of point-to-plane rows r = (p - q).n, J = [p x n, n] over fp64
  inputs, as open3d and icp.cu define them."""
  P, Q, N = _f64(P), _f64(Q), _f64(N)
  A = [[Fraction(0)] * 6 for _ in range(6)]
  g = [Fraction(0)] * 6
  for p, q, n in zip(P, Q, N):
    p, q, n = [Fraction(float(v)) for v in p], [Fraction(float(v)) for v in q], [Fraction(float(v)) for v in n]
    r = sum((p[a] - q[a]) * n[a] for a in range(3))
    J = [p[1] * n[2] - p[2] * n[1], p[2] * n[0] - p[0] * n[2], p[0] * n[1] - p[1] * n[0], n[0], n[1], n[2]]
    for a in range(6):
      g[a] += J[a] * r
      for b in range(a, 6):
        A[a][b] += J[a] * J[b]
  for a in range(6):
    for b in range(a):
      A[a][b] = A[b][a]
  return A, g


def gn_step64(A, g):
  """x = -A^-1 g solved exactly over the rationals (A, g as plane_system returns them), with cond_2(A).
  -> (x float64 [6], cond); x is None when A is singular."""
  n = 6
  M = [list(A[r]) + [-g[r]] for r in range(n)]
  for c in range(n):
    piv = next((r for r in range(c, n) if M[r][c] != 0), None)
    if piv is None:
      return None, math.inf
    M[c], M[piv] = M[piv], M[c]
    for r in range(n):
      if r != c and M[r][c] != 0:
        f = M[r][c] / M[c][c]
        M[r] = [a - f * b for a, b in zip(M[r], M[c])]
  x = np.array([float(M[r][n] / M[r][r]) for r in range(n)])
  Af = np.array([[float(v) for v in row] for row in A])
  return x, float(np.linalg.cond(Af))


def plane_sums(P, Q, N, dtype):
  """icp.cu's PointToPlane sums in `dtype`, added row by row: the upper triangle of J^T J (21, row-major) and J^T r
  (6).  J and r are formed in fp64 from the float32 rows and rounded to dtype once."""
  P, Q, N = _rows32(P), _rows32(Q), _rows32(N)
  J = np.c_[np.cross(P, N), N].astype(dtype)
  r = ((P - Q) * N).sum(1).astype(dtype)
  seq = lambda v: np.cumsum(v, dtype=dtype)[-1]
  a = [seq(J[:, i] * J[:, j]) for i in range(6) for j in range(i, 6)]
  return np.array(a, np.float64), np.array([seq(J[:, i] * r) for i in range(6)], np.float64)


def cholesky6_step(a, g):
  """kabsch.cuh's cholesky6_step in fp64: x = -(A^-1 g) from the upper triangle a[21]; None on a non-positive
  pivot."""
  A = np.zeros((6, 6))
  A[np.triu_indices(6)] = a
  A = A + np.triu(A, 1).T
  L = np.zeros((6, 6))
  for j in range(6):
    d = A[j, j] - sum(L[j, m] * L[j, m] for m in range(j))
    if not d > 0.0:
      return None
    L[j, j] = math.sqrt(d)
    for i in range(j + 1, 6):
      L[i, j] = (A[i, j] - sum(L[i, m] * L[j, m] for m in range(j))) / L[j, j]
  y = np.zeros(6)
  for i in range(6):
    y[i] = (-g[i] - sum(L[i, m] * y[m] for m in range(i))) / L[i, i]
  x = np.zeros(6)
  for i in range(5, -1, -1):
    x[i] = (y[i] - sum(L[m, i] * x[m] for m in range(i + 1, 6))) / L[i, i]
  return x


def scaled_cond(A):
  """cond_2(D^-1 A D^-1), D = sqrt(diag A): the conditioning a Cholesky solve actually suffers (it is invariant to
  diagonal scaling), unlike cond_2(A) of a system that is only badly scaled."""
  Af = np.array([[float(v) for v in row] for row in A])
  d = 1.0 / np.sqrt(np.diag(Af))
  return float(np.linalg.cond(d[:, None] * Af * d[None, :]))


def step_floor(A, x):
  """The 6x6 step's fp64 floor: 2^-53 cond(D^-1 A D^-1) |x|_max."""
  return U64 * scaled_cond(A) * float(np.abs(x).max())


def step_pose_err(T, T64, spread):
  """max(|R - R64|_max, |t - t64| / (|t64| + spread)) of two 4x4 poses."""
  T, T64 = _f64(T), _f64(T64)
  return max(float(np.abs(T[:3, :3] - T64[:3, :3]).max()),
             float(np.linalg.norm(T[:3, 3] - T64[:3, 3]) / (np.linalg.norm(T64[:3, 3]) + spread)))


def zyx_update_left(x, T):
  """kabsch.cuh's zyx_update_left in fp64: [Rz(x2) Ry(x1) Rx(x0) | x3..5] T for a 4x4 T."""
  ca, sa, cb, sb, cc, sc = math.cos(x[0]), math.sin(x[0]), math.cos(x[1]), math.sin(x[1]), math.cos(x[2]), \
      math.sin(x[2])
  Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1.0]])
  Ry = np.array([[cb, 0, sb], [0, 1.0, 0], [-sb, 0, cb]])
  Rx = np.array([[1.0, 0, 0], [0, ca, -sa], [0, sa, ca]])
  D = np.eye(4)
  D[:3, :3] = Rz @ Ry @ Rx
  D[:3, 3] = x[3:6]
  return D @ _f64(T)


# --------------------------------------------------------------------------- #
# inputs with a prescribed cross-covariance
# --------------------------------------------------------------------------- #
def random_orthogonal(g, det=1.0):
  Q, R = np.linalg.qr(g.normal(size=(3, 3)))
  Q = Q * np.sign(np.diag(R))
  if np.linalg.det(Q) * det < 0:
    Q[:, 2] *= -1
  return Q


def whitened(g, n):
  """n rows with zero mean and covariance X^T X / n = I exactly in fp64 (n >= 4)."""
  X = g.normal(size=(n, 3))
  X -= X.mean(0)
  L = np.linalg.cholesky(X.T @ X / n)
  return X @ np.linalg.inv(L).T


def lattice_pairs(seed, offset=0.0, side=12):
  """ICP pairs known in advance.  Target: a jittered unit lattice (one point per 0.5 cell, far from cell walls);
  source: a 1 mrad / 1 cm motion of it about its centroid, far smaller than the spacing, so every source row's nearest
  target is its own row.  offset moves both clouds away from the origin.  -> (source, target) float32."""
  g = np.random.default_rng(seed)
  ijk = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing='ij'), -1).reshape(-1, 3).astype(np.float64)
  Q = ijk + 0.25 + g.uniform(-0.05, 0.05, ijk.shape)
  c = Q.mean(0)
  a = g.normal(size=3)
  a *= 1e-3 / np.linalg.norm(a)
  Rm = zyx_update_left(np.r_[a, 0, 0, 0], np.eye(4))[:3, :3]
  Ps = (Q - c) @ Rm.T + c + g.uniform(-0.01, 0.01, 3)
  shift = offset * np.array([0.6, -0.48, 0.64])
  return (Ps + shift).astype(np.float32), (Q + shift).astype(np.float32)


def plane_normals(g, n, eps):
  """Unit normals within about eps of +z: cond(J^T J) grows as 1 / eps^2, by scaling alone."""
  N = np.c_[eps * g.normal(size=(n, 2)), np.ones(n)]
  return (N / np.linalg.norm(N, axis=1, keepdims=True)).astype(np.float32)


PLANE_CASES = {'cond-1e2': 1.5, 'cond-1e8': 1.7e-3, 'cond-1e12': 1.7e-5}   # normal spread eps of each cond(J^T J)


def plane_case(name):
  """(source, target, normals) of a PLANE_CASES entry."""
  eps = PLANE_CASES[name]
  Ps, Q = lattice_pairs(2)
  return Ps, Q, plane_normals(np.random.default_rng(round(-np.log10(eps))), len(Q), eps)


def plane_check(T, Ps, Q, N):
  """The 6x6 step criterion for the pose T after one point-to-plane step from the identity on the pairs (Ps, Q):
  e(T) <= KAPPA * max(e64, floor) against the exact step, with e64 the error of an honest fp64 pipeline (numpy fp64
  sums, LAPACK's solve) and floor = step_floor.  -> dict(ok, e, e64, floor, bound, ratio, cond, scaled_cond)."""
  A, gv = plane_system(Ps, Q, N)
  x, cond = gn_step64(A, gv)
  T64 = zyx_update_left(x, np.eye(4))
  Pd, Qd, Nd = _rows32(Ps), _rows32(Q), _rows32(N)
  J = np.c_[np.cross(Pd, Nd), Nd]
  r = ((Pd - Qd) * Nd).sum(1)
  e64 = step_pose_err(zyx_update_left(np.linalg.solve(J.T @ J, -(J.T @ r)), np.eye(4)), T64, 1.0)
  e = step_pose_err(T, T64, 1.0)
  fl = step_floor(A, x)
  bound = KAPPA * max(e64, fl)
  return dict(ok=bool(e <= bound), e=e, e64=e64, floor=fl, bound=bound, ratio=e / max(e64, fl), cond=cond,
              scaled_cond=scaled_cond(A))


def plane_restated(Ps, Q, N, dtype=np.float64):
  """The kernel's step restated: sums in dtype (fp32 for the negative control), then cholesky6_step in fp64."""
  return zyx_update_left(cholesky6_step(*plane_sums(Ps, Q, N, dtype)), np.eye(4))


def plane_fp32(Ps, Q, N):
  """The step fp32 end to end (J, J^T J, J^T r and the solve): the second negative control."""
  Pd, Qd, Nd = _rows32(Ps), _rows32(Q), _rows32(N)
  J = np.c_[np.cross(Pd, Nd), Nd].astype(np.float32)
  r = ((Pd - Qd) * Nd).sum(1).astype(np.float32)
  return zyx_update_left(np.linalg.solve(J.T @ J, -(J.T @ r)).astype(np.float64), np.eye(4))


def prescribed(g, sig, n=512, det_u=1.0, scale=1.0, offset=0.0):
  """(X, Y, w) float32 with Y = X M^T, M = U diag(sig) V^T, X isotropic (C = I) and uniform weights, so that
  S = M C = U diag(sig) V^T up to the float32 rounding of the rows (the references use the rows, not M).
  det_u = -1 gives det(U) det(V) < 0.  scale multiplies both clouds; offset (a float times the spread) moves both
  centroids away from the origin in different directions."""
  U, V = random_orthogonal(g, det_u), random_orthogonal(g)
  M = U @ np.diag(sig) @ V.T
  X = whitened(g, n) * scale
  Y = X @ M.T
  if offset:
    X = X + offset * scale * np.array([0.6, -0.48, 0.64])
    Y = Y + offset * scale * np.array([-0.36, 0.8, 0.48])
  return X.astype(np.float32), Y.astype(np.float32), np.ones(n, np.float32)
