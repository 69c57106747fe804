"""ORACLE (test infrastructure only) - PointNetLK: Aoki, Goforth, Srivatsan & Lucey, "PointNetLK: Robust & Efficient
Point Cloud Registration using PointNet", CVPR 2019, the ``PointNetLK`` row of the reference's published comparison
(the reference ran the authors' code; it ships none).

PARITY UNPINNED: this restates the published method and the defaults of the authors' released code, with every
rounding step ``dgr_pointnetlk`` takes written here.  Two details are from memory of that code and cannot be checked
offline: the state-dict key names (``h1.0`` ... ``h2.7``, see ``layers_from_state_dict``) and whether the default
iteration cap is 10 or 20 (10 here).

1. Network phi(P) -> R^1024: five 1x1 layers, each Conv1d(cin, cout, 1) with bias, eval-mode BatchNorm1d (eps 1e-5)
   and ReLU: 3 -> 64 -> 64 (h1), 64 -> 64 -> 128 -> 1024 (h2); then the max over points of each channel.  Every
   feature is >= 0.  Folding: s = gamma / sqrt(var + eps), W' = W s, b' = (b - mean) s + beta, in fp64, rounded to
   fp32 once for the library (``fold(..., f32=True)``).
2. Network input (the rounding contract): q = fp32(((g00 d0 + g01 d1) + g02 d2) + g03, ...) with d = fp64(p) - c,
   every operation an fp64 operation without contraction, c the centre and g the fp64 pose.  Oracle and library
   feed the same points to the network whenever they hold the same pose bits.
3. LK, template T = cloud 1, source S = cloud 0: centre each on its fp64 mean (``oracle.goicp.stats_mean``: the
   library's statistics kernel order, so the means have the same bits); J[:, i] = (f0 - phi(exp(-delta e_i) T)) /
   delta with f0 = phi(T); H = J^T J; a non-positive pivot of H's Cholesky factorisation -> status 1, g = I.  Then for
   k < max_iter: r = phi(g S) - f0, dx = -H^-1 J^T r; stop when |dx| < xtol (iterations k + 1); else g <- exp(dx) g.
   Pose = translate(mean_T) g translate(-mean_S).  J, H, the solve, exp and the pose are fp64 (sums in numpy's order;
   the library's fixed-order sums agree to round-off, not bit for bit).
4. exp(xi), xi = (omega, v) rotation first: R = I + A W + B W^2, t = (I + B W + C W^2) v, A = sin t / t,
   B = (1 - cos t) / t^2, C = (t - sin t) / t^3; Taylor series (through t^8) below t = 1e-2.  libm's and CUDA's sin /
   cos may differ in the last bit, so exp's bits may too.
"""
import math

import numpy as np

from .goicp import stats_mean

EPS = 1e-5
WIDTHS = ((3, 64), (64, 64), (64, 64), (64, 128), (128, 1024))
# (conv module, BatchNorm module) names of the published PointNet_features, in layer order
MODULES = (('h1.0', 'h1.1'), ('h1.3', 'h1.4'), ('h2.0', 'h2.1'), ('h2.3', 'h2.4'), ('h2.6', 'h2.7'))
RESULT = ('iterations', 'last_dx', 'last_r', 'status', 'n_src', 'n_tgt', 'host_reads')
TAYLOR = 1e-2


def _np(x):
  if hasattr(x, 'detach'):
    x = x.detach().cpu().numpy()
  return np.asarray(x, np.float64)


def layers_from_state_dict(sd):
  """[(W [cout, cin], b, gamma, beta, mean, var)] fp64 per layer from a PointNet_features state dict (no prefix)."""
  out = []
  for (conv, bn), (cin, cout) in zip(MODULES, WIDTHS):
    out.append((_np(sd[conv + '.weight']).reshape(cout, cin), _np(sd[conv + '.bias']), _np(sd[bn + '.weight']),
                _np(sd[bn + '.bias']), _np(sd[bn + '.running_mean']), _np(sd[bn + '.running_var'])))
  return out


def fold(layers, f32=False):
  """[(W', b')] with BN folded in fp64; f32: rounded to fp32 once (the library's weights)."""
  out = []
  for W, b, g, beta, mean, var in layers:
    s = g / np.sqrt(var + EPS)
    Wf, bf = W * s[:, None], (b - mean) * s + beta
    out.append((Wf.astype(np.float32), bf.astype(np.float32)) if f32 else (Wf, bf))
  return out


def phi(folded, X, dtype=np.float64):
  """Max-pooled features [1024] of the points X [n, 3], every layer evaluated in `dtype`."""
  h = np.asarray(X, dtype)
  for W, b in folded:
    h = h @ np.asarray(W, dtype).T + np.asarray(b, dtype)
    h = np.maximum(h, dtype(0))
  return h.max(axis=0)


def transform32(P, g, c=(0.0, 0.0, 0.0)):
  """The network input of the fp32 points P [n, 3] under the pose g (3x4 or 4x4, fp64) about the centre c."""
  d = np.asarray(P, np.float32).astype(np.float64) - np.asarray(c, np.float64)
  g = np.asarray(g, np.float64)
  q = np.empty_like(d)
  for a in range(3):
    q[:, a] = ((g[a, 0] * d[:, 0] + g[a, 1] * d[:, 1]) + g[a, 2] * d[:, 2]) + g[a, 3]
  return q.astype(np.float32)


def se3_exp(xi):
  """4x4 SE(3) exponential of the twist xi = (omega, v)."""
  w, v = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
  th2 = float(w @ w)
  th = math.sqrt(th2)
  if th < TAYLOR:
    A = 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0)))
    B = 0.5 * (1.0 - th2 / 12.0 * (1.0 - th2 / 30.0 * (1.0 - th2 / 56.0 * (1.0 - th2 / 90.0))))
    C = (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0 * (1.0 - th2 / 110.0)))) / 6.0
  else:
    A, B, C = math.sin(th) / th, (1.0 - math.cos(th)) / th2, (th - math.sin(th)) / (th2 * th)
  W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
  W2 = W @ W
  E = np.eye(4)
  E[:3, :3] = np.eye(3) + A * W + B * W2
  E[:3, 3] = (np.eye(3) + B * W + C * W2) @ v
  return E


def jacobian(f_jac, delta):
  """J [1024, 6] from the 7 Jacobian features [f0, phi(exp(-delta e_0) T), ...] (fp32 or fp64)."""
  f = np.asarray(f_jac, np.float64)
  return (f[0][:, None] - f[1:].T) / delta


def jacobian_poses(delta):
  out = [np.eye(4)]
  for i in range(6):
    xi = np.zeros(6)
    xi[i] = -delta
    out.append(se3_exp(xi))
  return out


def step(J, H, f, f0):
  """(dx, |dx|, |r|) of one LK step from the features f of the current iterate; None when H is singular."""
  r = np.asarray(f, np.float64) - np.asarray(f0, np.float64)
  try:
    L = np.linalg.cholesky(H)
  except np.linalg.LinAlgError:
    return None
  dx = -np.linalg.solve(L.T, np.linalg.solve(L, J.T @ r))
  return dx, float(np.linalg.norm(dx)), float(np.linalg.norm(r))


def _chol_ok(H):
  """True when the fp64 Cholesky factorisation of H has only positive pivots (the library's test)."""
  L = np.zeros((6, 6))
  for j in range(6):
    d = H[j, j] - L[j, :j] @ L[j, :j]
    if not d > 0.0:
      return False
    L[j, j] = math.sqrt(d)
    for i in range(j + 1, 6):
      L[i, j] = (H[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
  return True


def pointnetlk(src, tgt, folded, delta=1e-2, max_iter=10, xtol=1e-7, features=None):
  """PointNetLK of src (cloud 0) onto tgt (cloud 1), fp32 points.  folded: ``fold(layers, f32=True)``.
  features(P32) -> phi (default: fp64 arithmetic on the folded weights).
  -> (4x4 pose mapping src into tgt, info dict of RESULT fields, log [iterations, 16], J)."""
  src, tgt = np.asarray(src, np.float32), np.asarray(tgt, np.float32)
  feat = features or (lambda P: phi(folded, P))
  ms, mt = stats_mean(src), stats_mean(tgt)
  fj = [feat(transform32(tgt, g, mt)) for g in jacobian_poses(delta)]
  f0 = np.asarray(fj[0], np.float64)
  J = jacobian(fj, delta)
  H = J.T @ J
  g = np.eye(4)
  info = dict(iterations=0, last_dx=0.0, last_r=0.0, status=0, n_src=len(src), n_tgt=len(tgt), host_reads=0)
  log = []
  if not _chol_ok(H):
    info['status'] = 1
  else:
    for k in range(max_iter):
      dx, ndx, nr = step(J, H, feat(transform32(src, g, ms)), f0)
      log.append(np.concatenate([g[:3].reshape(12), [ndx, nr, 0.0, 0.0]]))
      info.update(iterations=k + 1, last_dx=ndx, last_r=nr)
      if ndx < xtol:
        break
      g = se3_exp(dx) @ g
  T = np.eye(4)
  T[:3, :3] = g[:3, :3]
  T[:3, 3] = g[:3, 3] - g[:3, :3] @ ms + mt
  return T, info, np.array(log).reshape(-1, 16), J
