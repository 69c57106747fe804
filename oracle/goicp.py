"""ORACLE (test infrastructure only) - Go-ICP: Yang, Li, Campbell & Jia, "Go-ICP: A Globally Optimal Solution to 3D
ICP Point-Set Registration", TPAMI 2016, the ``Go-ICP`` row of the reference's published comparison (the reference
ran the authors' binary; it ships no Go-ICP code).

PARITY UNPINNED: this restates the published algorithm with the boundary conventions below pinned here (they are
what ``dgr_goicp`` implements).  Where it departs from the paper's code, it does so to keep the search deterministic
and batch-parallel.

1. Normalise: each cloud is centred on its own fp64 mean - summed in the order of the library's statistics kernel
   (1024 strided per-thread sums, a butterfly per warp, the warps in order), so the means have the same bits - and
   both are divided by s, the larger of the two largest centred norms.  The target is then rounded to fp32.
2. Distance transform: G^3 cells over [-e, e]^3, h = fp32(2e / G); a point occupies cell floor((q + e) / h) clamped
   to the grid (fp32 arithmetic); each cell stores the exact squared distance in cells to the nearest occupied cell
   (separable exact 1-D passes along x, y, z).  Lookup of q: h sqrt(stored) plus the distance from q to the box,
   every step an fp32 operation.
3. Objective: the K = max(1, floor(n_s (1 - rho))) smallest fp32 terms (all of them, in point order, when K = n_s;
   ascending otherwise), widened to fp64, padded with zeros to a power of two, summed pairwise level by level.
4. Cubes: key (L, kx, ky, kz), half-width width / 2^(L+1), centre min + sigma (2k + 1) in fp64; ordered by (value,
   key); cubes stop splitting at level 19.  A rotation child whose point nearest the origin lies outside the pi-ball
   is dropped.  R = exp([r]x) by Rodrigues in fp64; R x rounded to fp32 once per rotation cube; t rounded to fp32.
5. Bounds: gamma_ri = fp32(2 sin(min(sqrt(3) sigma_r / 2, pi / 2)) |x_i|), gamma_t = fp32(sqrt(3) sigma_t); a bound
   is the trimmed sum of max(e_i - gamma, 0)^2.
6. Inner search: best first over translation cubes, the 8 children of a popped cube evaluated together (u with
   gamma_ri, l with gamma_ri + gamma_t); E-bar <- the (u, key)-smallest u below it, then the children with l < E-bar
   are pushed; stop on an empty pool or E-bar - LB < eps.  A pool of `inner_cap` cubes that cannot take the
   children, or a popped cube at level 19, ends the search: the lower-bound pass then returns min(E-bar, the
   smallest LB left).
7. Rounds: the B smallest pool cubes; every child searched against the round's E*; ICP from the (UB, key)-smallest
   child when it beats E*; the incumbent is the better of the child and the ICP pose (the child on a tie); children
   with LB < E* join the pool, the rest of the pool is pruned to LB < E* (both with the updated E*).
8. ICP: trimmed point-to-point on the normalised clouds, nearest target points by ``ransac_fm.feature_nn`` (the
   library uses dgr_knn_top1's fp32 distances), the K nearest (d^2, row) pairs, Kabsch; at most 30 updates, stopping
   when the trimmed MSE falls by less than 1e-6 of its previous value.  Its sums run in numpy's order, so once an ICP
   pose is the incumbent the library agrees to round-off, not bit for bit.
"""
import math

import numpy as np

from .icp import kabsch
from .ransac_fm import feature_nn

F32 = np.float32
MAX_LEVEL = 19
SQRT3 = math.sqrt(3.0)
FAR = 1 << 40
RESULT = ('E', 'lb_min', 'eps', 'K', 'converged', 'rounds', 'children', 'translation_cubes', 'icp_runs',
          'inner_overflows', 'pool_high_water', 'scale', 'host_reads')


# --------------------------------------------------------------------------- #
# normalisation
# --------------------------------------------------------------------------- #
def stats_mean(X):
  """fp64 mean of X [n, 3] summed as the library's statistics kernel sums it."""
  X = np.asarray(X, np.float64)
  n = len(X)
  rows = -(-n // 1024) * 1024
  P = np.zeros((rows, 3))
  P[:n] = X
  acc = np.zeros((1024, 3))
  for r in range(0, rows, 1024):
    acc = acc + P[r:r + 1024]
  acc = acc.reshape(32, 32, 3)
  lane = np.arange(32)
  for d in (16, 8, 4, 2, 1):
    acc = acc + acc[:, lane ^ d]
  s = np.zeros(3)
  for w in range(32):
    s = s + acc[w, 0]
  return s / n


def _norm(d):
  return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def normalise(src, tgt):
  """-> (source fp64 [n_s, 3], target fp32 [n_t, 3], m_s, m_t, s)."""
  S = np.asarray(src, np.float32).astype(np.float64)
  T = np.asarray(tgt, np.float32).astype(np.float64)
  ms, mt = stats_mean(S), stats_mean(T)
  s = max(_norm(S - ms).max(), _norm(T - mt).max())
  s = s if s > 0 else 1.0
  return (S - ms) / s, ((T - mt) / s).astype(F32), ms, mt, s


# --------------------------------------------------------------------------- #
# distance transform
# --------------------------------------------------------------------------- #
def _edt_1d(f, axis, chunk=256):
  """d[q] = min_p (q - p)^2 + f[p] along `axis` (exact, int64)."""
  f = np.moveaxis(f, axis, -1)
  shape = f.shape
  G = shape[-1]
  lines = f.reshape(-1, G)
  q = np.arange(G)
  D2 = (q[:, None] - q[None, :]) ** 2
  out = np.empty_like(lines)
  for lo in range(0, len(lines), chunk):
    out[lo:lo + chunk] = (lines[lo:lo + chunk, None, :] + D2[None]).min(-1)
  return np.moveaxis(np.minimum(out, FAR).reshape(shape), -1, axis)


class DistanceTransform:
  def __init__(self, y32, G, e):
    self.G = int(G)
    self.e32 = F32(e)
    self.h32 = F32(2.0 * e / G)
    cells = self.cells(np.asarray(y32, F32))
    occ = np.zeros((self.G,) * 3, bool)
    occ[cells[:, 2], cells[:, 1], cells[:, 0]] = True
    f = np.where(occ, 0, FAR).astype(np.int64)
    for axis in (2, 1, 0):                              # x, y, z of the [z, y, x] grid
      f = _edt_1d(f, axis)
    self.grid = f

  def cells(self, q):
    u = np.floor((q + self.e32) / self.h32)
    return np.clip(u, F32(0), F32(self.G - 1)).astype(np.int64)

  def lookup(self, q):
    """fp32 [..., 3] -> fp32 [...]"""
    c = self.cells(q)
    v = self.grid[c[..., 2], c[..., 1], c[..., 0]].astype(F32)
    D = self.h32 * np.sqrt(v)
    o = np.maximum(np.abs(q) - self.e32, F32(0))
    o2 = (o[..., 0] * o[..., 0] + o[..., 1] * o[..., 1]) + o[..., 2] * o[..., 2]
    return D + np.sqrt(o2)


# --------------------------------------------------------------------------- #
# cubes, rotations, bounds
# --------------------------------------------------------------------------- #
def child_key(key, o):
  L, kx, ky, kz = key
  return (L + 1, 2 * kx + ((o >> 2) & 1), 2 * ky + ((o >> 1) & 1), 2 * kz + (o & 1))


def key_int(key):
  L, kx, ky, kz = key
  return (L << 57) | (kx << 38) | (ky << 19) | kz


def cube_geom(key, mn, width):
  sigma = math.ldexp(width, -(key[0] + 1))
  return np.array([mn[a] + sigma * float(2 * key[1 + a] + 1) for a in range(3)]), sigma


def rodrigues(r):
  th = math.sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2])
  if th == 0.0:
    return np.eye(3)
  kx, ky, kz = r[0] / th, r[1] / th, r[2] / th
  c, s = math.cos(th), math.sin(th)
  C = 1.0 - c
  return np.array([[c + (kx * kx) * C, (kx * ky) * C - kz * s, (kx * kz) * C + ky * s],
                   [(kx * ky) * C + kz * s, c + (ky * ky) * C, (ky * kz) * C - kx * s],
                   [(kx * kz) * C - ky * s, (ky * kz) * C + kx * s, c + (kz * kz) * C]])


def rotate32(R, X):
  """fp32(R x) per point, each row (R0 x0 + R1 x1) + R2 x2 in fp64."""
  out = np.empty(X.shape, F32)
  for a in range(3):
    out[:, a] = ((R[a, 0] * X[:, 0] + R[a, 1] * X[:, 1]) + R[a, 2] * X[:, 2]).astype(F32)
  return out


def rotation_gamma(X, sigma_r):
  g = 2.0 * math.sin(min((SQRT3 * sigma_r) / 2.0, math.pi / 2))
  return (g * _norm(X)).astype(F32)


def translation_gamma(sigma_t):
  return F32(SQRT3 * sigma_t)


def tree_sum(terms, K):
  """[m, n] fp32 -> [m] fp64: the K smallest (all, in order, when K = n) over the pairwise tree."""
  t = np.asarray(terms, F32)
  if K < t.shape[1]:
    t = np.sort(t, axis=1)[:, :K]
  v = t.astype(np.float64)
  P = 1
  while P < v.shape[1]:
    P *= 2
  v = np.concatenate([v, np.zeros((len(v), P - v.shape[1]))], axis=1)
  while v.shape[1] > 1:
    v = v.reshape(len(v), -1, 2).sum(2)
  return v[:, 0]


def bounds(dt, Xr, t32, gam, gt, K):
  """Xr fp32 [n, 3], t32 fp32 [m, 3], gam fp32 [n], gt fp32 [m] -> (u [m], l [m]) fp64."""
  e = dt.lookup(Xr[None] + t32[:, None])
  du = np.maximum(e - gam[None], F32(0))
  dl = np.maximum(e - (gam[None] + gt[:, None]), F32(0))
  return tree_sum(du * du, K), tree_sum(dl * dl, K)


def objective(dt, X, R, t, K):
  """E(R, t) of the normalised source X (fp64) with fp32(R x) and fp32(t)."""
  Xr = rotate32(R, X)
  u, _ = bounds(dt, Xr, np.asarray(t, np.float64).astype(F32)[None], np.zeros(len(X), F32), np.zeros(1, F32), K)
  return float(u[0])


# --------------------------------------------------------------------------- #
# searches
# --------------------------------------------------------------------------- #
def inner_search(dt, Xr, gam, E0, eps, K, tmin, tw, inner_cap):
  """-> (E-bar, t centre, translation cubes evaluated, overflowed)."""
  pool = [(0.0, key_int((0, 0, 0, 0)), (0, 0, 0, 0))]
  E = E0
  t_best, _ = cube_geom((0, 0, 0, 0), tmin, tw)
  evals, ovf, left = 0, False, math.inf
  while pool:
    i = min(range(len(pool)), key=lambda j: pool[j][:2])
    lb, _, key = pool.pop(i)
    if E - lb < eps:
      break
    if key[0] >= MAX_LEVEL:
      ovf, left = True, lb
      break
    kids = [child_key(key, o) for o in range(8)]
    geo = [cube_geom(k, tmin, tw) for k in kids]
    t32 = np.array([g[0] for g in geo]).astype(F32)
    gt = np.array([translation_gamma(g[1]) for g in geo], F32)
    u, l = bounds(dt, Xr, t32, gam, gt, K)
    evals += 8
    best = -1
    for o in range(8):
      if u[o] < E and (best < 0 or u[o] < u[best]):
        best = o
    if best >= 0:
      E, t_best = float(u[best]), geo[best][0]
    push = [o for o in range(8) if l[o] < E]
    if len(pool) + len(push) > inner_cap:
      ovf = True
      left = min([lb for lb, _, _ in pool] + [float(l[o]) for o in push])
      break
    pool += [(float(l[o]), key_int(kids[o]), kids[o]) for o in push]
  return E, t_best, evals, ovf, left


def trimmed_icp(X, Y32, T, K, max_updates=30):
  """-> 4x4 pose of the normalised frame."""
  T = np.array(T, np.float64)
  Y = Y32.astype(np.float64)
  prev = math.inf
  for _ in range(max_updates):
    P = X @ T[:3, :3].T + T[:3, 3]
    nn = feature_nn(P.astype(F32), Y32)
    d2 = ((P - Y[nn]) ** 2).sum(1)
    order = np.lexsort((np.arange(len(X)), d2))[:K]
    mse = d2[order].sum() / K
    if prev - mse < 1e-6 * prev:
      break
    R, t = kabsch(X[order], Y[nn[order]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    prev = mse
  return T


def goicp(src, tgt, mse_thresh=1e-3, trim_fraction=0.0, dt_size=300, dt_expand=2.0, rot_min=(-math.pi,) * 3,
          rot_width=2 * math.pi, trans_min=(-1.0, -1.0, -1.0), trans_width=2.0, cubes_per_round=64,
          max_rounds=100000, max_rotation_cubes=1 << 20, inner_cap=1536):
  """-> (4x4 pose mapping src into tgt, info dict with the fields of RESULT)."""
  X, Y32, ms, mt, s = normalise(src, tgt)
  n = len(X)
  K = max(1, int(math.floor(n * (1.0 - trim_fraction))))
  eps = mse_thresh * K
  dt = DistanceTransform(Y32, dt_size, dt_expand)
  info = dict(eps=eps, K=K, children=0, translation_cubes=0, icp_runs=1, inner_overflows=0, host_reads=0,
              scale=s, converged=0, rounds=0)
  T = trimmed_icp(X, Y32, np.eye(4), K)
  E = objective(dt, X, T[:3, :3], T[:3, 3], K)
  pool = [(0.0, key_int((0, 0, 0, 0)), (0, 0, 0, 0))]      # sorted by (LB, key)
  lb_min, hw, stop = 0.0, 1, False
  while True:
    info['host_reads'] += 1
    if stop:
      break
    if not pool or E - lb_min < eps:
      info['converged'] = 1
      break
    if info['rounds'] >= max_rounds:
      break
    Bp = min(cubes_per_round, len(pool))
    kids = []
    for _, _, pkey in pool[:Bp]:
      for o in range(8):
        if pkey[0] >= MAX_LEVEL:
          stop = True
          continue
        key = child_key(pkey, o)
        r0, sr = cube_geom(key, rot_min, rot_width)
        d = np.maximum(np.abs(r0) - sr, 0.0)
        if (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] > math.pi * math.pi:
          continue
        R = rodrigues(r0)
        Xr = rotate32(R, X)
        ub, tc, ev1, o1, _ = inner_search(dt, Xr, np.zeros(n, F32), E, eps, K, trans_min, trans_width, inner_cap)
        lb, _, ev2, o2, left = inner_search(dt, Xr, rotation_gamma(X, sr), E, eps, K, trans_min, trans_width,
                                            inner_cap)
        if o2:
          lb = min(lb, left)
        info['children'] += 1
        info['translation_cubes'] += ev1 + ev2
        info['inner_overflows'] += int(o1) + int(o2)
        kids.append((ub, lb, key_int(key), key, R, tc))
    if kids:
      ub, _, _, _, R, tc = min(kids, key=lambda k: (k[0], k[2]))
      if ub < E:
        info['icp_runs'] += 1
        Tc = np.eye(4)
        Tc[:3, :3], Tc[:3, 3] = R, tc
        Ti = trimmed_icp(X, Y32, Tc, K)
        Ei = objective(dt, X, Ti[:3, :3], Ti[:3, 3], K)
        E, T = (Ei, Ti) if Ei < ub else (ub, Tc)
    new = sorted([(lb, ki, key) for _, lb, ki, key, _, _ in kids if lb < E] +
                 [p for p in pool[Bp:] if p[0] < E], key=lambda p: p[:2])
    lb_min = new[0][0] if new else E
    info['rounds'] += 1
    if len(new) > max_rotation_cubes:
      stop = True
    else:
      pool = new
      hw = max(hw, len(pool))
  info.update(E=E, lb_min=lb_min if pool else E, pool_high_water=hw)
  Tn = np.eye(4)
  Tn[:3, :3] = T[:3, :3]
  Tn[:3, 3] = mt + s * T[:3, 3] - T[:3, :3] @ ms
  return Tn, info
