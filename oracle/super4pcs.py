"""ORACLE (test infrastructure only) - Super4PCS: Mellado, Aiger & Mitra, "Super 4PCS: Fast Global Pointcloud
Registration via Smart Indexing", SGP 2014 (after 4PCS: Aiger, Mitra & Cohen-Or, SIGGRAPH 2008), the ``Super4PCS``
row of the reference's published comparison (the reference ran the authors' binary; it ships no Super4PCS code).

PARITY UNPINNED: this restates the published algorithm with the conventions below pinned here (they are what
``dgr_super4pcs`` implements).  Geometry is fp64 in the operation order written below, with no contraction; the
one fp32 step is the distance-transform lookup (Go-ICP's, ``oracle.goicp``).  Departures from the paper and from
OpenGR (the authors' library) are marked [dep] and keep the search deterministic and batch-parallel.

1. Normalise: the source sample P (n_s <= 1024 rows, sampled by the caller) and the whole target by Go-ICP's rule
   (``oracle.goicp.normalise``: each centred, both divided by s); the target's distance transform is built over them
   (``oracle.goicp.DistanceTransform``, G = dt_size over [-e, e]^3).  Q: rows floor(k n1 / n_t) of the normalised
   fp32 target, widened to fp64.  delta = delta_m / s; r = max_i |p_i| (norm sqrt((x^2 + y^2) + z^2)); D =
   overlap (2 r).
2. Base b: T = 32 triplets; triplet t takes rows draws 3 (T b + t) + {0, 1, 2} of the counter-hash stream of
   ``seed`` (``oracle.ransac``'s mix).  Valid: three distinct rows, every squared edge in [(D / 4)^2, D^2], area
   key A = |(p2 - p1) x (p3 - p1)|^2 > 0.  The largest A wins, ties to the lowest t.  The fourth point is the row l
   minimising |((p2 - p1) x (p3 - p1)) . (p_l - p1)| (ties: lowest l) [dep: the plane distance times |cross|, the
   same order up to ties], among rows not in the triplet, within D of each triplet point (squared distances against
   D^2), for which one of the pairings (12|34), (13|24), (14|23), tried in that order, has both closest-point line
   parameters s, t in [0, 1] (den = a11 a22 - a12^2 > 0, s = (a12 e2 - a22 e1) / den, t = (a11 e2 - a12 e1) / den).
   The base is invalid when there is no triplet, no fourth point, or the plane distance key / sqrt(A) > delta.  The
   base (b1, b2 | b3, b4) is the pairing's order; r1 = s, r2 = t; d1 = |b2 - b1|, d2 = |b4 - b3|;
   cos = ((b2 - b1) . (b4 - b3)) / (d1 d2).
3. Pairs: S_k = ordered (u, v), u != v, of Q with lo^2 <= |q_v - q_u|^2 <= hi^2, lo = max(d_k - delta, 0),
   hi = d_k + delta [dep: | |q_v - q_u| - d_k | <= delta without a square root], in row-major (u, v) order; the
   first max_pairs are kept, the rest counted as dropped.
4. Congruent sets: (i in S1, j in S2) with u, v, w, x distinct, |e1 - e2|^2 <= delta^2 (e1 = q_u + r1 (q_v - q_u),
   e2 = q_w + r2 (q_x - q_w), per component), and cos(min(theta + tol, pi)) <= c <= cos(max(theta - tol, 0)) for
   c = ((q_v - q_u) . (q_x - q_w)) / (|q_v - q_u| |q_x - q_w|) and theta = acos(clip(cos, -1, 1)).  tol =
   angle_tol, or 2 delta / min(d1, d2) when angle_tol = 0.  Ordered by (i, j); the first max_candidates are kept.
   These three transcendental calls per base are the one place the library may differ from numpy by an ulp.
5. Fit: Kabsch of (b1..b4) -> (q_u, q_v, q_w, q_x) (``oracle.ransac.kabsch_batch``, LAPACK's SVD; the library
   runs ``kabsch_rotation``'s fp64 Jacobi on the same means and cross-covariance without contraction, and the two
   rotations agree to round-off, not bit for bit); rejected when some |R b_k + t - q_k|^2 > delta^2 (R b per row
   ((R0 b0 + R1 b1) + R2 b2), then + t).  So the residual test, the prefilter and the LCP counts - and the base log
   - equal the library's unless a residual or a transformed point lies within round-off of delta or of a cell
   boundary of the distance transform (the pose then agrees to ~1e-15, not the counts).  The candidates of step 4
   have no such exception: the library's join hashes e2 into cells delta (1 + 2^-20) wide, so every pair within
   delta lies in the 27 cells around e1 whatever the rounding of the cell division, and both sides then apply the
   same exact predicate.
6. Verify: the prefilter count of a fit is the number of the 64 rows floor(k n_s / 64) whose fp32(R p + t) has a
   distance-transform lookup <= fp32(delta).  The V = verify_per_base fits of largest (count, then lowest
   candidate index) are scored on all of P the same way (the LCP).  A base's best is its largest LCP, lowest
   candidate on a tie.
7. Rounds of B = bases_per_round bases (the last may be shorter) up to max_bases; the best over all bases wins by
   (LCP descending, base ascending, candidate ascending).  The search stops at the end of the first round whose best
   LCP is >= terminate_fraction n_s.  The pose is de-normalised into the input frame as Go-ICP's is.
"""
import math

import numpy as np
from scipy.spatial import cKDTree

from .goicp import DistanceTransform, normalise
from .ransac import _mix64, kabsch_batch

F32 = np.float32
TRIPLETS = 32
PREFILTER = 64
LOG = ('b1', 'b2', 'b3', 'b4', 'valid', 's1', 's2', 'candidates', 'candidates_dropped', 'verified', 'best_lcp',
       'best_candidate', 'pad0', 'pad1', 'pad2', 'pad3')
RESULT = ('lcp_fraction', 'lcp', 'bases', 'valid_bases', 'candidates', 'pairs_dropped', 'candidates_dropped',
          'best_base', 'best_candidate', 'rounds', 'scale', 'host_reads')
PAIRINGS = ((0, 1, 2, 3), (0, 2, 1, 3), (0, 3, 1, 2))


def draws(seed, first, count, n):
  d = np.arange(first, first + count, dtype=np.uint64)
  with np.errstate(over='ignore'):
    z = _mix64(np.uint64(int(seed) & (2**64 - 1)) + (d + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15))
  return (((z >> np.uint64(32)) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def dot(a, b):
  return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
  return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                   a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def seg_params(x1, x2, x3, x4):
  """closest-point parameters (s on x1 -> x2, t on x3 -> x4) and whether both lie in [0, 1]"""
  d1, d2, r = x2 - x1, x4 - x3, x1 - x3
  a11, a12, a22, e1, e2 = dot(d1, d1), dot(d1, d2), dot(d2, d2), dot(d1, r), dot(d2, r)
  den = a11 * a22 - a12 * a12
  ok = den > 0
  sd = np.where(ok, den, 1.0)
  s = (a12 * e2 - a22 * e1) / sd
  t = (a11 * e2 - a12 * e1) / sd
  return s, t, ok & (s >= 0) & (s <= 1) & (t >= 0) & (t <= 1)


def select_base(X, b, seed, D, delta):
  """-> None (invalid) or dict(rows [4] in pairing order, r1, r2, d1, d2, cos)."""
  n = len(X)
  idx = draws(seed, 3 * TRIPLETS * b, 3 * TRIPLETS, n).reshape(TRIPLETS, 3)
  A, B, C = X[idx[:, 0]], X[idx[:, 1]], X[idx[:, 2]]
  lo2, hi2 = (D * 0.25) * (D * 0.25), D * D
  e = [dot(B - A, B - A), dot(C - B, C - B), dot(A - C, A - C)]
  area = dot(cross(B - A, C - A), cross(B - A, C - A))
  ok = (idx[:, 0] != idx[:, 1]) & (idx[:, 1] != idx[:, 2]) & (idx[:, 0] != idx[:, 2]) & (area > 0)
  for x in e:
    ok &= (x >= lo2) & (x <= hi2)
  if not ok.any():
    return None
  t = int(np.argmax(np.where(ok, area, -1.0)))
  tri = idx[t]
  a, bb, c = X[tri[0]], X[tri[1]], X[tri[2]]
  cr = cross(bb - a, c - a)
  key = np.abs(dot(cr[None], X - a))
  near = (dot(X - a, X - a) <= hi2) & (dot(X - bb, X - bb) <= hi2) & (dot(X - c, X - c) <= hi2)
  near &= (np.arange(n) != tri[0]) & (np.arange(n) != tri[1]) & (np.arange(n) != tri[2])
  pts = [np.broadcast_to(a, X.shape), np.broadcast_to(bb, X.shape), np.broadcast_to(c, X.shape), X]
  which = np.full(n, -1)
  for k in (2, 1, 0):                                     # the first pairing that works wins
    _, _, okp = seg_params(*(pts[o] for o in PAIRINGS[k]))
    which = np.where(okp, k, which)
  cand = near & (which >= 0)
  if not cand.any():
    return None
  l = int(np.argmin(np.where(cand, key, np.inf)))
  if key[l] / math.sqrt(area[t]) > delta:
    return None
  rows4 = [int(tri[0]), int(tri[1]), int(tri[2]), l]
  order = PAIRINGS[int(which[l])]
  rows = [rows4[o] for o in order]
  P4 = X[rows]
  s, tt, _ = seg_params(P4[0], P4[1], P4[2], P4[3])
  v1, v2 = P4[1] - P4[0], P4[3] - P4[2]
  d1, d2 = math.sqrt(dot(v1, v1)), math.sqrt(dot(v2, v2))
  return dict(rows=rows, P4=P4, r1=float(s), r2=float(tt), d1=d1, d2=d2, cos=float(dot(v1, v2) / (d1 * d2)))


def pairs(Q, d, delta):
  """all ordered (u, v), u != v, with | |q_v - q_u| - d | <= delta (squared form), row-major order"""
  lo, hi = max(d - delta, 0.0), d + delta
  diff = Q[None, :, :] - Q[:, None, :]
  dd = dot(diff, diff)
  m = (dd >= lo * lo) & (dd <= hi * hi)
  np.fill_diagonal(m, False)
  u, v = np.nonzero(m)
  return u, v


def angle_bounds(base, delta, angle_tol):
  tol = angle_tol if angle_tol > 0 else 2.0 * delta / min(base['d1'], base['d2'])
  th = math.acos(min(max(base['cos'], -1.0), 1.0))
  return math.cos(min(th + tol, math.pi)), math.cos(max(th - tol, 0.0))


def cosines(Q, u, v, w, x):
  a, b = Q[v] - Q[u], Q[x] - Q[w]
  return dot(a, b) / (np.sqrt(dot(a, a)) * np.sqrt(dot(b, b)))


def congruent(Q, S1, S2, base, delta, angle_tol):
  """candidate (i, j) index pairs into S1, S2 in (i, j) order: the predicates of step 4"""
  (u, v), (w, x) = S1, S2
  if len(u) == 0 or len(w) == 0:
    return np.zeros(0, np.int64), np.zeros(0, np.int64)
  e1 = Q[u] + base['r1'] * (Q[v] - Q[u])
  e2 = Q[w] + base['r2'] * (Q[x] - Q[w])
  near = cKDTree(e2).query_ball_point(e1, delta * (1 + 1e-6) + 1e-12)
  ii = np.repeat(np.arange(len(u)), [len(l) for l in near])
  jj = np.concatenate([np.asarray(l, np.int64) for l in near]) if len(ii) else np.zeros(0, np.int64)
  lo_c, hi_c = angle_bounds(base, delta, angle_tol)
  return filter_candidates(Q, S1, S2, base, delta, lo_c, hi_c, ii, jj)


def filter_candidates(Q, S1, S2, base, delta, lo_c, hi_c, ii, jj):
  (u, v), (w, x) = S1, S2
  u, v, w, x = u[ii], v[ii], w[jj], x[jj]
  e1 = Q[u] + base['r1'] * (Q[v] - Q[u])
  e2 = Q[w] + base['r2'] * (Q[x] - Q[w])
  c = cosines(Q, u, v, w, x)
  ok = (u != w) & (u != x) & (v != w) & (v != x) & (dot(e1 - e2, e1 - e2) <= delta * delta)
  ok &= (c >= lo_c) & (c <= hi_c)
  ii, jj = ii[ok], jj[ok]
  o = np.lexsort((jj, ii))
  return ii[o], jj[o]


def transform(R, t, X):
  """fp64 rows ((R0 x0 + R1 x1) + R2 x2) + t; R [m, 3, 3], t [m, 3], X [n, 3] -> [m, n, 3]"""
  out = np.empty((len(R), len(X), 3))
  for a in range(3):
    out[..., a] = ((R[:, a, 0, None] * X[None, :, 0] + R[:, a, 1, None] * X[None, :, 1]) +
                   R[:, a, 2, None] * X[None, :, 2]) + t[:, a, None]
  return out


def fits(Q, S1, S2, base, ci, cj, delta):
  """-> (R [m, 3, 3], t [m, 3], ok [m])"""
  (u, v), (w, x) = S1, S2
  dst = np.stack([Q[u[ci]], Q[v[ci]], Q[w[cj]], Q[x[cj]]], 1)
  src = np.broadcast_to(base['P4'], dst.shape)
  if len(ci) == 0:
    return np.zeros((0, 3, 3)), np.zeros((0, 3)), np.zeros(0, bool)
  R, t = kabsch_batch(src, dst)
  res = np.stack([transform(R[k:k + 1], t[k:k + 1], base['P4'])[0] for k in range(len(R))]) - dst
  return R, t, (dot(res, res) <= delta * delta).all(1)


def lcp(dt, R, t, X, d32):
  """points of X within delta of the target after the pose: fp32(R x + t), lookup <= fp32(delta)"""
  if len(R) == 0:
    return np.zeros(0, np.int64)
  P = transform(R, t, X).astype(F32)
  return (dt.lookup(P) <= d32).sum(1)


def super4pcs(src, tgt, n_sample_tgt=1024, overlap=0.5, delta=0.1, angle_tol=0.0, dt_size=300, dt_expand=2.0,
              max_bases=256, bases_per_round=64, max_pairs=262144, max_candidates=65536, verify_per_base=64,
              terminate_fraction=0.9, seed=0):
  """-> (4x4 pose mapping src into tgt, info dict with the fields of RESULT, base log int32 [bases, 16])."""
  X, Y32, ms, mt, s = normalise(src, tgt)
  n_s, n1 = len(X), len(Y32)
  Q = Y32[(np.arange(n_sample_tgt) * n1) // n_sample_tgt].astype(np.float64)
  dt = DistanceTransform(Y32, dt_size, dt_expand)
  dl = delta / s
  d32 = F32(dl)
  r = float(np.sqrt((X[:, 0] * X[:, 0] + X[:, 1] * X[:, 1]) + X[:, 2] * X[:, 2]).max())
  D = overlap * (2.0 * r)
  pf = (np.arange(PREFILTER) * n_s) // PREFILTER
  info = dict(lcp=0, bases=0, valid_bases=0, candidates=0, pairs_dropped=0, candidates_dropped=0, best_base=-1,
              best_candidate=-1, rounds=0, scale=s, host_reads=0)
  best_lcp, best_pose = -1, (np.eye(3), np.zeros(3))
  log = []
  b = 0
  while b < max_bases:
    for b in range(b, min(b + bases_per_round, max_bases)):
      rec = np.zeros(16, np.int32)
      rec[:4] = -1
      rec[10:12] = -1
      info['bases'] += 1
      base = select_base(X, b, seed, D, dl)
      if base is not None:
        info['valid_bases'] += 1
        rec[:5] = base['rows'] + [1]
        S1, S2 = pairs(Q, base['d1'], dl), pairs(Q, base['d2'], dl)
        rec[5:7] = len(S1[0]), len(S2[0])
        info['pairs_dropped'] += max(0, len(S1[0]) - max_pairs) + max(0, len(S2[0]) - max_pairs)
        S1 = (S1[0][:max_pairs], S1[1][:max_pairs])
        S2 = (S2[0][:max_pairs], S2[1][:max_pairs])
        ci, cj = congruent(Q, S1, S2, base, dl, angle_tol)
        kept = min(len(ci), max_candidates)
        rec[7:9] = kept, min(len(ci) - kept, 2**31 - 1)               # int32 log field, saturated
        info['candidates'] += kept
        info['candidates_dropped'] += len(ci) - kept
        ci, cj = ci[:kept], cj[:kept]
        R, t, ok = fits(Q, S1, S2, base, ci, cj, dl)
        pre = lcp(dt, R, t, X[pf], d32)
        k_ok = np.nonzero(ok)[0]
        order = k_ok[np.lexsort((k_ok, -pre[k_ok]))][:verify_per_base]
        sel = np.sort(order)
        rec[9] = len(sel)
        full = lcp(dt, R[sel], t[sel], X, d32)
        if len(sel):
          k = int(np.argmax(full))                         # the first largest: lowest candidate index
          rec[10:12] = full[k], sel[k]
          if full[k] > best_lcp:
            best_lcp = int(full[k])
            info['best_base'], info['best_candidate'] = b, int(sel[k])
            best_pose = (R[sel[k]], t[sel[k]])
      log.append(rec)
    b += 1
    info['rounds'] += 1
    if max(best_lcp, 0) >= terminate_fraction * n_s:
      break
  info['lcp'] = max(best_lcp, 0)
  info['lcp_fraction'] = info['lcp'] / n_s
  R, t = best_pose
  T = np.eye(4)
  T[:3, :3] = R
  T[:3, 3] = mt + s * t - R @ ms
  return T, info, np.array(log, np.int32).reshape(-1, 16)
