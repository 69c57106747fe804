"""oracle/super4pcs.py (Super4PCS) on the CPU: its congruent sets against brute force, rigid invariance on an exact
copy, the base conditions, and the recovery of a room turned by 120 degrees where ICP from the identity fails."""
import itertools
import math

import numpy as np

from deepglobalregistration_b200 import synthetic as syn
from oracle import icp as oicp
from oracle import super4pcs as o4
from oracle.goicp import normalise
from test_oracle_goicp import goicp_case

ROT90 = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])


def dyadic_pair(seed, n=64):
  """(src, tgt, T): n = 64 points on a 1/8 grid, symmetric about a dyadic centre with one pair at distance 2, and
  the same points turned by 90 degrees and shifted by a dyadic offset, so normalising either is exact in fp32."""
  g = np.random.default_rng(seed)
  half = []
  while len(half) < n // 2 - 1:
    p = g.integers(-11, 12, 3) / 8.0
    if 0 < np.linalg.norm(p) < 1.9 and not any(np.array_equal(p, q) or np.array_equal(-p, q) for q in half):
      half.append(p)
  pts = np.array(half + [np.array([2.0, 0.0, 0.0])])
  src = np.concatenate([pts, -pts]) + np.array([0.25, -0.5, 0.125])
  T = np.eye(4)
  T[:3, :3], T[:3, 3] = ROT90, [0.5, -0.25, 1.0]
  return src.astype(np.float32), syn.apply_se3(T, src).astype(np.float32), T


def _setup(src, tgt, n_t, delta, overlap=1.0):
  X, Y32, _, _, s = normalise(src, tgt)
  Q = Y32[(np.arange(n_t) * len(Y32)) // n_t].astype(np.float64)
  r = float(np.sqrt((X[:, 0] * X[:, 0] + X[:, 1] * X[:, 1]) + X[:, 2] * X[:, 2]).max())
  return X, Q, delta / s, overlap * (2.0 * r)


def test_congruent_sets_equal_brute_force():
  src, tgt, _ = dyadic_pair(0, n=32)
  tgt = tgt + np.random.default_rng(1).normal(0, 0.01, tgt.shape).astype(np.float32)
  X, Q, dl, D = _setup(src, tgt, 32, 0.1)
  checked = 0
  for b in range(40):
    base = o4.select_base(X, b, 7, D, dl)
    if base is None:
      continue
    S1, S2 = o4.pairs(Q, base['d1'], dl), o4.pairs(Q, base['d2'], dl)
    ci, cj = o4.congruent(Q, S1, S2, base, dl, 0.0)
    got = {(S1[0][i], S1[1][i], S2[0][j], S2[1][j]) for i, j in zip(ci, cj)}
    assert len(got) == len(ci)
    lo_c, hi_c = o4.angle_bounds(base, dl, 0.0)
    n = len(Q)
    u, v, w, x = (a.reshape(-1) for a in np.meshgrid(*([np.arange(n)] * 4), indexing='ij'))
    a, c = Q[v] - Q[u], Q[x] - Q[w]
    aa, cc = o4.dot(a, a), o4.dot(c, c)
    e = (Q[u] + base['r1'] * (Q[v] - Q[u])) - (Q[w] + base['r2'] * (Q[x] - Q[w]))
    with np.errstate(invalid='ignore', divide='ignore'):
      cs = o4.dot(a, c) / (np.sqrt(aa) * np.sqrt(cc))
    ok = (u != v) & (u != w) & (u != x) & (v != w) & (v != x) & (w != x)
    ok &= (aa >= max(base['d1'] - dl, 0.0) ** 2) & (aa <= (base['d1'] + dl) ** 2)
    ok &= (cc >= max(base['d2'] - dl, 0.0) ** 2) & (cc <= (base['d2'] + dl) ** 2)
    ok &= (o4.dot(e, e) <= dl * dl) & (cs >= lo_c) & (cs <= hi_c)
    want = set(zip(u[ok], v[ok], w[ok], x[ok]))
    assert got == want, (b, len(got), len(want))
    # and in (i, j) order
    assert all((ci[k], cj[k]) < (ci[k + 1], cj[k + 1]) for k in range(len(ci) - 1))
    checked += 1
    if checked == 3:
      break
  assert checked == 3


def test_rigid_copy_keeps_the_true_correspondents_and_recovers_the_pose():
  src, tgt, T_gt = dyadic_pair(2)
  X, Q, dl, D = _setup(src, tgt, 64, 0.05)
  valid = 0
  for b in range(24):
    base = o4.select_base(X, b, 3, D, dl)
    if base is None:
      continue
    valid += 1
    S1, S2 = o4.pairs(Q, base['d1'], dl), o4.pairs(Q, base['d2'], dl)
    ci, cj = o4.congruent(Q, S1, S2, base, dl, 0.0)
    quads = {(S1[0][i], S1[1][i], S2[0][j], S2[1][j]) for i, j in zip(ci, cj)}
    assert tuple(base['rows']) in quads, b
  assert valid >= 8
  T, info, log = o4.super4pcs(src, tgt, n_sample_tgt=64, overlap=1.0, delta=0.05, dt_size=32, max_bases=16,
                              bases_per_round=8, terminate_fraction=1.0, seed=3)
  assert info['lcp'] == 64 and info['rounds'] == 1 and log.shape == (8, 16)
  assert np.abs(T - T_gt).max() <= 1e-9, np.abs(T - T_gt).max()


def test_valid_bases_meet_the_base_conditions():
  src, tgt, _, _ = goicp_case(5, n_s=200, n_t=400)
  X, _, dl, D = _setup(src, tgt, 400, 0.1, overlap=0.6)
  n_valid = 0
  for b in range(64):
    base = o4.select_base(X, b, 11, D, dl)
    if base is None:
      continue
    n_valid += 1
    P4 = X[base['rows']]
    assert len(set(base['rows'])) == 4
    rows = base['rows']
    d2 = [o4.dot(X[p] - X[q], X[p] - X[q]) for p, q in itertools.combinations(rows, 2)]
    assert max(d2) <= D * D
    h = []                                                               # one point within delta of the others' plane
    for k in range(4):
      o = [P4[m] for m in range(4) if m != k]
      cr = np.cross(o[1] - o[0], o[2] - o[0])
      h.append(abs(cr @ (P4[k] - o[0])) / np.linalg.norm(cr))
    assert min(h) <= dl * (1 + 1e-9)
    s, t, ok = o4.seg_params(P4[0], P4[1], P4[2], P4[3])
    assert ok and 0 <= s <= 1 and 0 <= t <= 1 and s == base['r1'] and t == base['r2']
  assert n_valid >= 32


def test_recovers_a_room_turned_by_120_degrees():
  src, tgt, T_gt, _ = goicp_case(1, n_s=256, n_t=4000, angle_deg=120)
  T_icp, _ = oicp.icp_point_to_point(src, tgt, 0.25)
  assert syn.rte_rre(T_icp, T_gt)[1] > math.radians(10)                 # ICP from the identity fails
  T, info, log = o4.super4pcs(src, tgt, n_sample_tgt=512, delta=0.1, dt_size=64, max_bases=16, bases_per_round=8,
                              terminate_fraction=0.95)
  te, re = syn.rte_rre(T, T_gt)
  assert info['valid_bases'] > 0 and info['lcp_fraction'] > 0.5, info
  assert re < math.radians(10) and te < 0.3, (te, math.degrees(re), info)
