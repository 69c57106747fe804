"""oracle/fpfh.py (open3d 0.10's ComputeFPFHFeature, float64) on hand-worked pair features and bins, the SPFH and
FPFH normalisations, and rigid-motion invariance."""
import math

import numpy as np

from deepglobalregistration_b200 import synthetic as syn
from oracle import fpfh as ofp


def _feature(p1, n1, p2, n2):
  a, f, t, amb = ofp.pair_features(np.array(p1, float), np.array(n1, float), np.array(p2, float), np.array(n2, float))
  return (float(a), float(f), float(t)), bool(amb)


def test_pair_features_hand_worked():
  s, c = math.sin(0.3), math.cos(0.3)
  # n1 tilted towards d, n2 along z: |a1| > |a2|, no swap; theta = a1, alpha = -0.3
  (a, f, t), amb = _feature((0, 0, 0), (s, 0, c), (1, 0, 0), (0, 0, 1))
  assert abs(a + 0.3) < 1e-15 and abs(f) < 1e-15 and abs(t - s) < 1e-15 and not amb
  # the swap branch: n2 tilted towards d; n1 / n2 swap, d flips, theta = -a2, alpha = +0.3
  (a, f, t), amb = _feature((0, 0, 0), (0, 0, 1), (1, 0, 0), (s, 0, c))
  assert abs(a - 0.3) < 1e-15 and abs(f) < 1e-15 and abs(t + s) < 1e-15 and not amb
  # phi: n2 tilted across d (towards v = d x n1 = -y)
  (a, f, t), amb = _feature((0, 0, 0), (0, 0, 1), (0.5, 0, 0), (0, -s, c))
  assert abs(f - s) < 1e-15 and abs(t) < 1e-15 and amb          # |a1| == |a2| == 0: the swap test ties
  # |d| = 0 and d parallel to n1 are degenerate: the zero feature, bins 5 / 16 / 27
  for p2, n2, want_amb in (((0, 0, 0), (1, 0, 0), False), ((0, 0, 2), (1, 0, 0), True)):
    (a, f, t), amb = _feature((0, 0, 0), (0, 0, 1), p2, n2)
    assert (a, f, t) == (0.0, 0.0, 0.0) and amb == want_amb
    assert ofp.bins(np.float64(a), np.float64(f), np.float64(t)).tolist() == [5, 16, 27]


def test_bins_clamp_at_the_ends():
  assert ofp.bins(np.float64(math.pi), np.float64(1.0), np.float64(-1.0)).tolist() == [10, 21, 22]
  assert ofp.bins(np.float64(-math.pi), np.float64(-1.0), np.float64(1.0)).tolist() == [0, 11, 32]
  assert ofp.bins(np.float64(2 * math.pi), np.float64(3.0), np.float64(-3.0)).tolist() == [10, 21, 22]
  # the +-pi wrap of alpha: atan2(+-0, negative)
  assert ofp.bins(np.arctan2(0.0, -1.0), np.float64(0), np.float64(0))[0] == 10
  assert ofp.bins(np.arctan2(-0.0, -1.0), np.float64(0), np.float64(0))[0] == 0
  # antiparallel normals across d: alpha = atan2(0, -1) is on the band's edge
  _, amb = _feature((0, 0, 0), (0, 0, 1), (1, 0, 0.3), (0, 0, -1))
  assert amb


def _cloud(seed, n=600):
  g = np.random.default_rng(seed)
  P = g.uniform(0.0, 1.0, size=(n, 3))
  N = g.normal(size=(n, 3))
  return P, N / np.linalg.norm(N, axis=1, keepdims=True)


def test_spfh_and_fpfh_normalisation():
  P, N = _cloud(1)
  P = np.vstack([P, [[5.0, 5.0, 5.0]]])                    # an isolated point: m = 0
  N = np.vstack([N, [[0.0, 0.0, 1.0]]])
  out = ofp.compute_fpfh(P, N, 0.2, 30)
  m, spfh, fpfh = out['m'], out['spfh'], out['fpfh']
  assert m[-1] == 0 and not spfh[-1].any() and not fpfh[-1].any()
  assert (out['counts'] > 30).any() and m.max() == 29      # the max_nn truncation ran
  live = m > 0
  groups = spfh.reshape(-1, 3, 11).sum(2)
  assert np.all(np.abs(groups[live] - 100.0) <= 1e-9)
  assert np.all(groups[~live] == 0.0)
  # each FPFH group: 100 from the normalised neighbour sum plus 100 from the point's own SPFH
  weighted = np.zeros((len(P), 3))
  for i in np.flatnonzero(live):
    for k in range(m[i]):
      weighted[i] += spfh[out['nb'][i, k]].reshape(3, 11).sum(1) / out['d2'][i, k]
  fg = fpfh.reshape(-1, 3, 11).sum(2)
  nz = live[:, None] & (weighted != 0.0)
  assert nz.any() and np.all(np.abs(fg[nz] - 200.0) <= 1e-9)


def test_repeated_addition_is_not_a_product():
  """100 / m added m times is the SPFH value, not m * (100 / m): the two differ for some m."""
  incr = np.array([100.0 / 7])
  got = ofp._repeated_sum(incr, np.array([[7]]))[0, 0]
  want = 0.0
  for _ in range(7):
    want += 100.0 / 7
  assert got == want


def test_rigid_motion_invariance():
  P, N = _cloud(2, 800)
  T = syn.random_se3(np.random.default_rng(3), 60.0, 2.0)
  Q = P @ T[:3, :3].T + T[:3, 3]
  NQ = N @ T[:3, :3].T
  a = ofp.compute_fpfh(P, N, 0.15, 128)
  b = ofp.compute_fpfh(Q, NQ, 0.15, 128)
  assert np.array_equal(a['nb'], b['nb']) and a['counts'].max() < 128     # the same lists, none truncated
  ok = ~(a['ambiguous'] | b['ambiguous'])
  assert ok.mean() > 0.9, ok.mean()
  assert np.abs(a['fpfh'][ok] - b['fpfh'][ok]).max() <= 1e-9
