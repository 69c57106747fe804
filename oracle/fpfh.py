"""ORACLE (test infrastructure only) - FPFH features as open3d's global-registration recipe computes them:
``compute_fpfh_feature(pcd, KDTreeSearchParamHybrid(radius=5 * voxel, max_nn=100))`` after
``estimate_normals(KDTreeSearchParamHybrid(radius=2 * voxel, max_nn=30))``, i.e. open3d 0.10's
ComputeFPFHFeature (ComputePairFeatures, ComputeSPFHFeature, ComputeFPFHFeature), in float64.

PARITY UNPINNED: open3d is not installable offline, so this restates its published algorithm and pins the
conventions the GPU kernels (csrc/fpfh.cu, dgr_compute_fpfh) follow:

* search: oracle.normals.neighbours as it is - rows strictly within the radius, the point itself included,
  d^2 = (ex ex + ey ey) + ez ez, the max_nn smallest by (d^2, row), max_nn counting the point itself;
* self: open3d skips the first hit as the query point; with one point per cell that is row i, which is dropped.
  m = the neighbours left; a point with m = 0 gets all-zero SPFH and FPFH rows;
* pair feature of (p1, n1) = (p_i, n_i), (p2, n2) = (p_j, n_j): d = p2 - p1 ((0, 0, 0) when |d| = 0);
  a1 = n1.d / |d|, a2 = n2.d / |d|; if acos|a1| > acos|a2| swap n1 / n2, d = -d, theta = -a2, else theta = a1;
  v = d x n1 ((0, 0, 0) when |v| = 0), v /= |v|; w = n1 x v; phi = v.n2; alpha = atan2(w.n2, n1.n2);
* SPFH: 33 bins, alpha -> floor(11 (alpha + pi) / 2 pi), phi -> 11 + floor(11 (phi + 1) / 2),
  theta -> 22 + floor(11 (theta + 1) / 2), each clamped to [0, 10] within its group; every pair adds
  hist_incr = 100 / m to its three bins by repeated addition (all addends are equal, so the order of the pairs
  does not matter); a degenerate pair lands in bins 5, 16, 27;
* FPFH (m > 0): over the neighbours in (d^2, row) order, skipping d^2 = 0, val = spfh[k][j] / d^2_k is added to
  f[j] and to sum[j / 11] (neighbour-major, then j); s_g = 100 / sum[g] where sum[g] != 0; then
  f[j] = f[j] s_{j/11} + spfh[i][j] (only + spfh[i][j] where the group's sum is 0);
* ambiguity band: a pair feature is ambiguous when a scaled feature lies within 1e-9 bin units of a bin edge (the
  integers 0 .. 11, which counts the +-pi wrap of alpha), when |a1| and |a2| are within 1e-12 (the swap test) while
  n2 != +-n1, or when |v| < 1e-12 |d|.  (Where n2 = +-n1 exactly, |a1| and |a2| are the same number however the dot
  products round, so no implementation swaps: voxelised scans hold many such pairs, and flagging them would mark
  most FPFH rows ambiguous.)  A point's SPFH is ambiguous when any of its pairs is; its FPFH when its own SPFH or the
  SPFH of any kept neighbour is.  Outside the band the bins do not depend on libm's last bits, so the GPU's rows
  equal these rounded to float32 bit for bit.
"""
import numpy as np

from .normals import neighbours

BINS = 11
DIM = 3 * BINS
EDGE_BAND = 1e-9
SWAP_BAND = 1e-12
CROSS_BAND = 1e-12


def _cross(a, b):
  return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                   a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
  return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def pair_features(p1, n1, p2, n2):
  """ComputePairFeatures over arrays [..., 3] -> (alpha, phi, theta, ambiguous), float64 [...] each."""
  p1, n1, p2, n2 = (np.asarray(a, np.float64) for a in (p1, n1, p2, n2))
  d = p2 - p1
  dn = np.sqrt(_dot(d, d))
  live = dn != 0.0
  safe = np.where(live, dn, 1.0)
  a1, a2 = _dot(n1, d) / safe, _dot(n2, d) / safe
  swap = np.arccos(np.abs(a1)) > np.arccos(np.abs(a2))
  m1 = np.where(swap[..., None], n2, n1)
  m2 = np.where(swap[..., None], n1, n2)
  d = np.where(swap[..., None], -d, d)
  theta = np.where(swap, -a2, a1)
  v = _cross(d, m1)
  vn = np.sqrt(_dot(v, v))
  live &= vn != 0.0
  v = v / np.where(vn != 0.0, vn, 1.0)[..., None]
  w = _cross(m1, v)
  phi = _dot(v, m2)
  alpha = np.arctan2(_dot(w, m2), _dot(m1, m2))
  alpha, phi, theta = (np.where(live, x, 0.0) for x in (alpha, phi, theta))
  # n2 = +-n1 component for component gives |a1| = |a2| exactly on every implementation: no swap anywhere
  same = np.all(n1 == n2, -1) | np.all(n1 == -n2, -1)
  amb = (np.abs(np.abs(a1) - np.abs(a2)) <= SWAP_BAND) & ~same
  amb |= vn < CROSS_BAND * dn
  for s in scaled(alpha, phi, theta):
    amb |= np.abs(s - np.round(s)) <= EDGE_BAND
  return alpha, phi, theta, amb & (dn != 0.0)


def scaled(alpha, phi, theta):
  """The three features in bin units (before the floor)."""
  return 11.0 * (alpha + np.pi) / (2.0 * np.pi), 11.0 * (phi + 1.0) * 0.5, 11.0 * (theta + 1.0) * 0.5


def bins(alpha, phi, theta):
  """-> int [..., 3]: the bin of each feature in 0 .. 32 (groups of 11, clamped within the group)."""
  out = [np.clip(np.floor(s), 0, BINS - 1).astype(np.int64) + BINS * g
         for g, s in enumerate(scaled(alpha, phi, theta))]
  return np.stack(out, -1)


def _repeated_sum(incr, count):
  """incr added count times to +0.0, one addition at a time (float64 [n], int [n, 33] -> [n, 33])."""
  out = np.zeros(count.shape)
  for step in range(int(count.max(initial=0))):
    out = np.where(count > step, out + incr[:, None], out)
  return out


def neighbour_lists(xyz, radius, max_nn):
  """-> (nb int [n, max(max_nn - 1, 1)] (-1 padded) in (d^2, row) order without row i, d2 float64 likewise,
  m int [n], counts within the radius int [n])."""
  xyz = np.asarray(xyz, np.float64)
  lists, counts = neighbours(xyz, radius, max_nn)
  K = max(max_nn - 1, 1)
  nb = np.full((len(xyz), K), -1, np.int64)
  d2 = np.zeros((len(xyz), K))
  m = np.zeros(len(xyz), np.int64)
  for i, rows in enumerate(lists):
    rows = rows[rows != i]
    m[i] = len(rows)
    nb[i, :len(rows)] = rows
    e = xyz[rows] - xyz[i]
    d2[i, :len(rows)] = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
  return nb, d2, m, counts


def compute_fpfh(xyz, normals, radius, max_nn):
  """-> dict(fpfh float64 [n, 33], spfh float64 [n, 33], counts int [n], m int [n], ambiguous bool [n] (FPFH),
  spfh_ambiguous bool [n], nb, d2)."""
  xyz = np.asarray(xyz, np.float64)
  nrm = np.asarray(normals, np.float64)
  n = len(xyz)
  nb, d2, m, counts = neighbour_lists(xyz, radius, max_nn)
  valid = nb >= 0
  I, K = np.nonzero(valid)
  J = nb[I, K]
  alpha, phi, theta, amb = pair_features(xyz[I], nrm[I], xyz[J], nrm[J])
  b = bins(alpha, phi, theta)
  count = np.zeros((n, DIM), np.int64)
  for g in range(3):
    np.add.at(count, (I, b[:, g]), 1)
  incr = np.where(m > 0, 100.0 / np.maximum(m, 1), 0.0)
  spfh = _repeated_sum(incr, count)
  spfh_amb = np.zeros(n, bool)
  np.logical_or.at(spfh_amb, I, amb)
  # FPFH: neighbour-major, then bin, as open3d's loop
  f = np.zeros((n, DIM))
  s = np.zeros((n, 3))
  for k in range(nb.shape[1]):
    use = valid[:, k] & (d2[:, k] != 0.0)
    if not use.any():
      continue
    rows = spfh[np.where(use, nb[:, k], 0)]
    dist = np.where(use, d2[:, k], 1.0)
    for j in range(DIM):
      val = rows[:, j] / dist
      f[:, j] = np.where(use, f[:, j] + val, f[:, j])
      s[:, j // BINS] = np.where(use, s[:, j // BINS] + val, s[:, j // BINS])
  scale = np.where(s != 0.0, 100.0 / np.where(s != 0.0, s, 1.0), 0.0)
  for j in range(DIM):
    g = j // BINS
    f[:, j] = np.where(s[:, g] != 0.0, f[:, j] * scale[:, g] + spfh[:, j], f[:, j] + spfh[:, j])
  f[m == 0] = 0.0
  amb = spfh_amb | (valid & spfh_amb[np.where(valid, nb, 0)]).any(1)
  return dict(fpfh=f, spfh=spfh, counts=counts, m=m, ambiguous=amb, spfh_ambiguous=spfh_amb, nb=nb, d2=d2)
