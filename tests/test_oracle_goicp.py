"""oracle/goicp.py (Go-ICP) on the CPU: its distance transform against scipy's exact EDT, Go-ICP's rotation and
translation uncertainty bounds, and small searches on a restricted rotation domain."""
import math

import numpy as np
from scipy import ndimage
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from deepglobalregistration_b200 import synthetic as syn
from oracle import goicp as og


def goicp_case(seed, n_s=128, n_t=2000, angle_deg=90.0, extent=(3.6, 3.0, 2.5)):
  """(src fp32 [n_s, 3], tgt fp32 [n_t, 3], T_gt, angle-axis of T_gt): the source sampled from one scan of a room,
  the target from another scan of the same room, moved by a rotation of angle_deg about a random axis."""
  g = np.random.default_rng(seed)
  x = syn.room_scan(seed, 20000, extent, scene_seed=seed)
  y = syn.room_scan(seed + 100, 20000, extent, scene_seed=seed)
  axis = g.normal(size=3)
  rv = axis / np.linalg.norm(axis) * math.radians(angle_deg)
  T = np.eye(4)
  T[:3, :3] = Rotation.from_rotvec(rv).as_matrix()
  T[:3, 3] = g.uniform(-0.3, 0.3, 3)
  src = x[g.choice(len(x), n_s, replace=False)]
  tgt = syn.apply_se3(T, y[g.choice(len(y), n_t, replace=False)])
  return src.astype(np.float32), tgt.astype(np.float32), T, rv


def scipy_dt(dt, y32):
  occ = np.zeros((dt.G,) * 3, bool)
  c = dt.cells(y32)
  occ[c[:, 2], c[:, 1], c[:, 0]] = True
  return np.rint(ndimage.distance_transform_edt(~occ) ** 2).astype(np.int64)


def test_distance_transform_is_the_exact_edt():
  g = np.random.default_rng(0)
  clouds = [g.uniform(-1, 1, (300, 3)), np.zeros((1, 3)) + 0.3,
            np.array([[1.0, -1.0, 1.0], [-1.0, 1.0, 0.2], [0.0, 0.0, -1.0]])]    # touching the [-1, 1]^3 boundary
  for y in clouds:
    for G, e in ((32, 2.0), (37, 1.5), (16, 1.0)):
      dt = og.DistanceTransform(y.astype(np.float32), G, e)
      assert np.array_equal(dt.grid, scipy_dt(dt, y.astype(np.float32))), (len(y), G, e)
  # the lookup: zero in an occupied cell, h sqrt(stored) + the distance to the box outside it
  dt = og.DistanceTransform(np.zeros((1, 3), np.float32), 16, 1.0)
  q = np.array([[0.01, 0.01, 0.01], [3.0, 0.01, 0.01]], np.float32)
  v = dt.lookup(q)
  assert v[0] == 0.0 and abs(v[1] - (2.0 + dt.h32 * 7)) < 1e-5


def test_rotation_uncertainty_bound():
  """Go-ICP's Lemma: for r in a cube of half-width sigma around r0, angle(R_r x, R_r0 x) <= sqrt(3) sigma."""
  g = np.random.default_rng(1)
  for _ in range(200):
    sigma = g.uniform(0.01, 0.8)
    r0 = g.uniform(-math.pi, math.pi, 3)
    x = g.normal(size=3)
    R0 = og.rodrigues(r0)
    for r in r0 + g.uniform(-sigma, sigma, (20, 3)):
      a, b = og.rodrigues(r) @ x, R0 @ x
      ang = math.acos(np.clip(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)), -1, 1))
      assert ang <= SQRT3 * sigma + 1e-12


SQRT3 = math.sqrt(3.0)


def test_bounds_lower_bound_the_continuous_objective():
  """With the continuous distance to the occupied-cell centres in place of the lookup, the bound formulas
  lower-bound that objective at poses sampled inside random (rotation, translation) cube pairs."""
  src, tgt, _, _ = goicp_case(3, n_s=64, n_t=800)
  X, Y32, _, _, _ = og.normalise(src, tgt)
  dt = og.DistanceTransform(Y32, 32, 2.0)
  occ = np.argwhere(dt.grid == 0)[:, ::-1]                             # (x, y, z) cells
  tree = cKDTree((occ + 0.5) * float(dt.h32) - float(dt.e32))
  g = np.random.default_rng(2)
  for trim in (0.0, 0.3):
    K = max(1, int(math.floor(len(X) * (1 - trim))))
    for _ in range(30):
      sr, st = g.uniform(0.02, 0.5), g.uniform(0.01, 0.3)
      r0, t0 = g.uniform(-2, 2, 3), g.uniform(-0.5, 0.5, 3)
      Xr = og.rotate32(og.rodrigues(r0), X).astype(np.float64)
      e0 = tree.query(Xr + t0)[0]
      gam = 2 * math.sin(min(SQRT3 * sr / 2, math.pi / 2)) * og._norm(X)
      terms = np.maximum(e0 - gam - SQRT3 * st, 0) ** 2
      lb = np.sort(terms)[:K].sum()
      for _ in range(10):
        r, t = r0 + g.uniform(-sr, sr, 3), t0 + g.uniform(-st, st, 3)
        e = tree.query(X @ og.rodrigues(r).T + t)[0]
        assert lb <= np.sort(e ** 2)[:K].sum() * (1 + 1e-6) + 1e-9


def test_restricted_domain_search_recovers_the_pose():
  src, tgt, T_gt, rv = goicp_case(1)
  hw = math.pi / 4
  kw = dict(dt_size=64, rot_min=rv - hw, rot_width=2 * hw, cubes_per_round=8)
  T, info = og.goicp(src, tgt, **kw)
  te, re = syn.rte_rre(T, T_gt)
  assert info['converged'] == 1 and info['E'] - info['lb_min'] < info['eps'], info
  assert re < math.radians(2) and te < 0.02 * 3.6, (te, re)
  # a tiny inner pool: searches overflow and end early, the lower bounds stay sound (LB_min <= E*)
  _, small = og.goicp(src, tgt, max_rounds=3, inner_cap=8, **kw)
  assert small['inner_overflows'] > 0 and small['lb_min'] <= small['E'] and small['rounds'] == 3
