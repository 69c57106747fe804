"""oracle/normals.py and oracle/icp_plane.py (the float64 restatements of open3d's EstimateNormals with a hybrid search
and point-to-plane ICP) on known answers, and the open3d stand-in's argument checks for both, which raise before a
device is needed."""
import types

import numpy as np
import pytest

from deepglobalregistration_b200 import synthetic as syn
from oracle import icp_plane as oip
from oracle import normals as onm


def grid(n=12, pitch=0.1, seed=0, jitter=0.02):
  g = np.random.default_rng(seed)
  x, y = np.meshgrid(np.arange(n) * pitch, np.arange(n) * pitch)
  P = np.stack([x.ravel(), y.ravel(), np.zeros(n * n)], 1)
  P[:, :2] += g.uniform(-jitter, jitter, size=(n * n, 2))
  return P


def test_plane_sphere_and_isolated_point():
  nrm, counts, _ = onm.estimate_normals(grid(), 0.25, 30)
  assert np.array_equal(nrm, np.tile([0.0, 0.0, 1.0], (len(nrm), 1))) and counts.min() >= 3
  tilted = grid() @ syn.random_se3(np.random.default_rng(1), 40.0, 0.0)[:3, :3].T
  nrm_t, _, _ = onm.estimate_normals(tilted, 0.25, 30)
  axis = np.cross(tilted[1] - tilted[0], tilted[20] - tilted[0])
  axis /= np.linalg.norm(axis)
  assert np.all(np.abs(nrm_t @ axis) > 1 - 1e-12)
  k = np.arange(2000) + 0.5                                           # Fibonacci sphere, radius 1
  phi, th = np.arccos(1 - 2 * k / 2000), np.pi * (1 + 5 ** 0.5) * k
  S = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
  nrm_s, _, _ = onm.estimate_normals(S, 0.2, 30)
  assert np.all(np.abs((nrm_s * S).sum(1)) > 1 - 1e-3)               # within ~2.5 degrees of radial
  lone = np.vstack([grid(4), [[5.0, 5.0, 5.0]], [[5.05, 5.0, 5.0]]])
  nrm_l, counts_l, eig = onm.estimate_normals(lone, 0.2, 30)
  assert np.array_equal(nrm_l[-2:], [[0, 0, 1], [0, 0, 1]]) and list(counts_l[-2:]) == [2, 2]
  assert np.array_equal(eig[-2:], np.zeros((2, 3)))


def test_truncation_order_and_strict_radius():
  # around the origin: rows at d^2 = 0.25 (rows 1, 2: a tie), 0.09, 0.49, and one exactly on the radius
  P = np.array([[0, 0, 0], [0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.3], [0, -0.7, 0], [1.0, 0, 0]], np.float64)
  nb, counts = onm.neighbours(P, 1.0, 64)
  assert counts[0] == 5 and list(nb[0]) == [0, 3, 1, 2, 4]               # (d^2, row); row 5 at d = radius is out
  nb3, counts3 = onm.neighbours(P, 1.0, 3)
  assert counts3[0] == 5 and list(nb3[0]) == [0, 3, 1]
  nb4, _ = onm.neighbours(P, 1.0, 4)
  assert list(nb4[0]) == [0, 3, 1, 2]                                  # of the tie, the lower row first
  _, c_out, _ = onm.estimate_normals(P, np.nextafter(0.3, 0.0), 64)
  assert c_out[0] == 1                                                 # d = 0.3 is not < 0.3 - 1 ulp


def test_orientation_against_previous_normals():
  P = grid()
  nrm, _, _ = onm.estimate_normals(P, 0.25, 30)
  prev = np.tile([0.1, 0.0, -1.0], (len(P), 1))
  flipped, _, _ = onm.estimate_normals(P, 0.25, 30, prev=prev)
  assert np.array_equal(flipped, -nrm)
  kept, _, _ = onm.estimate_normals(P, 0.25, 30, prev=-prev)
  assert np.array_equal(kept, nrm)


def room_copy(deg=3.0, cm=3.0, seed=0):
  vs = 0.0625
  x = syn.room_scan(3, 20000, (1.8, 1.5, 1.25), scene_seed=1) - np.array([0.9, 0.75, 0.625])
  _, first = np.unique(np.floor(x / vs).astype(np.int64), axis=0, return_index=True)
  P = x[np.sort(first)]
  g = np.random.default_rng(seed)
  T = syn.random_se3(g, deg, 0.0)
  T[:3, 3] = g.normal(size=3) * cm / 100 / np.sqrt(3)
  return P, syn.apply_se3(T, P), T, vs


def test_point_to_plane_converges_on_a_rigid_copy():
  P, Q, T_gt, vs = room_copy()
  nrm, _, _ = onm.estimate_normals(Q, 2 * vs, 30)
  T, info = oip.icp_point_to_plane(P, Q, nrm, 2 * vs)
  te, re = syn.rte_rre(T, T_gt)
  assert te < 1e-6 and re < 1e-6, (te, re, info)
  assert info['fitness'] == 1.0 and info['inlier_rmse'] < 1e-6 and 0 < info['iterations'] < 30
  assert info['solves_failed'] == 0
  T1, info1 = oip.icp_point_to_plane(P, Q, nrm, 2 * vs, max_iter=1)
  assert info1['iterations'] == 1 and syn.rte_rre(T1, T_gt)[1] < syn.rte_rre(np.eye(4), T_gt)[1]


def test_single_plane_uses_the_identity_update():
  tgt = grid(10)
  src = tgt + np.array([0.01, -0.02, 0.05])
  nrm = np.tile([0.0, 0.0, 1.0], (len(tgt), 1))
  T, info = oip.icp_point_to_plane(src, tgt, nrm, 0.1)
  assert np.all(np.isfinite(T)) and info['solves_failed'] >= 1 and np.array_equal(T, np.eye(4))
  # no correspondence in range: the identity update, then the rule stops on unchanged fitness / RMSE
  T2, info2 = oip.icp_point_to_plane(src + 10.0, tgt, nrm, 0.1)
  assert np.array_equal(T2, np.eye(4)) and info2['iterations'] == 1 and info2['n_corr'] == 0
  T3, info3 = oip.icp_point_to_plane(np.zeros((0, 3)), tgt, nrm, 0.1)
  assert np.array_equal(T3, np.eye(4)) and info3['fitness'] == 0.0 and info3['iterations'] == 1


def test_rmse_is_euclidean():
  tgt = grid(10, jitter=0.0)
  src = tgt + np.array([0.03, 0.0, 0.0])                               # point-to-plane residuals are all 0
  nrm = np.tile([0.0, 0.0, 1.0], (len(tgt), 1))
  _, info = oip.icp_point_to_plane(src, tgt, nrm, 0.05, max_iter=0)
  assert info['fitness'] == 1.0 and abs(info['inlier_rmse'] - 0.03) < 1e-12 and info['iterations'] == 0


def test_cholesky_step_and_update_match_numpy():
  g = np.random.default_rng(5)
  M = g.normal(size=(20, 6))
  A, b = M.T @ M, g.normal(size=6)
  np.testing.assert_allclose(oip.cholesky_step(A, b), -np.linalg.solve(A, b), rtol=1e-10)
  assert oip.cholesky_step(np.zeros((6, 6)), b) is None
  U = oip.zyx_update(np.array([0.1, -0.2, 0.3, 1.0, 2.0, 3.0]))
  assert np.allclose(U[:3, :3] @ U[:3, :3].T, np.eye(3), atol=1e-15) and np.array_equal(U[:3, 3], [1, 2, 3])


# ---- the open3d stand-in: names and argument checks (no device needed) ----------------------------------------
def test_stand_in_names_under_every_module_path():
  from deepglobalregistration_b200 import o3d_registration as reg
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  for mod in (o3d.pipelines.registration, o3d.registration):
    assert mod.TransformationEstimationPointToPlane is reg.TransformationEstimationPointToPlane
    assert mod.TransformationEstimationPointToPoint is reg.TransformationEstimationPointToPoint
  for name in ('KDTreeSearchParamHybrid', 'KDTreeSearchParamKNN', 'KDTreeSearchParamRadius'):
    assert getattr(o3d.geometry, name) is getattr(reg, name) and getattr(o3d, name) is getattr(reg, name)
  p = o3d.KDTreeSearchParamHybrid(radius=0.1, max_nn=30)
  assert (p.radius, p.max_nn) == (0.1, 30)


def test_stand_in_argument_checks():
  from deepglobalregistration_b200 import io as dio
  from deepglobalregistration_b200 import o3d_registration as reg
  with pytest.raises(NotImplementedError):
    reg.TransformationEstimationPointToPlane(object())                 # a robust kernel (open3d >= 0.12)
  pcd = dio.PointCloud(grid())
  for param in (reg.KDTreeSearchParamKNN(30), reg.KDTreeSearchParamRadius(0.1)):
    with pytest.raises(NotImplementedError):
      pcd.estimate_normals(param)
  for bad in (reg.KDTreeSearchParamHybrid(0.1, 65), reg.KDTreeSearchParamHybrid(0.1, 0),
              reg.KDTreeSearchParamHybrid(0.0, 30)):
    with pytest.raises(ValueError):
      pcd.estimate_normals(bad)
  assert pcd.normals is None and not pcd.has_normals()
  with pytest.raises(RuntimeError, match='estimate_normals'):
    reg.registration_icp(pcd, dio.PointCloud(grid()), 0.1, np.eye(4), reg.TransformationEstimationPointToPlane())
  with pytest.raises(RuntimeError, match='estimate_normals'):
    reg.registration_icp(pcd, grid(), 0.1, np.eye(4), reg.TransformationEstimationPointToPlane())
  with pytest.raises(NotImplementedError):
    reg.registration_icp(pcd, pcd, 0.1, np.eye(4), object())


def test_transform_rotates_normals():
  from deepglobalregistration_b200 import io as dio
  pcd = dio.PointCloud(grid())
  T = syn.random_se3(np.random.default_rng(2), 40.0, 0.5)
  pcd.transform(T)
  assert pcd.normals is None
  pcd.normals = np.tile([0.0, 0.0, 1.0], (len(pcd), 1))
  pcd.transform(T)
  assert np.allclose(pcd.normals, np.tile(T[:3, 2], (len(pcd), 1)), atol=1e-15)


def test_icp_baseline_arguments_and_branch_codes():
  from deepglobalregistration_b200 import sharding
  from deepglobalregistration_b200.core.icp_baseline import ICPBaseline
  dgr = types.SimpleNamespace(voxel_size=0.05)
  b = ICPBaseline(dgr)
  assert b.method == 'point_to_plane' and b._distance() == 0.1 and b.max_iteration == 30
  assert np.array_equal(b.init, np.eye(4))
  assert ICPBaseline(dgr, 'point_to_point', 0.2)._distance() == 0.2
  for kw in (dict(max_correspondence_distance=0.21), dict(max_correspondence_distance=0.0), dict(max_iteration=-1),
             dict(method='colored')):
    with pytest.raises(ValueError):
      ICPBaseline(dgr, **kw)
  assert sharding.BRANCH_CODE['icp'] == 4.0 and sharding.BRANCH_CODE['icp_plane'] == 5.0
  assert sharding.BRANCH_CODE['fgr'] == 3.0 and sharding.BRANCH_CODE[None] == -1.0
