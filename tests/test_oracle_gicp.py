"""oracle/gicp.py (open3d's generalized ICP, per-point covariances and robust losses) on known answers, and the host
side of the feature: the stand-in's names and the checks it makes before needing a device, PointCloud covariances
and the new C declarations.  No GPU."""
import ctypes

import numpy as np
import pytest

from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import synthetic as syn
from oracle import gicp as og
from oracle import icp as oicp
from oracle import normals as onm

GICP_EPSILON = 1e-3

# the LiDAR case: lidar_pair(0) with the sensors LIDAR_ADVANCE apart, both scans voxelised at LIDAR_VOXEL, ICP at
# 2 voxels from a start LIDAR_START (deg, m) off the truth.  Measured with the oracles (seed 0): point-to-point ICP
# leaves 0.0052 m, generalized ICP on covariances from normals 0.0067 m.  At this voxel size the scene does NOT show
# generalized ICP beating point-to-point ICP; both numbers are pinned as measured.
LIDAR_VOXEL = 0.3
LIDAR_ADVANCE = 3.0
LIDAR_START = (2.0, 0.3)
LIDAR_P2P_LEFT = 0.0052
LIDAR_GICP_LEFT = 0.0067

# the outlier case: room_pair(0) at OUTLIER_VOXEL, plus a ghost copy of the source's x = max wall moved
# OUTLIER_GHOST inwards (0.6 max_dist), point-to-plane ICP at 2 voxels.  Measured with the oracle: L2 is pulled
# 0.0090 m, TukeyLoss(0.02) leaves 0.00025 m
OUTLIER_VOXEL = 0.05
OUTLIER_GHOST = 0.06
OUTLIER_TUKEY_K = 0.02
OUTLIER_L2_PULLED = 0.006          # L2 leaves at least this much
OUTLIER_TUKEY_LEFT = 0.001         # Tukey leaves at most this much


def voxelise(x, cell):
  """float32-representable points, the first per cell of size `cell`."""
  x32 = np.asarray(x, np.float32).astype(np.float64)
  _, first = np.unique(np.floor(x32 / cell).astype(np.int64), axis=0, return_index=True)
  return x32[np.sort(first)]


def lidar_case(seed=0):
  """-> (S, Q, T_gt, T_init, vs) of the LiDAR case."""
  x0, x1, T = syn.lidar_pair(0, advance=LIDAR_ADVANCE)
  S, Q = voxelise(x0, LIDAR_VOXEL), voxelise(x1, LIDAR_VOXEL)
  T0 = syn.random_se3(np.random.default_rng(seed), *LIDAR_START) @ T
  return S, Q, T, T0, LIDAR_VOXEL


def outlier_case(seed=0):
  """-> (source with its ghost wall, Q, T_gt, T_init, vs) of the outlier case."""
  vs = OUTLIER_VOXEL
  x0, x1, T = syn.room_pair(0, n_raw=60000)
  S, Q = voxelise(x0, vs), voxelise(x1, vs)
  wall = S[:, 0] > S[:, 0].max() - 0.02
  Sg = np.concatenate([S, S[wall] - [OUTLIER_GHOST, 0.0, 0.0]]).astype(np.float32).astype(np.float64)
  T0 = syn.random_se3(np.random.default_rng(seed), 2.0, 0.02) @ T
  return Sg, Q, T, T0, vs


# ---------------------------------------------------------------------------------------------------------------
# losses and covariances
# ---------------------------------------------------------------------------------------------------------------
def test_loss_weights():
  w = og.loss_weight
  r = np.array([-2.0, -0.5, 0.0, 0.25, 0.5, 1.0, 3.0])
  assert np.array_equal(w(None, r), np.ones(7)) and np.array_equal(w(('L2', 1.0), r), np.ones(7))
  assert np.array_equal(w(('L1', 1.0), r), [0.5, 2.0, 0.0, 4.0, 2.0, 1.0, 1 / 3])          # 0 at r = 0 (pinned)
  assert np.array_equal(w(('Huber', 0.5), r), [0.25, 1.0, 1.0, 1.0, 1.0, 0.5, 0.5 / 3])    # |r| = k: 1
  assert np.allclose(w(('Cauchy', 0.5), r), 1.0 / (1.0 + (r / 0.5) ** 2), rtol=1e-15)
  assert w(('Cauchy', 0.5), [0.5])[0] == 0.5
  assert np.allclose(w(('GM', 0.5), r), 0.5 / (0.5 + r * r) ** 2, rtol=1e-15)
  assert w(('GM', 0.5), [0.0])[0] == 2.0
  tk = w(('Tukey', 1.0), r)
  assert tk[5] == 0.0 and tk[0] == 0.0 and tk[6] == 0.0                                     # |r| = k and beyond: 0
  assert tk[2] == 1.0 and tk[4] == (1 - 0.25) ** 2 and tk[1] == tk[4]


def test_covariances_match_brute_force():
  g = np.random.default_rng(0)
  P = voxelise(g.uniform(0.0, 1.0, size=(3000, 3)), 0.05)
  far = np.array([[5.0, 5.0, 5.0], [5.01, 5.0, 5.0]])                  # two isolated points: fewer than 3 neighbours
  P = np.concatenate([P, far])
  radius, max_nn = 0.1, 10
  cov, counts = og.estimate_covariances(P, radius, max_nn)
  nbrs, c2 = onm.neighbours(P, radius, max_nn)
  assert np.array_equal(counts, c2) and (counts > max_nn).any()
  for i in range(len(P)):
    if len(nbrs[i]) >= 3:
      assert np.allclose(cov[i], np.cov(P[nbrs[i]].T, bias=True), rtol=0, atol=1e-15)
    else:
      assert np.array_equal(cov[i], np.eye(3))
  assert np.array_equal(counts[-2:], [2, 2]) and np.array_equal(cov[-2:], np.tile(np.eye(3), (2, 1, 1)))


def test_covariances_from_normals():
  g = np.random.default_rng(1)
  n = g.normal(size=(4000, 3))
  n /= np.linalg.norm(n, axis=1, keepdims=True)
  lit, closed = og.covariances_from_normals(n, GICP_EPSILON), og.covariances_from_normals_closed(n, GICP_EPSILON)
  ok = n[:, 0] >= -0.99
  # the Rodrigues form divides by 1 + c: 1e-15 relative to that factor
  err = np.abs(lit - closed).max(axis=(1, 2))
  assert np.all(err[ok] <= 1e-15 / (1.0 + n[ok, 0])), (err[ok] * (1.0 + n[ok, 0])).max()
  assert np.all(err[ok & (n[:, 0] >= 0)] <= 1e-15)
  # the branch: c < -0.99 gives diag(eps, 1, 1) whatever the normal
  branch = np.array([[-1.0, 0.0, 0.0], [-0.995, np.sqrt(1 - 0.995 ** 2), 0.0]])
  assert np.array_equal(og.rotation_e1_to_x(branch[1]), np.diag([-1.0, -1.0, 1.0]))
  assert np.array_equal(og.covariances_from_normals(branch, GICP_EPSILON),
                        np.tile(np.diag([GICP_EPSILON, 1.0, 1.0]), (2, 1, 1)))
  assert np.abs(og.covariances_from_normals_closed(branch, GICP_EPSILON)[1] -
                np.diag([GICP_EPSILON, 1.0, 1.0])).max() > 1e-3             # the closed form differs there
  # a plane's covariance is flat along its normal
  C = og.covariances_from_normals([[0.0, 0.0, 1.0]], GICP_EPSILON)[0]
  assert np.allclose(C, np.diag([1.0, 1.0, GICP_EPSILON]), rtol=0, atol=1e-16)


def test_sym6_layout():
  g = np.random.default_rng(2)
  A = g.normal(size=(5, 3, 3))
  C = A @ A.transpose(0, 2, 1)
  assert np.array_equal(og.full33(og.sym6(C)), C)


# ---------------------------------------------------------------------------------------------------------------
# generalized ICP and the weighted estimators
# ---------------------------------------------------------------------------------------------------------------
def test_generalized_icp_rigid_copy():
  x0, _, T = syn.room_pair(0, n_raw=20000, rigid_copy=True)
  vs = 0.0625
  S = voxelise(x0, vs)
  Q = S @ T[:3, :3].T + T[:3, 3]
  C_s = og.covariances_from_normals(onm.estimate_normals(S, 2 * vs, 30)[0], GICP_EPSILON)
  C_q = og.covariances_from_normals(onm.estimate_normals(Q, 2 * vs, 30)[0], GICP_EPSILON)
  T0 = syn.random_se3(np.random.default_rng(1), 3.0, 0.03) @ T
  Tg, info = og.generalized_icp(S, C_s, Q, C_q, 2 * vs, T0, max_iter=60, rel_fitness=0.0, rel_rmse=0.0)
  assert np.abs(Tg - T).max() <= 1e-9, np.abs(Tg - T).max()
  assert info['fitness'] == 1.0 and info['rows_skipped'] == 0


def test_l2_kernel_is_no_kernel():
  Sg, Q, T, T0, vs = outlier_case()
  nQ = onm.estimate_normals(Q, 2 * vs, 30)[0]
  Ta, ia = og.icp_point_to_plane(Sg, Q, nQ, 2 * vs, T0, max_iter=5)
  Tb, ib = og.icp_point_to_plane(Sg, Q, nQ, 2 * vs, T0, kernel=('L2', 1.0), max_iter=5)
  assert ia['iterations'] == ib['iterations'] and np.abs(Ta - Tb).max() <= 1e-12


def test_cholesky_failure_adds_no_row():
  M = np.stack([np.eye(3), np.diag([1.0, 0.0, 1.0]), np.diag([1.0, 1.0, -1e-20])])
  assert np.array_equal(og.cholesky3_ok(M), [True, False, False])
  P = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
  zero = np.zeros((3, 3, 3))                                          # M = 0 for every pair: no row at all
  Tg, info = og.generalized_icp(P, zero, P + 0.01, zero, 0.1, max_iter=3)
  assert info['n_corr'] == 3 and info['fitness'] == 1.0 and info['rows_skipped'] == 3
  assert info['solves_failed'] == 1 and np.array_equal(Tg, np.eye(4))


def test_lidar_case():
  S, Q, T, T0, vs = lidar_case()
  C_s = og.covariances_from_normals(onm.estimate_normals(S, 2 * vs, 30)[0], GICP_EPSILON)
  C_q = og.covariances_from_normals(onm.estimate_normals(Q, 2 * vs, 30)[0], GICP_EPSILON)
  Tg, _ = og.generalized_icp(S, C_s, Q, C_q, 2 * vs, T0)
  Tp, _ = oicp.icp_point_to_point(S, Q, 2 * vs, T0)
  te_g, te_p = syn.rte_rre(Tg, T)[0], syn.rte_rre(Tp, T)[0]
  print(f'LiDAR: start {syn.rte_rre(T0, T)[0]:.4f} m, point-to-point leaves {te_p:.4f} m, generalized {te_g:.4f} m')
  assert abs(te_p - LIDAR_P2P_LEFT) <= 1e-4 and abs(te_g - LIDAR_GICP_LEFT) <= 1e-4


def test_outlier_case():
  Sg, Q, T, T0, vs = outlier_case()
  nQ = onm.estimate_normals(Q, 2 * vs, 30)[0]
  T2, _ = og.icp_point_to_plane(Sg, Q, nQ, 2 * vs, T0)
  Tt, _ = og.icp_point_to_plane(Sg, Q, nQ, 2 * vs, T0, kernel=('Tukey', OUTLIER_TUKEY_K))
  left2, leftt = syn.rte_rre(T2, T)[0], syn.rte_rre(Tt, T)[0]
  print(f'ghost wall: L2 leaves {left2:.4f} m, Tukey {leftt:.5f} m')
  assert left2 >= OUTLIER_L2_PULLED and leftt <= OUTLIER_TUKEY_LEFT


# ---------------------------------------------------------------------------------------------------------------
# host side
# ---------------------------------------------------------------------------------------------------------------
NEW_NAMES = ('TransformationEstimationForGeneralizedICP', 'registration_generalized_icp', 'estimate_covariances',
             'L2Loss', 'L1Loss', 'HuberLoss', 'CauchyLoss', 'GMLoss', 'TukeyLoss')


def test_stand_in_names():
  from deepglobalregistration_b200 import o3d_registration as reg
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  for mod in (o3d.pipelines.registration, o3d.registration):
    for name in NEW_NAMES:
      assert getattr(mod, name) is getattr(reg, name), name


def test_stand_in_losses_and_estimators():
  from deepglobalregistration_b200 import _abi
  from deepglobalregistration_b200 import o3d_registration as reg
  for cls, k in ((reg.L2Loss, None), (reg.L1Loss, None), (reg.HuberLoss, 0.1), (reg.CauchyLoss, 0.2),
                 (reg.GMLoss, 0.3), (reg.TukeyLoss, 0.4)):
    loss = cls() if k is None else cls(k)
    assert loss.loss in _abi.LOSS_IDS and loss.k == (1.0 if k is None else k)
    for est in (reg.TransformationEstimationPointToPlane(loss), reg.TransformationEstimationForColoredICP(kernel=loss),
                reg.TransformationEstimationForGeneralizedICP(kernel=loss)):
      assert est.kernel is loss
  assert reg._loss_args(None) == (None, 1.0) and reg._loss_args(reg.TukeyLoss(0.5)) == ('Tukey', 0.5)
  for cls in (reg.HuberLoss, reg.CauchyLoss, reg.GMLoss, reg.TukeyLoss):
    for k in (0.0, -1.0, float('nan'), float('inf')):
      with pytest.raises(ValueError):
        cls(k)
  with pytest.raises(NotImplementedError):
    reg.TransformationEstimationPointToPlane(object())
  with pytest.raises(NotImplementedError):
    reg.TransformationEstimationForGeneralizedICP(kernel=object())
  est = reg.TransformationEstimationForGeneralizedICP()
  assert est.epsilon == 1e-3 and est.kernel is None
  for eps in (0.0, -1e-3, float('nan'), float('inf')):
    with pytest.raises(ValueError):
      reg.TransformationEstimationForGeneralizedICP(eps)


def test_stand_in_checks_before_any_device():
  from deepglobalregistration_b200 import o3d_registration as reg
  pts = np.random.default_rng(0).normal(size=(20, 3))
  src, tgt = dio.PointCloud(pts), dio.PointCloud(pts)
  with pytest.raises(RuntimeError, match='covariances or normals on the source'):
    reg.registration_generalized_icp(src, tgt, 0.1, np.eye(4))
  src.normals = np.tile([0.0, 0.0, 1.0], (20, 1))
  with pytest.raises(RuntimeError, match='covariances or normals on the target'):
    reg.registration_generalized_icp(src, tgt, 0.1, np.eye(4))
  with pytest.raises(RuntimeError, match='estimate_covariances'):
    reg.registration_icp(src, tgt, 0.1, np.eye(4), reg.TransformationEstimationForGeneralizedICP())
  with pytest.raises(NotImplementedError):
    reg.registration_generalized_icp(src, tgt, 0.1, np.eye(4), reg.TransformationEstimationPointToPlane())
  with pytest.raises(ValueError):
    reg.registration_generalized_icp(src, tgt, 0.0, np.eye(4))
  for param in (reg.KDTreeSearchParamKNN(30), reg.KDTreeSearchParamRadius(0.1)):
    with pytest.raises(NotImplementedError):
      reg.estimate_covariances(pts, param)
  with pytest.raises(ValueError):
    reg.estimate_covariances(pts, reg.KDTreeSearchParamHybrid(0.1, 65))
  with pytest.raises(NotImplementedError):
    dio.PointCloud(pts).estimate_covariances()
  with pytest.raises(NotImplementedError):
    dio.PointCloud(pts).estimate_covariances(reg.KDTreeSearchParamKNN(30))


def test_point_cloud_covariances():
  g = np.random.default_rng(3)
  pts = g.normal(size=(6, 3))
  pcd = dio.PointCloud(pts)
  assert pcd.covariances is None and not pcd.has_covariances()
  A = g.normal(size=(6, 3, 3))
  C = A @ A.transpose(0, 2, 1)
  pcd.covariances = C
  assert pcd.has_covariances() and pcd.covariances.dtype == np.float64
  with pytest.raises(ValueError):
    pcd.covariances = np.zeros((6, 6))
  T = syn.random_se3(np.random.default_rng(4), 40.0, 1.0)
  pcd.transform(T)
  R = T[:3, :3]
  assert np.allclose(pcd.covariances, R @ C @ R.T, rtol=0, atol=1e-12)
  assert np.allclose(pcd.points, pts @ R.T + T[:3, 3], rtol=0, atol=1e-12)
  pcd.covariances = C[:5]                                          # open3d's rule: one per point
  assert not pcd.has_covariances()


def test_gicp_declarations():
  from deepglobalregistration_b200 import _abi
  p, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
  D = _abi.DECLARATIONS
  assert D['dgr_estimate_covariances'] == (i32, [p, i64, p, p, p, i64, i32, f64, f64, i32, p, p, p])
  assert D['dgr_covariances_from_normals'] == (i32, [p, i64, f64, p, p])
  assert D['dgr_generalized_icp'] == (i32, [p, p, i64, p, p, p, p, p, i64, i32, f64, f64, i32, f64, p, i32, f64, f64,
                                            p, p, p])
  assert D['dgr_icp_loss'] == (i32, [p, i64, p, p, p, p, p, i64, i32, f64, f64, i32, f64, p, i32, f64, f64, p, p, p])
  assert D['dgr_colored_icp_loss'] == (i32, [p, p, i64, p, p, p, p, p, p, p, i64, i32, f64, f64, f64, i32, f64, p, i32,
                                             f64, f64, p, p, p])
  assert _abi.LOSS_IDS == dict(L2=0, L1=1, Huber=2, Cauchy=3, GM=4, Tukey=5)


def test_branch_code_and_cli_method():
  from deepglobalregistration_b200 import evaluate, sharding
  from deepglobalregistration_b200.core.icp_baseline import METHODS
  assert sharding.BRANCH_CODE['icp_generalized'] == 9.0 and METHODS['generalized'] == 'icp_generalized'
  import argparse
  ap = argparse.ArgumentParser()
  evaluate.add_method_arguments(ap)
  assert ap.parse_args(['--weights', 'w', '--method', 'icp_generalized']).method == 'icp_generalized'
