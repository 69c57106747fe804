"""oracle/colored_icp.py (open3d's colour gradient and colored ICP) on known answers, and the host side of colored ICP:
PointCloud colours, the PLY reader, the stand-in's argument forms and the checks it makes before needing a device,
multiway refinement's input checks and the two new C declarations.  No GPU."""
import ctypes

import numpy as np
import pytest

from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import synthetic as syn
from oracle import colored_icp as oc
from oracle import icp_plane as oip
from oracle import normals as onm

# the sliding wall: checker_wall(0) as target, checker_wall(1) as source, both voxelised at WALL_VOXEL, the source
# started WALL_SHIFT along the wall from the true pose (the identity).  Calibrated with the oracles: point-to-plane
# ICP leaves 0.032 m of the 0.036 m slide, colored ICP 0.0025 m
WALL_VOXEL = 0.04
WALL_SHIFT = (0.03, 0.02, 0.0)
WALL_P2PLANE_LEFT = 0.02          # point-to-plane leaves at least this much of the slide
WALL_COLORED_LEFT = 0.005         # colored ICP leaves at most this much


def voxelise(x, cell):
  """Rows of the float32-representable points, the first per cell (what a one-point-per-cell hash holds)."""
  x32 = np.asarray(x, np.float32).astype(np.float64)
  _, first = np.unique(np.floor(x32 / cell).astype(np.int64), axis=0, return_index=True)
  return np.sort(first)


def wall_case():
  """-> (P, I_P, Q, I_Q, target normals float32, T_init) with intensities as float32."""
  q, cq = syn.checker_wall(0)
  p, cp = syn.checker_wall(1)
  iq, ip = voxelise(q, WALL_VOXEL), voxelise(p, WALL_VOXEL)
  Q, P = q[iq].astype(np.float32).astype(np.float64), p[ip].astype(np.float32).astype(np.float64)
  nrm = onm.estimate_normals(Q, 2 * WALL_VOXEL, 30)[0].astype(np.float32)
  T0 = np.eye(4)
  T0[:3, 3] = WALL_SHIFT
  return P, oc.intensity(cp[ip]).astype(np.float32), Q, oc.intensity(cq[iq]).astype(np.float32), nrm, T0


def test_gradient_of_a_linear_intensity_on_a_plane():
  g = np.random.default_rng(0)
  xy = g.uniform(-0.5, 0.5, size=(2000, 2))
  P = np.concatenate([xy, np.zeros((2000, 1))], axis=1)
  a, b = 0.7, -1.3
  inten = a * P[:, 0] + b * P[:, 1] + 0.25
  nrm = np.tile([0.0, 0.0, 1.0], (len(P), 1))
  grad, counts, pivot = oc.color_gradient(P, nrm, inten, 0.08, 30)
  ok = counts >= 4
  assert ok.mean() > 0.99
  assert np.abs(grad[ok] - [a, b, 0.0]).max() <= 1e-12
  # a point with fewer than 4 neighbours (itself included) has no gradient
  far = np.array([[5.0, 5.0, 0.0], [5.01, 5.0, 0.0], [5.0, 5.01, 0.0]])
  P2 = np.concatenate([P, far])
  grad2, counts2, pivot2 = oc.color_gradient(P2, np.tile([0.0, 0.0, 1.0], (len(P2), 1)),
                                             a * P2[:, 0] + b * P2[:, 1], 0.08, 30)
  assert np.array_equal(counts2[-3:], [3, 3, 3]) and np.array_equal(grad2[-3:], np.zeros((3, 3)))
  assert np.array_equal(pivot2[-3:], np.zeros(3))


def test_solve3_matches_numpy_and_fails_on_a_singular_system():
  g = np.random.default_rng(1)
  M = g.normal(size=(3, 3))
  A = M @ M.T + 0.1 * np.eye(3)
  b = g.normal(size=3)
  x, piv = oc.solve3(A, b)
  assert np.allclose(x, np.linalg.solve(A, b), rtol=1e-12, atol=0) and piv > 0
  x, piv = oc.solve3(np.diag([1.0, 0.0, 1.0]), b)
  assert np.array_equal(x, np.zeros(3)) and piv <= 0


def test_lambda_one_is_point_to_plane():
  P, I_P, Q, I_Q, nrm, _ = wall_case()
  x0, x1, _ = syn.room_pair(0, n_raw=30000)
  vs = 0.0625
  S, T = x0[voxelise(x0, vs)], x1[voxelise(x1, vs)]
  n_t = onm.estimate_normals(T, 2 * vs, 30)[0].astype(np.float32)
  T_gt = syn.room_pair(0, n_raw=30000)[2]
  T_init = syn.random_se3(np.random.default_rng(2), 4.0, 0.03) @ T_gt
  g = np.random.default_rng(3)
  T_o, info_o = oip.icp_point_to_plane(S, T, n_t, 2 * vs, T_init)
  T_c, info_c = oc.colored_icp(S, g.random(len(S)), T, n_t, g.random(len(T)), g.normal(size=(len(T), 3)), 2 * vs,
                               T_init, lambda_geometric=1.0)
  assert info_c['iterations'] == info_o['iterations'] and info_c['n_corr'] == info_o['n_corr']
  assert np.abs(T_c - T_o).max() <= 1e-12


def test_sliding_wall():
  P, I_P, Q, I_Q, nrm, T0 = wall_case()
  assert np.linalg.norm(WALL_SHIFT) > 0.03
  T_p, _ = oip.icp_point_to_plane(P, Q, nrm, WALL_VOXEL, T0)
  grad = oc.color_gradient(Q, nrm, I_Q, 2 * WALL_VOXEL, 30)[0].astype(np.float32)
  T_c, info = oc.colored_icp(P, I_P, Q, nrm, I_Q, grad, WALL_VOXEL, T0)
  left_p, left_c = np.linalg.norm(T_p[:3, 3]), np.linalg.norm(T_c[:3, 3])
  assert left_p >= WALL_P2PLANE_LEFT, left_p
  assert left_c <= WALL_COLORED_LEFT, left_c
  assert info['fitness'] > 0.9


# ---------------------------------------------------------------------------------------------------------------
# host side
# ---------------------------------------------------------------------------------------------------------------
def test_point_cloud_colours():
  pcd = dio.PointCloud(np.zeros((4, 3)))
  assert pcd.colors is None and not pcd.has_colors() and pcd.attributes == {}
  pcd.colors = [[0.1, 0.2, 0.3]] * 4
  assert pcd.colors.dtype == np.float64 and pcd.has_colors()
  with pytest.raises(ValueError):
    pcd.colors = np.zeros((4, 2))
  before = pcd.colors.copy()
  T = np.eye(4)
  T[:3, 3] = [1.0, 2.0, 3.0]
  pcd.transform(T)
  assert np.array_equal(pcd.colors, before) and np.array_equal(pcd.points[0], [1.0, 2.0, 3.0])
  pcd.colors = np.zeros((3, 3))                        # open3d's rule: one colour per point
  assert not pcd.has_colors()
  assert not dio.PointCloud().has_colors()


@pytest.mark.parametrize('fmt', ['ascii', 'binary_little_endian', 'binary_big_endian'])
def test_read_point_cloud_colours(tmp_path, fmt):
  g = np.random.default_rng(0)
  pts = g.normal(size=(50, 3))
  c8 = g.integers(0, 256, size=(50, 3)).astype(np.uint8)
  dio.write_ply(tmp_path / 'u8.ply', pts, fmt=fmt, red=c8[:, 0], green=c8[:, 1], blue=c8[:, 2])
  pcd = dio.read_point_cloud(str(tmp_path / 'u8.ply'))
  assert np.array_equal(pcd.colors, c8 / 255.0)
  assert sorted(pcd.attributes) == ['blue', 'green', 'red']          # attributes as before
  assert all(np.array_equal(pcd.attributes[k], v) for k, v in dio.read_ply(str(tmp_path / 'u8.ply'))[1].items())
  cf = g.random((50, 3)).astype(np.float32)
  dio.write_ply(tmp_path / 'f.ply', pts, fmt=fmt, red=cf[:, 0], green=cf[:, 1], blue=cf[:, 2])
  assert np.array_equal(dio.read_point_cloud(str(tmp_path / 'f.ply')).colors, cf.astype(np.float64))
  dio.write_ply(tmp_path / 'none.ply', pts, fmt=fmt, red=cf[:, 0])
  assert dio.read_point_cloud(str(tmp_path / 'none.ply')).colors is None


def test_mesh_reads_back_as_a_coloured_cloud(tmp_path):
  V = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
  cols = np.array([[1.0, 0, 0], [0, 1, 0], [0, 0, 1], [0.5, 0.5, 0.5]])
  dio.write_triangle_mesh(str(tmp_path / 'm.ply'), dio.TriangleMesh(V, [[0, 1, 2], [0, 2, 3]], cols))
  pcd = dio.read_point_cloud(str(tmp_path / 'm.ply'))
  assert pcd.has_colors() and np.allclose(pcd.points, V)
  assert np.array_equal(pcd.colors, np.clip(np.round(cols * 255), 0, 255) / 255.0)


def test_stand_in_checks_before_any_device():
  from deepglobalregistration_b200 import o3d_registration as reg
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  for mod in (o3d.pipelines.registration, o3d.registration):
    assert mod.registration_colored_icp is reg.registration_colored_icp
    assert mod.TransformationEstimationForColoredICP is reg.TransformationEstimationForColoredICP
  with pytest.raises(NotImplementedError):
    reg.TransformationEstimationForColoredICP(kernel=object())
  assert reg.TransformationEstimationForColoredICP(1.5).lambda_geometric == 0.968
  assert reg.TransformationEstimationForColoredICP(-0.1).lambda_geometric == 0.968
  assert reg.TransformationEstimationForColoredICP(0.5).lambda_geometric == 0.5
  pts = np.random.default_rng(0).normal(size=(20, 3))
  src, tgt = dio.PointCloud(pts), dio.PointCloud(pts)
  with pytest.raises(RuntimeError, match='normals'):
    reg.registration_colored_icp(src, tgt, 0.05, np.eye(4))
  tgt.normals = np.tile([0.0, 0.0, 1.0], (20, 1))
  with pytest.raises(RuntimeError, match='colours'):
    reg.registration_colored_icp(src, tgt, 0.05, np.eye(4))
  tgt.colors = np.full((20, 3), 0.5)
  with pytest.raises(RuntimeError, match='source'):
    reg.registration_colored_icp(src, tgt, 0.05, np.eye(4), reg.TransformationEstimationForColoredICP(),
                                 reg.ICPConvergenceCriteria())
  src.colors = np.full((20, 3), 0.5)
  tgt.colors = None
  with pytest.raises(RuntimeError, match='target'):
    reg.registration_colored_icp(src, tgt, 0.05, np.eye(4), reg.ICPConvergenceCriteria(), 0.9)


def test_stand_in_argument_forms():
  from deepglobalregistration_b200 import o3d_registration as reg
  crit = reg.ICPConvergenceCriteria(max_iteration=7)
  T = np.eye(4)
  parse = reg._colored_icp_arguments
  assert parse((0.05, T, crit, 0.9), {}) == (0.05, T, crit, 0.9)                         # 0.10
  assert parse((0.05, T, crit), {}) == (0.05, T, crit, 0.968)
  assert parse((0.05,), dict(lambda_geometric=2.0)) == (0.05, None, None, 0.968)
  est = reg.TransformationEstimationForColoredICP(0.8)
  assert parse((0.05, T, est, crit), {}) == (0.05, T, crit, 0.8)                         # >= 0.12
  assert parse((), dict(max_correspondence_distance=0.05, estimation_method=est)) == (0.05, None, None, 0.8)
  assert parse((0.05, T), dict(estimation_method=est, criteria=crit)) == (0.05, T, crit, 0.8)
  with pytest.raises(TypeError):
    parse((0.05, T, est, crit), dict(lambda_geometric=0.5))
  with pytest.raises(TypeError):
    parse((0.05, T, crit, 0.9, 1), {})


def test_multiway_refinement_inputs(tmp_path):
  from deepglobalregistration_b200.core.multiway import MultiwayRegistration, coloured_fragments
  method = type('M', (), {'voxel_size': 0.05})()
  with pytest.raises(ValueError):
    MultiwayRegistration(method, refine='point_to_plane')
  assert MultiwayRegistration(method).refine is None
  pts = np.random.default_rng(0).normal(size=(10, 3))
  plain = dio.PointCloud(pts)
  with pytest.raises(ValueError, match='fragment 0'):
    coloured_fragments([plain])
  coloured = dio.PointCloud(pts)
  coloured.colors = np.full((10, 3), 0.5)
  with pytest.raises(ValueError, match='fragment 1'):                 # raised before the pairwise stage needs a device
    MultiwayRegistration(method, refine='colored_icp').register_sequence([coloured, pts])
  c8 = np.full((10, 3), 128, np.uint8)
  dio.write_ply(tmp_path / 'c.ply', pts, red=c8[:, 0], green=c8[:, 1], blue=c8[:, 2])
  dio.write_ply(tmp_path / 'p.ply', pts)
  (P, C), = coloured_fragments([tmp_path / 'c.ply'])
  assert np.allclose(P, pts.astype(np.float32)) and np.array_equal(C, np.full((10, 3), 128 / 255.0))
  with pytest.raises(ValueError, match='no colours'):
    coloured_fragments([str(tmp_path / 'p.ply')])


def test_colored_declarations():
  from deepglobalregistration_b200 import _abi
  p, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
  D = _abi.DECLARATIONS
  assert D['dgr_color_gradient'] == (i32, [p, p, p, i64, p, p, p, i64, i32, f64, f64, i32, p, p, p])
  assert D['dgr_colored_icp'] == (i32, [p, p, i64, p, p, p, p, p, p, p, i64, i32, f64, f64, f64, p, i32, f64, f64, p,
                                        p, p])
