"""CPU tests of the multiway-registration oracle (oracle/pose_graph.py), the driver's host logic
(core/multiway.py) and the stand-in's argument checks."""
import math

import numpy as np
import pytest

from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import synthetic as syn
from oracle import pose_graph as pg


def _chain_start(g):
  """The odometry chain of a synthetic graph: where the driver starts."""
  edges = [dict(s=int(s), t=int(t), T=T) for (s, t), T in zip(g['ends'], g['T'])]
  from deepglobalregistration_b200.core.multiway import odometry_chain
  return odometry_chain(len(g['poses_gt']), edges)


def test_information_closed_form_equals_g_sum():
  rng = np.random.default_rng(1)
  src = rng.uniform(-1, 1, size=(500, 3)).astype(np.float32)
  T = syn.random_se3(rng, 10.0, 0.05)
  tgt = (syn.apply_se3(T, src.astype(np.float64)) + rng.normal(0, 0.01, size=(500, 3))).astype(np.float32)
  L, n = pg.information_matrix(src, tgt, T, 0.03)
  q = pg.correspondences(src, tgt, T, 0.03)
  assert 0 < n < 500 and len(q) == n
  np.testing.assert_allclose(pg.information_closed_form(q), L, rtol=1e-12, atol=1e-9)
  np.testing.assert_allclose(syn.information_from_points(q), L, rtol=1e-12, atol=1e-9)
  assert np.array_equal(L, L.T) or np.abs(L - L.T).max() < 1e-12
  assert np.linalg.eigvalsh(L).min() > -1e-9
  assert L[5, 5] == n and L[3, 3] == n and L[4, 4] == n


def test_nearest_within_tie_and_radius_rule():
  tgt = np.array([[1.0, 0, 0], [-1.0, 0, 0], [0, 0.5, 0]])
  j = pg.nearest_within(np.array([[0.0, 0, 0], [0, 0.5, 0.0], [5.0, 0, 0]]), tgt, 1.0)
  assert j.tolist() == [2, 2, -1]
  # equidistant rows: the lower one; exactly at the radius: no match (strict)
  assert pg.nearest_within(np.array([[0.0, 0, 0]]), tgt[:2], 1.5).tolist() == [0]
  assert pg.nearest_within(np.array([[0.0, 0, 0]]), tgt[:2], 1.0).tolist() == [-1]


def test_consistent_graph_is_a_fixed_point():
  g = syn.pose_graph(2, 8, 6, noise=0.0)
  P, kept, l, st = pg.global_optimization(g['poses_gt'], g['ends'], g['T'], g['info'], g['uncertain'],
                                          option=dict(reference_node=0))
  np.testing.assert_allclose(P, g['poses_gt'], atol=1e-9)
  assert np.allclose(l, 1.0) and kept.all() and st['pruned'] == 0 and st['status'] == 0


@pytest.mark.parametrize('ref', [-1, 0, 4])
def test_noisy_graph_cost_decreases_and_reference_keeps_its_pose(ref):
  g = syn.pose_graph(3, 9, 10, noise=0.02)
  P0 = _chain_start(g)
  P, kept, l, st = pg.global_optimization(P0, g['ends'], g['T'], g['info'], g['uncertain'],
                                          option=dict(reference_node=ref))
  assert st['status'] == 0 and st['iterations'] >= 1
  assert st['cost_first_pass'] <= st['cost_start']
  assert st['cost'] <= st['cost_first_pass'] + 1e-9
  if ref >= 0:
    assert np.array_equal(P[ref], P0[ref])


def test_wrong_loop_closures_are_pruned():
  g = syn.pose_graph(5, 12, 14, noise=0.005, n_wrong=3)
  P0 = _chain_start(g)
  P, kept, l, st = pg.global_optimization(P0, g['ends'], g['T'], g['info'], g['uncertain'],
                                          option=dict(reference_node=0))
  assert np.array_equal(~kept, g['wrong']), (l, g['wrong'])
  assert (l[g['wrong']] < 0.25).all() and st['pruned'] == 3
  ok = ~g['wrong']
  Pc, kc, lc, sc = pg.global_optimization(P0, g['ends'][ok], g['T'][ok], g['info'][ok], g['uncertain'][ok],
                                          option=dict(reference_node=0))
  assert kc.all()
  for k in range(len(P)):
    te, re = syn.rte_rre(P[k], Pc[k])
    assert te < 1e-3 and re < 1e-3, (k, te, re)


def test_closed_form_line_process_minimises_the_edge_term():
  for mu in (0.1, 1.0, 7.5):
    for q in (0.0, 0.05, 1.0, 30.0):
      l_star = pg.line_process(mu, q)
      grid = np.linspace(0.0, 1.0, 2001)
      f = grid * q + mu * (np.sqrt(grid) - 1.0) ** 2
      assert pg.edge_cost(q, l_star, mu, True) <= f.min() + 1e-12


def test_exp6_matches_the_zyx_convention():
  x = np.array([0.1, -0.2, 0.3, 1.0, 2.0, 3.0])
  T = pg.exp6(x)
  assert np.allclose(pg.pose_vector(T), x)
  assert np.allclose(syn._exp6(x), T)
  d = 1e-6
  for i, G in enumerate(pg.GENERATORS):
    e = np.zeros(6)
    e[i] = d
    np.testing.assert_allclose((pg.exp6(e) - np.eye(4)) / d, G, atol=1e-5)


def test_driver_edge_selection_chain_and_ate():
  from deepglobalregistration_b200.core.multiway import absolute_trajectory_error, odometry_chain, select_edges
  rng = np.random.default_rng(0)
  P = np.stack([np.eye(4)] + [syn.random_se3(rng, 20.0, 0.5) for _ in range(3)])
  edges = []
  for i in range(4):
    for j in range(i + 1, 4):
      info = np.zeros((6, 6))
      info[5, 5] = 100 if j == i + 1 or (i, j) == (0, 3) else 10
      edges.append(dict(s=i, t=j, T=np.linalg.inv(P[j]) @ P[i], info=info))
  kept = select_edges(edges, [200, 150, 300, 100], 0.3)
  assert [(e['s'], e['t']) for e in kept] == [(0, 1), (0, 3), (1, 2), (2, 3)]
  assert [e['uncertain'] for e in kept] == [False, True, False, False]
  assert math.isclose(next(e for e in edges if (e['s'], e['t']) == (0, 3))['overlap'], 1.0)
  C = odometry_chain(4, edges)
  np.testing.assert_allclose(C, P, atol=1e-12)
  assert absolute_trajectory_error(C, P) < 1e-12
  G = P.copy()
  G[:, :3, 3] += 0.1                                   # a common shift changes nothing relative to node 0
  G[0, :3, 3] -= 0.1
  moved = P.copy()
  moved[2, :3, 3] += np.array([0.3, 0.0, 0.4])
  assert math.isclose(absolute_trajectory_error(moved, P), math.sqrt(0.25 / 4))


def test_trajectory_round_trip(tmp_path):
  rng = np.random.default_rng(4)
  P = np.stack([syn.random_se3(rng) for _ in range(5)])
  path = tmp_path / 'traj.log'
  dio.write_trajectory(str(path), [([k, k, 5], T) for k, T in enumerate(P)])
  back = dio.read_trajectory(str(path))
  assert [cp.metadata for cp in back] == [[k, k, 5] for k in range(5)]
  assert np.array_equal(np.stack([cp.pose for cp in back]), P)


def test_room_fragments_overlap_and_close_the_loop():
  clouds, P = syn.room_fragments(0, n_frag=6, n_raw=30_000)
  assert len(clouds) == 6 and P.shape == (6, 4, 4)
  world = [syn.apply_se3(P[k], c) for k, c in enumerate(clouds)]
  from scipy.spatial import cKDTree
  for a, b in [(0, 1), (2, 3), (5, 0)]:
    d, _ = cKDTree(world[b]).query(world[a], k=1)
    assert (d < 0.05).mean() > 0.6, (a, b)            # ~4 cm sample spacing at 30k points per room


def test_stand_in_argument_checks_without_a_device():
  from deepglobalregistration_b200 import o3d_registration as reg
  g = reg.PoseGraph()
  g.nodes += [reg.PoseGraphNode(np.eye(4)), reg.PoseGraphNode(np.eye(4))]
  g.edges.append(reg.PoseGraphEdge(0, 1, np.eye(4), np.eye(6), uncertain=False))
  crit, opt = reg.GlobalOptimizationConvergenceCriteria(), reg.GlobalOptimizationOption()
  assert (crit.max_iteration, crit.max_iteration_lm, crit.upper_scale_factor) == (100, 20, 2 / 3)
  assert (opt.max_correspondence_distance, opt.edge_prune_threshold, opt.reference_node) == (0.075, 0.25, -1)
  with pytest.raises(NotImplementedError):
    reg.global_optimization(g, reg.GlobalOptimizationGaussNewton(), crit, opt)
  with pytest.raises(ValueError):
    reg.global_optimization(g, reg.GlobalOptimizationLevenbergMarquardt(), crit,
                            reg.GlobalOptimizationOption(reference_node=2))
  with pytest.raises(ValueError):
    reg.global_optimization(g, reg.GlobalOptimizationLevenbergMarquardt(), crit,
                            reg.GlobalOptimizationOption(max_correspondence_distance=0.0))
  bad = reg.PoseGraph()
  bad.nodes = list(g.nodes)
  bad.edges = [reg.PoseGraphEdge(1, 1)]
  with pytest.raises(ValueError):
    reg.global_optimization(bad)
  bad.edges = [reg.PoseGraphEdge(0, 5)]
  with pytest.raises(ValueError):
    reg.global_optimization(bad)
  bad.edges = [reg.PoseGraphEdge(0, 1, information=np.full((6, 6), np.nan))]
  with pytest.raises(ValueError):
    reg.global_optimization(bad)
  with pytest.raises(ValueError):
    reg.get_information_matrix_from_point_clouds(np.zeros((3, 3)), np.zeros((3, 3)), -1.0, np.eye(4))
