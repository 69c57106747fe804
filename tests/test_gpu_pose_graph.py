"""dgr_information_matrix and dgr_pose_graph_optimize against the fp64 restatement (oracle/pose_graph.py), the caps and
argument checks, and the open3d stand-in on top of them.

Agreement bars: the kernel and the oracle run the same algorithm in fp64 with different summation orders and a
different Cholesky, so they agree to round-off; the bars below sit above the largest differences observed on an
H100 (printed by each test)."""
import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import _abi
from deepglobalregistration_b200 import synthetic as syn
from oracle import pose_graph as pg

pytestmark = pytest.mark.gpu

POSE_ATOL = 1e-9          # pose entries, kernel vs oracle (largest observed: 2.4e-11, N = 7 without compensation)
LP_ATOL = 1e-9            # line process (largest observed: 2.7e-11, N = 256)


def _hash(tgt64, cell):
  _, spec, table, sel, _, n = _abi.voxelise(tgt64, cell)
  return tgt64[sel.long()].float().contiguous(), (spec, table), n


def _info_case(src, tgt, T, max_dist, cell):
  dev = torch.device('cuda')
  _abi.refresh_stream()
  t_vox, h, _ = _hash(torch.from_numpy(np.ascontiguousarray(tgt, dtype=np.float64)).to(dev), cell)
  s = torch.from_numpy(np.ascontiguousarray(src, dtype=np.float32)).to(dev)
  out = _abi.information_matrix(s, t_vox, h, cell, max_dist, T).cpu().numpy()
  L, n = pg.information_matrix(src, t_vox.cpu().numpy(), T, max_dist)
  return out, L, n, (s, t_vox, h)


@pytest.mark.parametrize('n_src', [1, 255, 256, 257])
def test_information_matrix_vs_oracle(n_src):
  rng = np.random.default_rng(n_src)
  vs = 0.05
  lattice = np.stack(np.meshgrid(*[np.arange(12)] * 3, indexing='ij'), -1).reshape(-1, 3)
  tgt = (lattice + rng.uniform(0.05, 0.95, size=lattice.shape)) * vs           # one point per voxel
  T = syn.random_se3(rng, 5.0, 0.02)
  src = syn.apply_se3(np.linalg.inv(T), tgt[rng.choice(len(tgt), n_src, replace=False)])
  src = src + rng.normal(0, 0.01, size=src.shape)
  if n_src > 1:
    src[: n_src // 10] += 5.0                          # points with no neighbour
  out, L, n, _ = _info_case(src, tgt, T, 2 * vs, vs)
  assert out[36] == n and out[35] == n
  scale = max(np.abs(L).max(), 1.0)
  diff = np.abs(out[:36].reshape(6, 6) - L).max() / scale
  print(f'n_src={n_src} count={n} max relative difference {diff:.2e}')
  assert diff < 1e-12


def test_information_matrix_bench_pair_and_determinism():
  vs = 0.05
  xyz0, xyz1, T = syn.room_pair(0)
  dev = torch.device('cuda')
  s, _, n0 = _hash(torch.from_numpy(xyz0).to(dev), vs)
  out, L, n, (s_d, t_vox, h) = _info_case(s.cpu().numpy(), xyz1, T, 2 * vs, vs)
  assert out[36] == n and n > 1000
  scale = np.abs(L).max()
  diff = np.abs(out[:36].reshape(6, 6) - L).max() / scale
  print(f'bench pair {n0} / {len(t_vox)} voxels: {n} correspondences, max relative difference {diff:.2e}')
  assert diff < 1e-12
  again = _abi.information_matrix(s_d, t_vox, h, vs, 2 * vs, T).cpu().numpy()
  assert np.array_equal(out, again)


def _graph(seed, n, n_loops, noise=0.01, n_wrong=0):
  g = syn.pose_graph(seed, n, n_loops, noise=noise, n_wrong=n_wrong)
  from deepglobalregistration_b200.core.multiway import odometry_chain
  edges = [dict(s=int(s), t=int(t), T=T) for (s, t), T in zip(g['ends'], g['T'])]
  g['start'] = odometry_chain(n, edges) if n > 1 else np.eye(4)[None]
  return g


def _compare(g, ref=0, **option):
  E = len(g['ends'])
  conf = np.ones(E)
  P, kept, lp, st = _abi.pose_graph_optimize(g['start'], g['ends'], g['T'], g['info'], g['uncertain'], conf,
                                             reference_node=ref, **option)
  Po, ko, lo, so = pg.global_optimization(g['start'], g['ends'], g['T'], g['info'], g['uncertain'], conf,
                                          option=dict(reference_node=ref, **option))
  dp = np.abs(P - Po).max() if len(P) else 0.0
  dl = np.abs(lp - lo).max() if E else 0.0
  print(f'N={len(P)} E={E} ref={ref}: iterations {st["iterations"]}/{st["iterations_pruned"]} (oracle '
        f'{so["iterations"]}/{so["iterations_pruned"]}), pruned {st["pruned"]}, max |dP| {dp:.2e}, max |dl| {dl:.2e}, '
        f'cost {st["cost"]:.6e} vs {so["cost"]:.6e}')
  assert st['status'] == so['status'] == 0
  assert np.array_equal(kept, ko)
  assert (st['iterations'], st['iterations_pruned'], st['pruned']) == (so['iterations'], so['iterations_pruned'],
                                                                     so['pruned'])
  assert dp < POSE_ATOL and dl < LP_ATOL
  assert abs(st['cost'] - so['cost']) <= 1e-9 * max(1.0, abs(so['cost']))
  if ref >= 0:
    assert np.array_equal(P[ref], g['start'][ref])
  return P, kept, lp, st


def test_optimiser_single_node_and_no_edges():
  g = _graph(0, 1, 0)
  P, kept, lp, st = _compare(g)
  assert np.array_equal(P[0], np.eye(4)) and st['iterations'] == 0 and len(kept) == 0
  g = _graph(1, 4, 0)
  g['ends'], g['T'], g['info'], g['uncertain'] = g['ends'][:0], g['T'][:0], g['info'][:0], g['uncertain'][:0]
  P, kept, lp, st = _compare(g, ref=-1)
  assert np.array_equal(P, g['start']) and st['iterations'] == 0


@pytest.mark.parametrize('n,n_loops', [(2, 0), (3, 1)])
def test_optimiser_small_graphs(n, n_loops):
  _compare(_graph(n, n, n_loops))


@pytest.mark.parametrize('ref', [-1, 0, 6])
def test_optimiser_across_the_panel_width(ref):
  g = _graph(7, 7, 8, noise=0.02, n_wrong=2)         # 6 N = 42 crosses the 32-column panel
  P, kept, lp, st = _compare(g, ref=ref)
  assert (~kept)[g['wrong']].all()                     # every wrong closure goes (noisy correct ones may too)


def test_optimiser_all_pairs_of_60_nodes():
  n = 60
  g = _graph(60, n, n * (n - 1) // 2 - (n - 1), noise=0.005, n_wrong=(n * (n - 1) // 2 - (n - 1)) // 5)
  assert len(g['ends']) == 1770
  P, kept, lp, st = _compare(g)
  assert np.array_equal(~kept, g['wrong'])


def test_optimiser_256_nodes():
  g = _graph(256, 256, 300, noise=0.005, n_wrong=30)
  P, kept, lp, st = _compare(g)
  assert (~kept)[g['wrong']].all()


def test_optimiser_is_deterministic():
  g = _graph(9, 20, 40, noise=0.01, n_wrong=5)
  a = _abi.pose_graph_optimize(g['start'], g['ends'], g['T'], g['info'], g['uncertain'], np.ones(len(g['ends'])),
                               reference_node=0)
  b = _abi.pose_graph_optimize(g['start'], g['ends'], g['T'], g['info'], g['uncertain'], np.ones(len(g['ends'])),
                               reference_node=0)
  assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and a[3] == b[3]


def _err(fn, match):
  with pytest.raises(_abi.DgrError, match=match):
    fn()


def test_caps_and_invalid_input():
  g = _graph(3, 5, 3)
  args = [g['start'], g['ends'], g['T'], g['info'], g['uncertain'], np.ones(len(g['ends']))]

  names = ('poses', 'ends', 'T', 'info', 'uncertain', 'confidence')

  def run(**kw):
    a = list(args)
    for k, v in kw.items():
      if k in names:
        a[names.index(k)] = v
    opt = {k: v for k, v in kw.items() if k not in names}
    return _abi.pose_graph_optimize(*a, **opt)

  _err(lambda: _abi.pose_graph_optimize(np.tile(np.eye(4), (257, 1, 1)), np.zeros((0, 2)), np.zeros((0, 4, 4)),
                                        np.zeros((0, 6, 6)), [], []), 'node count')
  E = _abi.POSE_GRAPH_MAX_EDGES + 1
  ends = np.stack([np.zeros(E), np.ones(E)], 1)
  _err(lambda: _abi.pose_graph_optimize(np.tile(np.eye(4), (2, 1, 1)), ends, np.tile(np.eye(4), (E, 1, 1)),
                                        np.tile(np.eye(6), (E, 1, 1)), np.zeros(E), np.ones(E)), 'edge count')
  bad = g['ends'].copy(); bad[0, 1] = 5
  _err(lambda: run(ends=bad), 'node id')
  bad = g['ends'].copy(); bad[1, 1] = bad[1, 0]
  _err(lambda: run(ends=bad), 'itself')
  bad = g['start'].copy(); bad[2, 0, 3] = np.nan
  _err(lambda: run(poses=bad), 'poses')
  bad = g['info'].copy(); bad[0, 1, 1] = np.inf
  _err(lambda: run(info=bad), 'information')
  _err(lambda: run(reference_node=5), 'reference_node')
  _err(lambda: run(reference_node=-2), 'reference_node')
  _err(lambda: run(max_correspondence_distance=0.0), 'max_correspondence_distance')
  dev = torch.device('cuda')
  t = torch.rand(100, 3, device=dev, dtype=torch.float64)
  tv, h, _ = _hash(t, 0.05)
  _err(lambda: _abi.information_matrix(tv, tv, h, 0.05, 0.25, np.eye(4)), 'radius')
  _err(lambda: _abi.information_matrix(tv, tv, h, 0.05, 0.1, np.full((4, 4), np.nan)), 'finite')


def test_stand_in_equals_abi_and_oracle():
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  reg = o3d.pipelines.registration
  g = _graph(11, 10, 12, noise=0.01, n_wrong=2)
  pose_graph = reg.PoseGraph()
  for P in g['start']:
    pose_graph.nodes.append(reg.PoseGraphNode(P))
  for (s, t), T, L, u in zip(g['ends'], g['T'], g['info'], g['uncertain']):
    pose_graph.edges.append(reg.PoseGraphEdge(int(s), int(t), T, L, uncertain=bool(u)))
  option = reg.GlobalOptimizationOption(max_correspondence_distance=0.05, edge_prune_threshold=0.25,
                                        preference_loop_closure=2.0, reference_node=0)
  reg.global_optimization(pose_graph, reg.GlobalOptimizationLevenbergMarquardt(),
                          reg.GlobalOptimizationConvergenceCriteria(), option)
  P, kept, lp, st = _abi.pose_graph_optimize(g['start'], g['ends'], g['T'], g['info'], g['uncertain'],
                                             np.ones(len(g['ends'])), max_correspondence_distance=0.05,
                                             preference_loop_closure=2.0, reference_node=0)
  assert np.array_equal(np.stack([v.pose for v in pose_graph.nodes]), P)
  assert len(pose_graph.edges) == int(kept.sum()) == len(kept) - 2
  kept_l = lp[kept]
  assert np.array_equal([e.confidence if e.uncertain else 1.0 for e in pose_graph.edges], kept_l)
  Po, ko, lo, so = pg.global_optimization(g['start'], g['ends'], g['T'], g['info'], g['uncertain'],
                                          option=dict(max_correspondence_distance=0.05, preference_loop_closure=2.0,
                                                      reference_node=0))
  assert np.abs(P - Po).max() < POSE_ATOL and np.array_equal(kept, ko)
  with pytest.raises(NotImplementedError):
    reg.global_optimization(pose_graph, reg.GlobalOptimizationGaussNewton())
  # the information matrix through the stand-in: its own hash at cell = radius / 2
  rng = np.random.default_rng(3)
  xyz0, xyz1, T = syn.room_pair(3, n_raw=20000, extent=(1.8, 1.5, 1.25))
  dev = torch.device('cuda')
  v0, _, _ = _hash(torch.from_numpy(xyz0).to(dev), 0.05)
  v1, h1, _ = _hash(torch.from_numpy(xyz1).to(dev), 0.05)
  src, tgt = v0.double().cpu().numpy(), v1.double().cpu().numpy()
  L = reg.get_information_matrix_from_point_clouds(src, tgt, 0.1, T)
  ref = _abi.information_matrix(v0, v1, h1, 0.05, 0.1, T).cpu().numpy()
  assert L.dtype == np.float64 and L.shape == (6, 6) and np.array_equal(L, ref[:36].reshape(6, 6))
  Lo, n = pg.information_matrix(src, tgt, T, 0.1)
  assert L[5, 5] == n and np.abs(L - Lo).max() < 1e-12 * np.abs(Lo).max()
  del rng


def _poison(name, words, dev):
  """Fill the reused scratch arena the next call of that entry point gets with all-ones words (NaN as fp64)."""
  _abi.refresh_stream()
  _abi.scratch(name, words, torch.int64, dev).fill_(-1)


@pytest.mark.parametrize('n', [10, 60])
def test_optimiser_result_does_not_depend_on_workspace_contents(n):
  """The workspace is an arena that other calls reuse; stale words (NaN patterns included) in it, and in particular
  in the padding of the 6 N system up to the 32-column panel, must not reach the result."""
  import ctypes
  dev = _abi.require_device('cuda')           # the arena is keyed by the indexed device
  n_loops = 12 if n == 10 else n * (n - 1) // 2 - (n - 1)
  g = _graph(60 if n == 60 else 10, n, n_loops, noise=0.005, n_wrong=n_loops // 5)
  E = len(g['ends'])
  words = ctypes.c_int64(0)
  _abi.call('dgr_pose_graph_ws_elems', n, E, ctypes.byref(words))
  _abi.scratch('pose_graph', words.value, torch.int64, dev).zero_()
  clean = _abi.pose_graph_optimize(g['start'], g['ends'], g['T'], g['info'], g['uncertain'], np.ones(E),
                                   reference_node=0)
  _poison('pose_graph', words.value, dev)
  P, kept, lp, st = _compare(g)
  assert np.array_equal(P, clean[0]) and np.array_equal(kept, clean[1]) and np.array_equal(lp, clean[2])
  assert st == clean[3]


def test_information_matrix_does_not_depend_on_workspace_contents():
  import ctypes
  vs = 0.05
  dev = _abi.require_device('cuda')           # the arena is keyed by the indexed device
  xyz0, xyz1, T = syn.room_pair(3, n_raw=20000, extent=(1.8, 1.5, 1.25))
  v0, _, _ = _hash(torch.from_numpy(xyz0).to(dev), vs)
  v1, h1, _ = _hash(torch.from_numpy(xyz1).to(dev), vs)
  clean = _abi.information_matrix(v0, v1, h1, vs, 2 * vs, T).cpu().numpy()
  words = ctypes.c_int64(0)
  _abi.call('dgr_information_matrix_ws_elems', len(v0), ctypes.byref(words))
  _poison('information', words.value, dev)
  assert np.array_equal(_abi.information_matrix(v0, v1, h1, vs, 2 * vs, T).cpu().numpy(), clean)
