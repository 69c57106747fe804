"""dgr_estimate_normals and dgr_icp (open3d 0.10's EstimateNormals with KDTreeSearchParamHybrid and
point-to-plane ICP) against oracle/normals.py and oracle/icp_plane.py, the open3d stand-in that calls them, and the
ICP baselines.  The neighbour sets are compared exactly (both sides evaluate d^2 with the same rounding); the
cumulant sums and the ICP's normal equations run in a different order on the GPU, so normals and poses are compared
to round-off."""
import json
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import icp as oicp
from oracle import icp_plane as oip
from oracle import normals as onm
from test_gpu_fgr import rotation_angle
from test_gpu_ransac_fm import EXTENT, _card

pytestmark = pytest.mark.gpu


def _t(a, dt):
  return torch.as_tensor(np.asarray(a)).to('cuda', dt).contiguous()


def voxelise(x, cell):
  """float32-representable points, the first per cell of size `cell` (so the GPU hash holds one per cell)."""
  x32 = np.asarray(x, np.float32).astype(np.float64)
  _, first = np.unique(np.floor(x32 / cell).astype(np.int64), axis=0, return_index=True)
  return x32[np.sort(first)]


def cloud_hash(P, cell):
  """(spec, table) of the cloud's own voxel hash at `cell`, rows = rows of P."""
  from deepglobalregistration_b200 import _abi
  _, spec, table, _, _, n = _abi.voxelise(_t(P, torch.float64), cell)
  assert n == len(P)
  return spec, table


def gpu_normals(P, cell, radius, max_nn, prev=None):
  from deepglobalregistration_b200 import _abi
  nrm, counts = _abi.estimate_normals(_t(P, torch.float32), cloud_hash(P, cell), cell, radius, max_nn,
                                      prev=None if prev is None else _t(prev, torch.float32), return_counts=True)
  return nrm.cpu().numpy().astype(np.float64), counts.cpu().numpy()


def check_normals(n_gpu, counts, P, radius, max_nn, prev=None):
  n_o, c_o, eig = onm.estimate_normals(P, radius, max_nn, prev=prev)
  assert np.array_equal(counts, c_o)
  default = np.all(eig == 0.0, axis=1)                                 # the (0, 0, 1) points, oriented
  assert np.array_equal(n_gpu[default], n_o[default])
  unit = n_gpu / np.linalg.norm(n_gpu, axis=1, keepdims=True)
  gap = (eig[:, 1] - eig[:, 0]) / np.maximum(eig[:, 2], 1e-300)
  ok = ~default & (gap > 1e-6)
  dots = (unit * n_o).sum(1)
  assert np.all(np.abs(dots[ok]) >= 1 - 1e-9), np.sort(np.abs(dots[ok]))[:5]
  return n_o, ok, dots


def clouds():
  room = syn.room_pair(1, n_raw=60000)[0]
  lidar = syn.lidar_scan(2)
  return [('room', room, 0.05), ('lidar', lidar, 0.3)]


@pytest.mark.parametrize('ratio', [2, 3, 4])
def test_normals_match_the_oracle(ratio):
  for name, x, cell in clouds():
    P = voxelise(x, cell)
    radius = ratio * cell
    n_gpu, counts = gpu_normals(P, cell, radius, 30)
    assert (counts > 30).any() or ratio == 2, name                   # the selection path runs
    n_o, ok, _ = check_normals(n_gpu, counts, P, radius, 30)
    assert ok.mean() > 0.5, (name, ratio, ok.mean())
    # previous normals: the oracle's, each flipped at random (and tilted), away from orthogonal
    g = np.random.default_rng(ratio)
    prev = np.where(g.random(len(P))[:, None] < 0.5, -1.0, 1.0) * (n_o + g.normal(0, 0.05, size=n_o.shape))
    n_gpu_p, counts_p = gpu_normals(P, cell, radius, 30, prev=prev.astype(np.float32))
    prev32 = prev.astype(np.float32).astype(np.float64)
    n_op, ok_p, dots = check_normals(n_gpu_p, counts_p, P, radius, 30, prev=prev32)
    clear = ok_p & (np.abs((n_op * prev32).sum(1)) > 1e-3)
    assert np.all(dots[clear] > 0)                                     # the same sign as the oracle's
    assert np.all((n_gpu_p * prev32).sum(1)[clear] > 0)


def test_normals_max_nn_bounds():
  from deepglobalregistration_b200 import _abi
  P = voxelise(syn.room_pair(2, n_raw=30000)[0], 0.05)
  for max_nn in (1, 3, 64):
    n_gpu, counts = gpu_normals(P, 0.05, 0.2, max_nn)
    check_normals(n_gpu, counts, P, 0.2, max_nn)
  spec_table = cloud_hash(P, 0.05)
  for max_nn, radius in ((65, 0.1), (0, 0.1), (30, 0.25)):
    with pytest.raises(_abi.DgrError):
      _abi.estimate_normals(_t(P, torch.float32), spec_table, 0.05, radius, max_nn)


def plane_case(seed, max_iter=30):
  """Room pair (not a rigid copy) voxelised at 0.0625, the source started a few degrees / cm off the true pose."""
  vs = 0.0625
  x0, x1, T_gt = syn.room_pair(seed, n_raw=40000)
  P, Q = voxelise(x0, vs), voxelise(x1, vs)
  g = np.random.default_rng(seed)
  T_init = syn.random_se3(g, 4.0, 0.03) @ T_gt
  n_gpu, _ = gpu_normals(Q, vs, 2 * vs, 30)
  return P, Q, n_gpu, T_init, T_gt, vs


def run_plane(P, Q, nrm, vs, max_dist, T_init, max_iter=30, hashed=None):
  from deepglobalregistration_b200 import _abi
  hashed = hashed or cloud_hash(Q, vs)
  return _abi.icp_point_to_plane(_t(P, torch.float32), _t(Q, torch.float32), _t(nrm, torch.float32), hashed, vs,
                                 max_dist, T_init, max_iter).cpu().numpy()


def run_point(P, Q, vs, max_dist, T_init, hashed=None):
  from deepglobalregistration_b200 import _abi
  hashed = hashed or cloud_hash(Q, vs)
  return _abi.icp_point_to_point(_t(P, torch.float32), _t(Q, torch.float32), hashed, vs, max_dist,
                                 T_init).cpu().numpy()


def check_icp(res, P, Q, nrm, max_dist, T_init, max_iter=30):
  T_o, info = oip.icp_point_to_plane(P, Q, nrm.astype(np.float32), max_dist, T_init, max_iter)
  assert (int(res[18]), int(res[19])) == (info['iterations'], info['n_corr']), (res[16:], info)
  assert abs(res[16] - info['fitness']) <= 1e-9 and abs(res[17] - info['inlier_rmse']) <= 1e-9
  T = res[:16].reshape(4, 4)
  assert np.array_equal(T[3], [0, 0, 0, 1]) and np.all(np.isfinite(T))
  assert np.linalg.norm(T[:3, 3] - T_o[:3, 3]) <= 1e-7 and rotation_angle(T[:3, :3], T_o[:3, :3]) <= 1e-7
  return T, info


@pytest.mark.parametrize('seed', [1, 2, 3])
def test_point_to_plane_matches_the_oracle(seed):
  P, Q, nrm, T_init, T_gt, vs = plane_case(seed)
  res = run_plane(P, Q, nrm, vs, 2 * vs, T_init)
  T, info = check_icp(res, P, Q, nrm, 2 * vs, T_init)
  assert info['fitness'] > 0.5 and 1 <= info['iterations'] < 30
  te, re = syn.rte_rre(T, T_gt)
  assert te < 0.02 and re < 0.02, (te, re)
  res3 = run_plane(P, Q, nrm, vs, 3 * vs, T_init, max_iter=3)         # max_iteration reached
  check_icp(res3, P, Q, nrm, 3 * vs, T_init, max_iter=3)
  assert int(res3[18]) == 3


def test_reproducible():
  P, Q, nrm, T_init, _, vs = plane_case(4)
  a, ca = gpu_normals(Q, vs, 3 * vs, 30)
  b, cb = gpu_normals(Q, vs, 3 * vs, 30)
  assert np.array_equal(a, b) and np.array_equal(ca, cb)
  hashed = cloud_hash(Q, vs)
  r1 = run_plane(P, Q, nrm, vs, 2 * vs, T_init, hashed=hashed)
  r2 = run_plane(P, Q, nrm, vs, 2 * vs, T_init, hashed=hashed)
  assert np.array_equal(r1, r2)
  p1 = run_point(P, Q, vs, 2 * vs, T_init, hashed=hashed)
  p2 = run_point(P, Q, vs, 2 * vs, T_init, hashed=hashed)
  assert np.array_equal(p1, p2)


def test_edge_cases():
  from deepglobalregistration_b200 import _abi
  g = np.random.default_rng(0)
  x, y = np.meshgrid(np.arange(12) * 0.1, np.arange(12) * 0.1)
  plane = np.stack([x.ravel(), y.ravel(), np.zeros(144)], 1)
  plane[:, :2] += g.uniform(-0.02, 0.02, size=(144, 2))
  plane = plane.astype(np.float32).astype(np.float64)
  n_gpu, counts = gpu_normals(plane, 0.05, 0.1, 30)
  check_normals(n_gpu, counts, plane, 0.1, 30)
  assert np.array_equal(n_gpu, np.tile([0.0, 0.0, 1.0], (144, 1)))
  src = (plane + np.array([0.01, -0.02, 0.03])).astype(np.float32).astype(np.float64)
  empty = np.zeros((0, 3))
  T0 = np.eye(4)
  cases = [('single plane', src, plane, n_gpu), ('out of range', src + 10.0, plane, n_gpu), ('empty source', empty,
           plane, n_gpu)]
  for name, S, Q, N in cases:
    res = run_plane(S, Q, N, 0.05, 0.1, T0)
    T, info = check_icp(res, S, Q, N, 0.1, T0)
    assert np.array_equal(T, np.eye(4)), name
  # empty target: an empty table (any key spec)
  spec = cloud_hash(plane, 0.05)[0]
  no_target = (spec, _abi.HashTable(1, torch.device('cuda')))
  res = run_plane(src, empty, empty, 0.05, 0.1, T0, hashed=no_target)
  T, info = check_icp(res, src, empty, empty, 0.1, T0)
  assert np.array_equal(T, np.eye(4)) and res[16] == 0 and int(res[18]) == 1
  # point-to-point where nothing matches: the identity, fitness 0, open3d's iteration count
  for name, S, Q, hashed in (('out of range', src + 10.0, plane, None), ('empty source', empty, plane, None),
                            ('empty target', src, empty, no_target)):
    res = run_point(S, Q, 0.05, 0.1, T0, hashed=hashed)
    _, info = oicp.icp_point_to_point(S, Q, 0.1, T0)
    assert np.array_equal(res[:16].reshape(4, 4), np.eye(4)) and res[16] == 0, name
    assert (int(res[18]), int(res[19])) == (info['iterations'], info['n_corr']) == (1, 0), name


def test_stand_in_reference_call_sequence():
  from deepglobalregistration_b200 import _abi, shims
  from deepglobalregistration_b200 import o3d_registration as reg
  o3d = shims._open3d_stub()
  P, Q, _, T_init, T_gt, vs = plane_case(5)
  src, tgt = o3d.geometry.PointCloud(), o3d.geometry.PointCloud()
  src.points, tgt.points = o3d.utility.Vector3dVector(P), o3d.utility.Vector3dVector(Q)
  tgt.estimate_normals(o3d.KDTreeSearchParamHybrid(radius=2 * vs, max_nn=30))        # util/pointcloud.py:60
  assert tgt.normals.dtype == np.float64 and tgt.normals.shape == Q.shape
  result = o3d.registration.registration_icp(src, tgt, 2 * vs, T_init,
                                             o3d.registration.TransformationEstimationPointToPlane())
  # the same thing through _abi directly, bit for bit
  cell, spec, table = reg._target_hash(_t(Q, torch.float64), 2 * vs)
  assert cell == vs
  nrm = _abi.estimate_normals(_t(Q, torch.float32), (spec, table), cell, 2 * vs, 30)
  assert np.array_equal(tgt.normals, nrm.cpu().numpy().astype(np.float64))
  want = _abi.icp_point_to_plane(_t(P, torch.float32), _t(Q, torch.float32), nrm, (spec, table), cell, 2 * vs,
                                 T_init).cpu().numpy()
  assert np.array_equal(result.transformation, want[:16].reshape(4, 4))
  assert (result.fitness, result.inlier_rmse, len(result.correspondence_set)) == (want[16], want[17], int(want[19]))
  te, re = syn.rte_rre(result.transformation, T_gt)
  assert te < 0.02 and re < 0.02, (te, re)
  # existing normals orient the new ones; transform rotates them
  flipped = o3d.geometry.PointCloud()
  flipped.points = o3d.utility.Vector3dVector(Q)
  flipped.normals = -tgt.normals
  flipped.estimate_normals(o3d.geometry.KDTreeSearchParamHybrid(radius=2 * vs, max_nn=30))
  unit = tgt.normals / np.linalg.norm(tgt.normals, axis=1, keepdims=True)
  assert np.all((flipped.normals * unit).sum(1)[np.any(tgt.normals != [0, 0, 1], axis=1)] < 0)
  before = tgt.normals.copy()
  tgt.transform(T_gt)
  assert np.allclose(tgt.normals, before @ T_gt[:3, :3].T, atol=1e-15)


def _dgr():
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  st = syn.make_checkpoint(4, voxel_size=0.0625)
  return DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))


def test_icp_baselines_recover_a_small_misalignment():
  from deepglobalregistration_b200.core.icp_baseline import ICPBaseline
  d = _dgr()
  xyz0 = syn.room_scan(2, 40000, EXTENT, scene_seed=1) - np.array(EXTENT) / 2
  T_gt = syn.random_se3(np.random.default_rng(3), 3.0, 0.03)
  xyz1 = syn.apply_se3(T_gt, xyz0)
  e0 = syn.rte_rre(np.eye(4), T_gt)
  for method, branch in (('point_to_plane', 'icp_plane'), ('point_to_point', 'icp')):
    b = ICPBaseline(d, method)
    T = b.register(xyz0, xyz1)
    assert b.last_branch == branch and T.dtype == np.float64 and T.shape == (4, 4)
    te, re = syn.rte_rre(T, T_gt)
    assert te < 0.01 and re < 0.005 and te < e0[0] / 3 and re < e0[1] / 3, (method, te, re, e0, b.last_info)
    info = b.last_info
    assert info['icp_fitness'] > 0.8 and info['icp_iterations'] >= 1 and info['icp_correspondences'] > 0


def test_evaluate_icp_point_to_plane_on_a_pair_list(tmp_path, capsys):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200 import io as dio
  from deepglobalregistration_b200 import sharding
  from deepglobalregistration_b200.core.icp_baseline import ICPBaseline
  state = syn.make_checkpoint(0)
  torch.save(state, tmp_path / 'ckpt.pth')
  xyz0 = syn.room_scan(2, 20000, EXTENT, scene_seed=1)
  T_gt = syn.random_se3(np.random.default_rng(1), 3.0, 0.03)
  dio.write_ply(tmp_path / 'a.ply', xyz0, dtype='double')
  np.savez(tmp_path / 'b.npz', pcd=syn.apply_se3(T_gt, xyz0))
  (tmp_path / 'pairs.txt').write_text(f'a.ply b.npz {" ".join(repr(float(x)) for x in T_gt.reshape(-1))} room\n'
                                      'a.ply b.npz\n')
  for method, stem, name in (('icp_point_to_plane', 'icp-p2plane-b200', 'ICP (Point-to-plane)'),
                             ('icp_point_to_point', 'icp-p2p-b200', 'ICP (Point-to-point)')):
    ev.main(['--pair_list', str(tmp_path / 'pairs.txt'), '--weights', str(tmp_path / 'ckpt.pth'), '--out_dir',
             str(tmp_path), '--method', method, '--icp_max_iteration', '40'])
    summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert summary['pairs'] == 2 and summary['with_ground_truth'] == 1 and summary['recall'] == 1.0
    saved = np.load(tmp_path / f'{stem}-stats.npz', allow_pickle=True)
    assert list(saved['names']) == [name] and saved['stats'].shape == (1, 2, 5)
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=str(tmp_path / 'ckpt.pth'), clip_weight_thresh=0.05,
                                                   verbose=False))
  out = ev.evaluate(ICPBaseline(d, 'point_to_plane'), ev.read_pair_list(tmp_path / 'pairs.txt'))
  assert np.array_equal(out['branch'], [sharding.BRANCH_CODE['icp_plane']] * 2)


def test_dgr_pair_size_time():
  """Normals and both ICPs at the DGR pair size: ~51k voxels per cloud, radius 2 voxels, max_nn 30, correspondences
  within 2 voxels, from a pose a few degrees / cm off."""
  from deepglobalregistration_b200 import _abi
  vs = 0.0625
  P = voxelise(syn.room_scan(8, 500000, (4.5, 3.75, 3.125)), vs)
  n = len(P)
  assert 45000 < n < 60000, n
  g = np.random.default_rng(0)
  T_gt = syn.random_se3(g, 3.0, 0.03)
  Q = voxelise(syn.apply_se3(T_gt, syn.room_scan(9, 500000, (4.5, 3.75, 3.125), scene_seed=8)), vs)
  hashed = cloud_hash(Q, vs)
  src, tgt = _t(P, torch.float32), _t(Q, torch.float32)
  T0 = _t(np.eye(4)[:3], torch.float64)

  def step():
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    nrm = _abi.estimate_normals(tgt, hashed, vs, 2 * vs, 30)
    ev[1].record()
    r_plane = _abi.icp_point_to_plane(src, tgt, nrm, hashed, vs, 2 * vs, T0)
    ev[2].record()
    r_point = _abi.icp_point_to_point(src, tgt, hashed, vs, 2 * vs, T0)
    ev[3].record()
    torch.cuda.synchronize()
    return [ev[k].elapsed_time(ev[k + 1]) for k in range(3)], r_plane.cpu().numpy(), r_point.cpu().numpy()
  step()                                                           # warm-up, workspaces allocated
  ms = []
  for _ in range(5):
    t, r_plane, r_point = step()
    ms.append(t)
  ms = np.array(ms)
  print(f'\n[icp] {_card()}: n_s = {n}, n_t = {len(Q)}, radius 2 voxels, max_nn 30: normals {np.median(ms[:, 0]):.3f} ms, '
        f'point-to-plane ICP {np.median(ms[:, 1]):.3f} ms ({int(r_plane[18])} iterations), point-to-point ICP '
        f'{np.median(ms[:, 2]):.3f} ms ({int(r_point[18])} iterations) (medians of 5; '
        f'{"; ".join(", ".join(f"{v:.3f}" for v in col) for col in ms.T)})')
  for r in (r_plane, r_point):
    te, re = syn.rte_rre(r[:16].reshape(4, 4), T_gt)
    assert te < 0.02 and re < 0.01, (te, re, r[16:])
