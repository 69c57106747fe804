"""dgr_ransac_feature_matching (open3d 0.10's registration_ransac_based_on_feature_matching,
core/deep_global_registration.py:29-47) against oracle/ransac_fm.py, the open3d stand-in that calls it,
and the FCGF + RANSAC baseline built on it.  Both sides draw the same hypotheses (counter-hash sampler)
and run the checkers in fp64, so the validated set is the same; scoring is fp64 on both sides too (voxel
hash on the GPU, KD-tree in the oracle), so the winner is the oracle's unless a point within round-off of
the radius tips a tie."""
import json
import subprocess
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import ransac as orn
from oracle import ransac_fm as orf

pytestmark = pytest.mark.gpu
EXTENT = (1.8, 1.5, 1.25)


def target_hash(tgt, max_dist):
  from deepglobalregistration_b200 import o3d_registration as reg
  return reg._target_hash(torch.as_tensor(np.asarray(tgt, np.float64)).cuda().contiguous(), max_dist)


def run(P, Q, nn, max_dist, M, V, seed=0, edge_ratio=0.0, check_dist=None, hashed=None):
  from deepglobalregistration_b200 import _abi
  cell, spec, table = hashed or target_hash(Q, max_dist)
  t = lambda a, dt: torch.as_tensor(np.asarray(a)).to('cuda', dt).contiguous()
  return _abi.ransac_feature_matching(t(P, torch.float32), t(Q, torch.float32), t(nn, torch.int32), spec, table, cell,
                                     max_dist, edge_ratio, max_dist if check_dist is None else check_dist, M, V,
                                     seed=seed).cpu().numpy()


def gpu_nn(fs, ft):
  from deepglobalregistration_b200 import _abi
  return _abi.knn_top1(torch.from_numpy(fs).cuda(), torch.from_numpy(ft).cuda()).cpu().numpy()


def check_against_oracle(res, P, Q, nn, max_dist, M, V, seed, edge_ratio=0.0, check_dist=None):
  cd = max_dist if check_dist is None else check_dist
  T_o, info = orf.ransac_feature_matching(P, Q, nn, max_dist, M, V, edge_ratio=edge_ratio, check_dist=cd, seed=seed)
  n = len(P)
  assert int(res[20]) == info['validated'] and int(res[21]) == info['drawn'], (res[16:], info)
  hyp = int(res[18])
  T = res[:16].reshape(4, 4)
  assert np.array_equal(T[3], [0, 0, 0, 1])
  if hyp < 0:
    assert info['hypothesis'] == -1 and np.array_equal(T, np.eye(4)) and res[16] == 0 and res[19] == 0
    return T, info
  # the pose is the Kabsch fit of the GPU winner's own four draws (checks the sampler and nn)
  s = orn.sample_indices(seed, [hyp], n)
  R, t = orn.kabsch_batch(np.asarray(P, np.float64)[s], np.asarray(Q, np.float64)[nn[s]])
  np.testing.assert_allclose(T[:3, :3], R[0], atol=1e-9)
  np.testing.assert_allclose(T[:3, 3], t[0], atol=1e-9)
  # as good as the oracle's best: the same hypothesis, or within 2 / n_s of its fitness
  from scipy.spatial import cKDTree
  mine, _ = orf.score(T[:3, :3], T[:3, 3], np.asarray(P, np.float64), cKDTree(np.asarray(Q, np.float64)),
                      np.asarray(Q, np.float64), max_dist)
  assert abs(mine - int(res[19])) <= 2 and abs(res[16] - res[19] / n) <= 1e-15
  assert hyp == info['hypothesis'] or mine >= info['matched'] - 2, (hyp, info, mine)
  if hyp == info['hypothesis']:
    assert abs(res[17] - info['inlier_rmse']) <= 1e-9
  return T, info


@pytest.mark.parametrize('seed,n,frac,edge', [(1, 2000, 0.3, 0.0), (2, 3000, 0.4, 0.0), (3, 1500, 0.5, 0.9)])
def test_same_winner_as_oracle(seed, n, frac, edge):
  P, Q, fs, ft, T_gt, perm, ident = syn.feature_matching_pair(seed, n=n, match_frac=frac)
  nn = gpu_nn(fs, ft)
  assert np.array_equal(nn, orf.feature_nn(fs, ft))
  res = run(P, Q, nn, 0.03, 6000, 1000, seed=seed + 10, edge_ratio=edge)
  T, info = check_against_oracle(res, P, Q, nn, 0.03, 6000, 1000, seed + 10, edge_ratio=edge)
  te, re = syn.rte_rre(T, T_gt)
  assert te < 0.01 and re < 0.01, (te, re)
  assert res[16] > 0.95


def test_reproducible_and_seeded():
  P, Q, fs, ft, _, _, _ = syn.feature_matching_pair(5, n=2500, match_frac=0.4)
  nn = gpu_nn(fs, ft)
  h = target_hash(Q, 0.03)
  a = run(P, Q, nn, 0.03, 20000, 1000, seed=1, hashed=h)
  b = run(P, Q, nn, 0.03, 20000, 1000, seed=1, hashed=h)
  c = run(P, Q, nn, 0.03, 20000, 1000, seed=2, hashed=h)
  assert np.array_equal(a, b)
  assert a[18] != c[18]


def test_counts_and_degenerate_cases():
  P, Q, fs, ft, _, _, _ = syn.feature_matching_pair(6, n=700, match_frac=0.5)
  nn = gpu_nn(fs, ft)
  h = target_hash(Q, 0.03)
  # M not a multiple of the 256-thread block; V above, at and below the number validated; V = 1
  for M, V in ((1000, 10 ** 6), (1025, 1000), (1000, 7), (3, 1), (1, 1), (4000, 1)):
    res = run(P, Q, nn, 0.03, M, V, seed=3, hashed=h)
    check_against_oracle(res, P, Q, nn, 0.03, M, V, 3)
    assert int(res[20]) <= min(M, V)
  # no checker: every hypothesis validates, so V validations take exactly V draws
  res = run(P, Q, nn, 0.03, 500, 33, seed=4, check_dist=0.0, hashed=h)
  assert int(res[20]) == 33 and int(res[21]) == 33
  check_against_oracle(res, P, Q, nn, 0.03, 500, 33, 4, check_dist=0.0)
  # nothing validates -> identity, hypothesis -1, nothing scored, every hypothesis drawn
  res = run(P, Q, nn, 0.03, 777, 100, seed=5, check_dist=1e-9, hashed=h)
  assert np.array_equal(res[:16].reshape(4, 4), np.eye(4)) and res[18] == -1
  assert res[16] == 0 and res[17] == 0 and res[19] == 0 and res[20] == 0 and res[21] == 777
  # validated, but no source point lands within the radius (0.1 mm, far below the 3 mm noise of every fit): still
  # the initial result
  res = run(P, Q, nn, 1e-4, 300, 50, seed=6, check_dist=0.0)
  assert res[18] == -1 and int(res[20]) == 50 and np.array_equal(res[:16].reshape(4, 4), np.eye(4))
  check_against_oracle(res, P, Q, nn, 1e-4, 300, 50, 6, check_dist=0.0)
  # argument checks come back as errors, not crashes
  from deepglobalregistration_b200 import _abi
  for kw in (dict(M=0, V=10), dict(M=10, V=0)):
    with pytest.raises(_abi.DgrError):
      run(P, Q, nn, 0.03, kw['M'], kw['V'], hashed=h)
  with pytest.raises(_abi.DgrError):            # radius above 4 cells
    run(P, Q, nn, 0.03 * 5, 10, 10, hashed=h)
  with pytest.raises(_abi.DgrError):
    run(P, Q, nn, 0.03, 10, 10, edge_ratio=-1.0, hashed=h)


def test_stand_in_as_the_reference_calls_it():
  """core/deep_global_registration.py:29-47 verbatim on the stand-in, against the direct ABI call."""
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  P, Q, fs, ft, T_gt, _, _ = syn.feature_matching_pair(7, n=3000, match_frac=0.35)
  pcd0, pcd1 = o3d.geometry.PointCloud(), o3d.geometry.PointCloud()
  pcd0.points, pcd1.points = o3d.utility.Vector3dVector(P), o3d.utility.Vector3dVector(Q)
  feats0, feats1, distance_threshold, num_iterations = fs, ft, 0.03, 80000

  source_feat = o3d.registration.Feature()
  source_feat.resize(feats0.shape[1], len(feats0))
  source_feat.data = feats0.astype('d').transpose()
  target_feat = o3d.registration.Feature()
  target_feat.resize(feats1.shape[1], len(feats1))
  target_feat.data = feats1.astype('d').transpose()
  result = o3d.registration.registration_ransac_based_on_feature_matching(
      pcd0, pcd1, source_feat, target_feat, distance_threshold,
      o3d.registration.TransformationEstimationPointToPoint(False), 4,
      [o3d.registration.CorrespondenceCheckerBasedOnDistance(distance_threshold)],
      o3d.registration.RANSACConvergenceCriteria(num_iterations, 1000))

  res = run(P, Q, gpu_nn(fs, ft), 0.03, 80000, 1000, seed=0)
  assert np.array_equal(result.transformation, res[:16].reshape(4, 4))
  assert result.fitness == res[16] and result.inlier_rmse == res[17] and len(result.correspondence_set) == int(res[19])
  te, re = syn.rte_rre(result.transformation, T_gt)
  assert te < 0.01 and re < 0.01, (te, re)


def _calibrated_rigid_copy():
  """The rigid-copy pair of test_gpu_pipeline.py::test_safeguard_branch_known_answer: cloud 1 = cloud 0 shifted by
  a multiple of 8 voxels, BatchNorm-calibrated random-init FCGF, so features identify the true matches."""
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.util.calibrate import calibrate_batchnorm
  vs = 0.0625
  st = syn.make_checkpoint(4, voxel_size=vs)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))
  xyz0 = syn.room_scan(2, 20000, EXTENT, scene_seed=1)
  T_gt = np.eye(4)
  T_gt[:3, 3] = vs * np.array([8, -16, 24])
  xyz1 = syn.apply_se3(T_gt, xyz0)
  with torch.no_grad():
    _, c0, f0 = d.preprocess(xyz0)
    calibrate_batchnorm(d.fcgf_model, ME.SparseTensor(f0, coordinates=c0, device='cuda'))
  return d, xyz0, xyz1, T_gt


def test_fcgf_ransac_known_answer():
  from deepglobalregistration_b200.core.fcgf_ransac import FCGFRansac
  d, xyz0, xyz1, T_gt = _calibrated_rigid_copy()
  method = FCGFRansac(d)
  assert (method.max_iteration, method.max_validation, method.edge_ratio) == (80000, 1000, 0.0)
  assert method.voxel_size == d.voxel_size
  for use_icp in (False, True):
    d.use_icp = use_icp
    T = method.register(xyz0, xyz1)
    assert method.last_branch == 'ransac' and T.dtype == np.float64 and T.shape == (4, 4)
    te, re = syn.rte_rre(T, T_gt)
    assert te <= 1e-3 and re <= 1e-3, (use_icp, te, re, method.last_info)
    info = method.last_info
    assert info['ransac_fitness'] > 0.9 and info['ransac_validated'] == 1000
    assert ('icp_fitness' in info) == use_icp


def test_evaluate_fcgf_ransac_on_a_pair_list(tmp_path, capsys):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200 import io as dio
  state = syn.make_checkpoint(0)
  torch.save(state, tmp_path / 'ckpt.pth')
  xyz0, xyz1, T_gt = syn.room_pair(2, n_raw=20000, extent=EXTENT)
  dio.write_ply(tmp_path / 'a.ply', xyz0, dtype='double')
  np.savez(tmp_path / 'b.npz', pcd=xyz1)
  (tmp_path / 'pairs.txt').write_text(f'a.ply b.npz {" ".join(repr(float(x)) for x in T_gt.reshape(-1))} room\n'
                                      'a.ply b.npz\n')
  ev.main(['--pair_list', str(tmp_path / 'pairs.txt'), '--weights', str(tmp_path / 'ckpt.pth'), '--out_dir',
           str(tmp_path), '--method', 'fcgf_ransac', '--ransac_max_iteration', '20000', '--ransac_max_validation',
           '300', '--ransac_edge_ratio', '0.9'])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  assert summary['pairs'] == 2 and summary['with_ground_truth'] == 1 and 'recall' in summary
  saved = np.load(tmp_path / 'fcgf-ransac-b200-stats.npz', allow_pickle=True)
  assert list(saved['names']) == ['RANSAC'] and saved['stats'].shape == (1, 2, 5)
  for T in saved['poses']:
    assert np.allclose(T[:3, :3] @ T[:3, :3].T, np.eye(3), atol=1e-9) and np.array_equal(T[3], [0, 0, 0, 1])
  assert saved['stats'][0, 0, 3] > 0


def _card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return out or f'{torch.cuda.get_device_name()}, power limit unknown'


def test_dgr_pair_size_search_time():
  """The baseline's setting at the DGR pair size: n_s ~ 51k voxels, M = 80000, V = 1000, cell = voxel,
  d = check distance = 2 voxels, half the features right."""
  vs = 0.0625
  x = syn.room_scan(8, 500000, (4.5, 3.75, 3.125))
  _, first = np.unique(np.floor(x / vs).astype(np.int64), axis=0, return_index=True)
  P = x[np.sort(first)]
  T_gt = np.eye(4)
  T_gt[:3, 3] = vs * np.array([8, -16, 24])
  Q = P + T_gt[:3, 3]
  n = len(P)
  g = np.random.default_rng(0)
  nn = np.where(g.random(n) < 0.5, np.arange(n), g.integers(0, n, size=n)).astype(np.int32)
  h = target_hash(Q, 2 * vs)
  assert h[0] == vs and 45000 < n < 60000, (h[0], n)
  from deepglobalregistration_b200 import _abi
  cell, spec, table = h
  src, tgt = torch.from_numpy(P).float().cuda(), torch.from_numpy(Q).float().cuda()
  nn_d = torch.from_numpy(nn).cuda()
  call = lambda M, V, seed: _abi.ransac_feature_matching(src, tgt, nn_d, spec, table, cell, 2 * vs, 0.0, 2 * vs, M, V,
                                                         seed=seed)
  call(80000, 1000, 99)                                             # warm-up, workspace allocated
  ms = []
  for rep in range(3):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    res = call(80000, 1000, rep)
    e1.record()
    torch.cuda.synchronize()
    ms.append(e0.elapsed_time(e1))
  res = res.cpu().numpy()
  t = float(np.median(ms))
  q = int(res[20]) * n
  print(f'\n[ransac_fm] {_card()}: n_s {n}, M 80000, V {int(res[20])} scored ({int(res[21])} drawn): '
        f'{t:.2f} ms (median of {", ".join(f"{m:.2f}" for m in ms)}) = {q / t / 1e6:.2f} G queries/s, '
        f'{q * 125 / t / 1e6:.1f} G cell probes/s (125 per query)')
  assert int(res[20]) == 1000
  te, re = syn.rte_rre(res[:16].reshape(4, 4), T_gt)
  assert te < 1e-3 and re < 1e-3 and res[16] > 0.99
