"""dgr_fgr_feature_matching (open3d's registration_fast_based_on_feature_matching) against oracle/fgr.py, the open3d
stand-in that calls it, and the FCGF + FGR baseline built on it.  The mutual list and the tuple correspondences
come from the same counter-hash draws on both sides and are compared exactly; the optimiser's sums run in a
different order on the GPU, so the pose is compared to round-off."""
import json

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import fgr as ofg
from oracle import ransac_fm as orf
from test_gpu_ransac_fm import EXTENT, _calibrated_rigid_copy, _card

pytestmark = pytest.mark.gpu


def _t(a, dt):
  return torch.as_tensor(np.asarray(a)).to('cuda', dt).contiguous()


def run(P, Q, nn_st, nn_ts, seed=0, **option):
  from deepglobalregistration_b200 import _abi
  res, corres = _abi.fgr_feature_matching(_t(P, torch.float32), _t(Q, torch.float32), _t(nn_st, torch.int32),
                                          _t(nn_ts, torch.int32), seed=seed, return_correspondences=True, **option)
  res = res.cpu().numpy()
  return res, corres.cpu().numpy()[:int(res[17])]


def gpu_nn(fs, ft):
  from deepglobalregistration_b200 import _abi
  return _abi.knn_top1(torch.from_numpy(fs).cuda(), torch.from_numpy(ft).cuda()).cpu().numpy()


def pair(seed, larger, n=2500, frac=0.5):
  """feature_matching_pair with 15 % of the other cloud's rows dropped, so `larger` has more points."""
  P, Q, fs, ft, T_gt, _, _ = syn.feature_matching_pair(seed, n=n, match_frac=frac)
  keep = np.random.default_rng(seed + 100).random(n) >= 0.15
  if larger == 'source':
    Q, ft = Q[keep], ft[keep]
  else:
    P, fs = P[keep], fs[keep]
  return P, Q, fs, ft, T_gt


def check_against_oracle(res, corres, P, Q, nn_st, nn_ts, seed, **option):
  T_o, info = ofg.fgr(P, Q, nn_st, nn_ts, seed=seed, **option)
  assert (int(res[16]), int(res[17]), int(res[18])) == (info['n_mut'], info['n_corr'], info['drawn']), (res[16:], info)
  assert bool(res[20]) == info['ran'] and bool(res[21]) == info['swapped'] and res[19] == info['mu']
  assert np.array_equal(corres, info['corres'])
  T = res[:16].reshape(4, 4)
  assert np.array_equal(T[3], [0, 0, 0, 1])
  te, re = np.linalg.norm(T[:3, 3] - T_o[:3, 3]), rotation_angle(T[:3, :3], T_o[:3, :3])
  assert te <= 1e-8 and re <= 1e-8, (te, re)
  return T, info


def rotation_angle(R1, R2):
  """Angle [rad] between two rotations from the chord |R1 - R2|_F = 2 sqrt(2) sin(angle / 2): resolves angles
  near 0 that arccos((trace - 1) / 2) cannot (its floor is ~1.5e-8 rad)."""
  return 2.0 * np.arcsin(min(1.0, np.linalg.norm(R1 - R2) / (2.0 * np.sqrt(2.0))))


@pytest.mark.parametrize('larger', ['source', 'target'])
@pytest.mark.parametrize('seed', [1, 2, 3])
def test_matches_the_oracle(seed, larger):
  P, Q, fs, ft, T_gt = pair(seed, larger)
  nn_st, nn_ts = gpu_nn(fs, ft), gpu_nn(ft, fs)
  assert np.array_equal(nn_st, orf.feature_nn(fs, ft)) and np.array_equal(nn_ts, orf.feature_nn(ft, fs))
  res, corres = run(P, Q, nn_st, nn_ts, seed=seed + 10)
  T, info = check_against_oracle(res, corres, P, Q, nn_st, nn_ts, seed + 10)
  assert bool(res[21]) == (larger == 'target') and info['n_corr'] == 3000
  te, re = syn.rte_rre(T, T_gt)
  assert te < 0.01 and re < 0.01, (te, re)
  # the mutual list itself, in order
  res_m, mutual = run(P, Q, nn_st, nn_ts, seed=seed + 10, tuple_test=False)
  assert np.array_equal(mutual, info['mutual']) and int(res_m[18]) == 0
  check_against_oracle(res_m, mutual, P, Q, nn_st, nn_ts, seed + 10, tuple_test=False)


def test_options_match_the_oracle():
  P, Q, fs, ft, _ = pair(4, 'source')
  nn_st, nn_ts = gpu_nn(fs, ft), gpu_nn(ft, fs)
  for option in (dict(decrease_mu=False), dict(use_absolute_scale=True), dict(iteration_number=5),
                 dict(tuple_scale=0.9, maximum_tuple_count=300), dict(division_factor=2.0, iteration_number=0),
                 dict(maximum_tuple_count=10 ** 6)):
    res, corres = run(P, Q, nn_st, nn_ts, seed=5, **option)
    check_against_oracle(res, corres, P, Q, nn_st, nn_ts, 5, **option)


def test_long_mutual_list_on_a_cluster():
  """tuple_test off with >= 16384 mutual candidates: the solver runs on a cluster of 8 CTAs."""
  g = np.random.default_rng(9)
  n = 20000
  P = g.uniform(-2.0, 2.0, size=(n, 3))
  T_gt = syn.random_se3(g, 30.0, 0.5)
  Q = syn.apply_se3(T_gt, P) + g.normal(0, 0.002, size=(n, 3))
  nn_st = np.where(g.random(n) < 0.7, np.arange(n), g.integers(0, n, size=n))
  nn_ts = np.where(g.random(n) < 0.9, np.arange(n), g.integers(0, n, size=n))
  res, corres = run(P, Q, nn_st, nn_ts, tuple_test=False)
  T, info = check_against_oracle(res, corres, P.astype(np.float32), Q.astype(np.float32), nn_st, nn_ts, 0,
                                 tuple_test=False)
  assert info['n_mut'] > 10000
  te, re = syn.rte_rre(T, T_gt)
  assert te < 0.01 and re < 0.01, (te, re)


def test_reproducible_and_seeded():
  P, Q, fs, ft, _ = pair(6, 'target')
  nn_st, nn_ts = gpu_nn(fs, ft), gpu_nn(ft, fs)
  a, ca = run(P, Q, nn_st, nn_ts, seed=1)
  b, cb = run(P, Q, nn_st, nn_ts, seed=1)
  c, cc = run(P, Q, nn_st, nn_ts, seed=2)
  assert np.array_equal(a, b) and np.array_equal(ca, cb)
  assert not np.array_equal(ca, cc)


def test_degenerate_cases_and_bad_arguments():
  from deepglobalregistration_b200 import _abi
  P, Q, fs, ft, _ = pair(7, 'source', n=300)
  pinned = np.eye(4)
  # 2 mutual pairs: no trial, the optimiser does not run
  nn_st, nn_ts = np.zeros(len(P), np.int64), np.full(len(Q), 2)
  nn_st[1], nn_ts[1] = 1, 1
  nn_ts[0] = 0
  res, corres = run(P, Q, nn_st, nn_ts)
  check_against_oracle(res, corres, P, Q, nn_st, nn_ts, 0)
  pinned[:3, 3] = Q.astype(np.float64).mean(0) - P.astype(np.float64).mean(0)
  assert (int(res[16]), int(res[17]), int(res[18]), res[20]) == (2, 0, 0, 0)
  np.testing.assert_allclose(res[:16].reshape(4, 4), pinned, atol=1e-12)
  # fewer than 10 correspondences: 3 tuples; 5 mutual pairs without the tuple test
  nn_st, nn_ts = gpu_nn(fs, ft), gpu_nn(ft, fs)
  res, corres = run(P, Q, nn_st, nn_ts, maximum_tuple_count=3)
  check_against_oracle(res, corres, P, Q, nn_st, nn_ts, 0, maximum_tuple_count=3)
  assert int(res[17]) == 9 and res[20] == 0
  nn5_st, nn5_ts = np.full(len(P), 5), np.zeros(len(Q), np.int64)      # rows >= 5 all point at a row that
  nn5_st[:5], nn5_ts[:5] = np.arange(5), np.arange(5)                   # points elsewhere
  res, corres = run(P, Q, nn5_st, nn5_ts, tuple_test=False)
  check_against_oracle(res, corres, P, Q, nn5_st, nn5_ts, 0, tuple_test=False)
  assert int(res[16]) == 5 and res[20] == 0
  for option in (dict(tuple_scale=0.0), dict(tuple_scale=1.5), dict(division_factor=1.0), dict(iteration_number=-1),
                 dict(maximum_tuple_count=0), dict(maximum_correspondence_distance=0.0)):
    with pytest.raises(_abi.DgrError):
      run(P, Q, nn_st, nn_ts, **option)


def test_stand_in_under_both_module_paths():
  from deepglobalregistration_b200 import _abi, shims
  o3d = shims._open3d_stub()
  P, Q, fs, ft, T_gt = pair(8, 'target')
  want = _abi.fgr_feature_matching(_t(P, torch.float32), _t(Q, torch.float32),
                                   _t(gpu_nn(fs, ft), torch.int32), _t(gpu_nn(ft, fs), torch.int32)).cpu().numpy()
  for reg in (o3d.pipelines.registration, o3d.registration):
    pcd0, pcd1 = o3d.geometry.PointCloud(), o3d.geometry.PointCloud()
    pcd0.points, pcd1.points = o3d.utility.Vector3dVector(P), o3d.utility.Vector3dVector(Q)
    f0, f1 = reg.Feature(), reg.Feature()
    f0.resize(fs.shape[1], len(fs))
    f0.data = fs.astype('d').transpose()
    f1.resize(ft.shape[1], len(ft))
    f1.data = ft.astype('d').transpose()
    result = reg.registration_fast_based_on_feature_matching(
        pcd0, pcd1, f0, f1, reg.FastGlobalRegistrationOption(maximum_correspondence_distance=0.025))
    assert np.array_equal(result.transformation, want[:16].reshape(4, 4))
    assert result.fitness == 0 and len(result.correspondence_set) == 0
  te, re = syn.rte_rre(result.transformation, T_gt)
  assert te < 0.01 and re < 0.01, (te, re)


def test_fcgf_fgr_known_answer():
  from deepglobalregistration_b200.core.fcgf_fgr import FCGFFastGlobal
  d, xyz0, xyz1, T_gt = _calibrated_rigid_copy()
  method = FCGFFastGlobal(d)
  assert method.option.tuple_scale == 0.95 and method.voxel_size == d.voxel_size
  for use_icp in (False, True):
    d.use_icp = use_icp
    T = method.register(xyz0, xyz1)
    assert method.last_branch == 'fgr' and T.dtype == np.float64 and T.shape == (4, 4)
    te, re = syn.rte_rre(T, T_gt)
    assert te <= 1e-3 and re <= 1e-3, (use_icp, te, re, method.last_info)
    info = method.last_info
    assert info['fgr_ran'] and info['fgr_correspondences'] == 3000 and info['fgr_mutual'] > 100
    assert ('icp_fitness' in info) == use_icp


def test_evaluate_fcgf_fgr_on_a_pair_list(tmp_path, capsys):
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
           str(tmp_path), '--method', 'fcgf_fgr'])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  assert summary['pairs'] == 2 and summary['with_ground_truth'] == 1 and 'recall' in summary
  saved = np.load(tmp_path / 'fcgf-fgr-b200-stats.npz', allow_pickle=True)
  assert list(saved['names']) == ['FGR'] and saved['stats'].shape == (1, 2, 5)
  for T in saved['poses']:
    assert np.allclose(T[:3, :3] @ T[:3, :3].T, np.eye(3), atol=1e-9) and np.array_equal(T[3], [0, 0, 0, 1])
  assert saved['stats'][0, 0, 3] > 0


def test_dgr_pair_size_time():
  """FGR at the DGR pair size: n ~ 51k voxels per cloud, 32-channel features, both kNN directions + FGR with
  open3d's default options; half the source features identify their partner."""
  from deepglobalregistration_b200 import _abi
  vs = 0.0625
  x = syn.room_scan(8, 500000, (4.5, 3.75, 3.125))
  _, first = np.unique(np.floor(x / vs).astype(np.int64), axis=0, return_index=True)
  P = x[np.sort(first)]
  n = len(P)
  g = np.random.default_rng(0)
  T_gt = syn.random_se3(g, 30.0, 0.5)
  perm = g.permutation(n)
  Q = np.empty_like(P)
  Q[perm] = syn.apply_se3(T_gt, P)
  ft = g.normal(size=(n, 32))
  ft /= np.linalg.norm(ft, axis=1, keepdims=True)
  fs = ft[np.where(g.random(n) < 0.5, perm, g.integers(0, n, size=n))] + g.normal(0, 1e-3, size=(n, 32))
  assert 45000 < n < 60000, n
  src, tgt = _t(P, torch.float32), _t(Q, torch.float32)
  fs_d, ft_d = _t(fs, torch.float32), _t(ft, torch.float32)

  def step(seed):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    nn_st, nn_ts = _abi.knn_top1(fs_d, ft_d), _abi.knn_top1(ft_d, fs_d)
    ev[1].record()
    res = _abi.fgr_feature_matching(src, tgt, nn_st, nn_ts, seed=seed)
    ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), res
  step(99)                                                         # warm-up, workspaces allocated
  knn_ms, fgr_ms = [], []
  for rep in range(5):
    a, b, res = step(rep)
    knn_ms.append(a)
    fgr_ms.append(b)
  res = res.cpu().numpy()
  print(f'\n[fgr] {_card()}: n_s = n_t = {n}, 32 channels, n_mut {int(res[16])}, {int(res[17])} correspondences '
        f'({int(res[18])} trials): kNN both ways {np.median(knn_ms):.2f} ms, FGR {np.median(fgr_ms):.2f} ms '
        f'(medians of 5; kNN {", ".join(f"{m:.2f}" for m in knn_ms)}; FGR {", ".join(f"{m:.2f}" for m in fgr_ms)})')
  assert int(res[17]) == 3000 and res[20] == 1
  te, re = syn.rte_rre(res[:16].reshape(4, 4), T_gt)
  assert te < 1e-3 and re < 1e-3, (te, re)
