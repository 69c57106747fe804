"""dgr_estimate_covariances, dgr_covariances_from_normals, dgr_generalized_icp and the robust losses of dgr_icp_loss /
dgr_colored_icp_loss against oracle/gicp.py, the open3d stand-in's generalized ICP and kernels, the generalized-ICP
baseline and its CLI.  Neighbour counts are compared exactly; covariances and poses to round-off, since the sums run
in a different order on the GPU."""
import json

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import gicp as og
from oracle import normals as onm
from test_gpu_colored_icp import colored_case, run_colored
from test_gpu_fgr import rotation_angle
from test_gpu_icp_plane import _t, cloud_hash, gpu_normals, run_plane
from test_oracle_gicp import (GICP_EPSILON, LIDAR_GICP_LEFT, LIDAR_P2P_LEFT, OUTLIER_L2_PULLED, OUTLIER_TUKEY_K,
                              OUTLIER_TUKEY_LEFT, lidar_case, outlier_case, voxelise)

pytestmark = pytest.mark.gpu

KERNELS = [('L2', 1.0), ('L1', 1.0), ('Huber', 0.02), ('Cauchy', 0.02), ('GM', 0.02), ('Tukey', 0.05)]


def gpu_covariances(P, cell, radius, max_nn):
  from deepglobalregistration_b200 import _abi
  c, n = _abi.estimate_covariances(_t(P, torch.float32), cloud_hash(P, cell), cell, radius, max_nn,
                                   return_counts=True)
  return c.cpu().numpy(), n.cpu().numpy()


def gpu_cov_from_normals(nrm, eps=GICP_EPSILON):
  from deepglobalregistration_b200 import _abi
  return _abi.covariances_from_normals(_t(nrm, torch.float32), eps).cpu().numpy()


def run_gicp(P, Cs, Q, Ct, vs, max_dist, T_init, max_iter=30, kernel=None, hashed=None):
  from deepglobalregistration_b200 import _abi
  loss, k = (None, 1.0) if kernel is None else kernel
  return _abi.icp_generalized(_t(P, torch.float32), _t(Cs, torch.float64), _t(Q, torch.float32), _t(Ct, torch.float64),
                              hashed or cloud_hash(Q, vs), vs, max_dist, T_init, max_iter, loss=loss,
                              loss_k=k).cpu().numpy()


def check_against(res, T_o, info):
  """The colored-ICP bars: equal iterations and correspondences, fitness / RMSE <= 1e-9, pose <= 1e-7."""
  assert (int(res[18]), int(res[19])) == (info['iterations'], info['n_corr']), (res[16:], info)
  assert abs(res[16] - info['fitness']) <= 1e-9 and abs(res[17] - info['inlier_rmse']) <= 1e-9
  T = res[:16].reshape(4, 4)
  assert np.array_equal(T[3], [0, 0, 0, 1]) and np.all(np.isfinite(T))
  assert np.linalg.norm(T[:3, 3] - T_o[:3, 3]) <= 1e-7 and rotation_angle(T[:3, :3], T_o[:3, :3]) <= 1e-7, \
      (np.linalg.norm(T[:3, 3] - T_o[:3, 3]), rotation_angle(T[:3, :3], T_o[:3, :3]))


@pytest.mark.parametrize('ratio', [2, 4])
def test_covariances_match_the_oracle(ratio):
  vs = 0.05
  x0, _, _ = syn.room_pair(0, n_raw=60000)
  P = voxelise(x0, vs)
  radius = ratio * vs
  cov, counts = gpu_covariances(P, vs, radius, 30)
  _, n_counts = gpu_normals(P, vs, radius, 30)
  assert np.array_equal(counts, n_counts)
  cov_o, c_o = og.estimate_covariances(P, radius, 30)
  assert np.array_equal(counts, c_o)
  assert ratio == 2 or (counts > 30).any()                               # max_nn truncation active at ratio 4
  err = np.abs(og.full33(cov) - cov_o).max()
  print(f'ratio {ratio}: {len(P)} points, max covariance error {err:.3g} (scale {radius ** 2:.3g})')
  assert err <= 1e-15 * max(1.0, radius ** 2) * 64
  few = np.minimum(counts, 30) < 3
  assert np.array_equal(cov[few], np.tile([1.0, 0, 0, 1.0, 0, 1.0], (few.sum(), 1)))
  again, _ = gpu_covariances(P, vs, radius, 30)
  assert np.array_equal(cov, again)


def test_covariances_from_normals_match_the_oracle():
  g = np.random.default_rng(0)
  n = g.normal(size=(5000, 3))
  n /= np.linalg.norm(n, axis=1, keepdims=True)
  n[:3] = [[-1.0, 0.0, 0.0], [-0.995, np.sqrt(1 - 0.995 ** 2), 0.0], [1.0, 0.0, 0.0]]
  n32 = n.astype(np.float32)
  got = og.full33(gpu_cov_from_normals(n32))
  want = og.covariances_from_normals(n32.astype(np.float64), GICP_EPSILON)
  err = np.abs(got - want).max(axis=(1, 2)) * (1.0 + np.maximum(n32[:, 0], -0.99))
  assert err.max() <= 1e-14, err.max()
  assert np.array_equal(got[:2], np.tile(np.diag([GICP_EPSILON, 1.0, 1.0]), (2, 1, 1)))


def gicp_room_case(seed=0, vs=0.05):
  """Fragments of room_pair(0) at vs with covariances from the GPU's normals, and a start a few degrees / cm off."""
  x0, x1, T = syn.room_pair(0, n_raw=60000)
  P, Q = voxelise(x0, vs), voxelise(x1, vs)
  Cs = gpu_cov_from_normals(gpu_normals(P, vs, 2 * vs, 30)[0].astype(np.float32))
  Ct = gpu_cov_from_normals(gpu_normals(Q, vs, 2 * vs, 30)[0].astype(np.float32))
  T0 = syn.random_se3(np.random.default_rng(seed), 3.0, 0.03) @ T
  return P, Cs, Q, Ct, T, T0, vs


def gicp_lidar_case():
  S, Q, T, T0, vs = lidar_case()
  Cs = gpu_cov_from_normals(gpu_normals(S, vs, 2 * vs, 30)[0].astype(np.float32))
  Ct = gpu_cov_from_normals(gpu_normals(Q, vs, 2 * vs, 30)[0].astype(np.float32))
  return S, Cs, Q, Ct, T, T0, vs


@pytest.mark.parametrize('case', ['room', 'lidar'])
def test_generalized_icp_matches_the_oracle(case):
  P, Cs, Q, Ct, T, T0, vs = gicp_room_case() if case == 'room' else gicp_lidar_case()
  for max_iter in (30, 3):
    res = run_gicp(P, Cs, Q, Ct, vs, 2 * vs, T0, max_iter)
    T_o, info = og.generalized_icp(P, Cs, Q, Ct, 2 * vs, T0, max_iter=max_iter)
    check_against(res, T_o, info)
  hashed = cloud_hash(Q, vs)
  a = run_gicp(P, Cs, Q, Ct, vs, 2 * vs, T0, hashed=hashed)
  b = run_gicp(P, Cs, Q, Ct, vs, 2 * vs, T0, hashed=hashed)
  assert np.array_equal(a, b)
  te, re = syn.rte_rre(a[:16].reshape(4, 4), T)
  print(f'{case}: generalized ICP leaves {te:.4f} m, {re:.2e} rad after {int(a[18])} updates')
  if case == 'lidar':
    assert abs(te - LIDAR_GICP_LEFT) <= 1e-3
    p2p = _abi_p2p(P, Q, vs, 2 * vs, T0)
    assert abs(syn.rte_rre(p2p[:16].reshape(4, 4), T)[0] - LIDAR_P2P_LEFT) <= 1e-3
  else:
    assert te < 0.02 and re < 0.02


def _abi_p2p(P, Q, vs, max_dist, T0):
  from deepglobalregistration_b200 import _abi
  return _abi.icp_point_to_point(_t(P, torch.float32), _t(Q, torch.float32), cloud_hash(Q, vs), vs, max_dist,
                                 T0).cpu().numpy()


@pytest.mark.parametrize('kernel', KERNELS, ids=[k[0] for k in KERNELS])
def test_losses_match_the_oracle(kernel):
  from deepglobalregistration_b200 import _abi
  # L1's weight 1 / |r| grows without bound as residuals vanish, so round-off differences between the two sides grow
  # with every reweighting; it is compared over 3 updates (1 for generalized ICP, whose three rows per pair include
  # near-zero residuals from the first update on), the others over the full 30
  it = 3 if kernel[0] == 'L1' else 30
  # point-to-plane on the outlier pair
  Sg, Q, T, T0, vs = outlier_case()
  nrm = gpu_normals(Q, vs, 2 * vs, 30)[0].astype(np.float32)
  res = _abi.icp_point_to_plane(_t(Sg, torch.float32), _t(Q, torch.float32), _t(nrm, torch.float32),
                                cloud_hash(Q, vs), vs, 2 * vs, T0, it, loss=kernel[0], loss_k=kernel[1]).cpu().numpy()
  check_against(res, *og.icp_point_to_plane(Sg, Q, nrm, 2 * vs, T0, kernel=kernel, max_iter=it))
  # colored
  P, I_P, Qc, I_Q, nc, grad, Tc0, _, vc = colored_case()
  k_c = (kernel[0], kernel[1] * 0.5)
  res = _abi.icp_colored(_t(P, torch.float32), _t(I_P, torch.float32), _t(Qc, torch.float32), _t(nc, torch.float32),
                         _t(I_Q, torch.float32), _t(grad, torch.float32), cloud_hash(Qc, vc), vc, vc, 0.968, Tc0,
                         it, loss=k_c[0], loss_k=k_c[1]).cpu().numpy()
  check_against(res, *og.colored_icp(P, I_P, Qc, nc, I_Q, grad, vc, Tc0, kernel=k_c, max_iter=it))
  # generalized (residuals are in units of M^(-1/2): about 1 / sqrt(eps) times a distance)
  P, Cs, Qg, Ct, _, Tg0, vg = gicp_room_case(1)
  k_g = (kernel[0], kernel[1] * 50.0)
  it = 1 if kernel[0] == 'L1' else it
  res = run_gicp(P, Cs, Qg, Ct, vg, 2 * vg, Tg0, it, kernel=k_g)
  check_against(res, *og.generalized_icp(P, Cs, Qg, Ct, 2 * vg, Tg0, kernel=k_g, max_iter=it))


def test_l2_loss_is_bitwise_no_loss():
  from deepglobalregistration_b200 import _abi
  P, I_P, Q, I_Q, nrm, grad, T0, _, vs = colored_case(1)
  plain = run_plane(P, Q, nrm, vs, 2 * vs, T0)
  l2 = _abi.icp_point_to_plane(_t(P, torch.float32), _t(Q, torch.float32), _t(nrm, torch.float32), cloud_hash(Q, vs),
                               vs, 2 * vs, T0, loss='L2').cpu().numpy()
  assert np.array_equal(plain, l2)
  plain = run_colored(P, I_P, Q, nrm, I_Q, grad, vs, vs, T0)
  l2 = _abi.icp_colored(_t(P, torch.float32), _t(I_P, torch.float32), _t(Q, torch.float32), _t(nrm, torch.float32),
                        _t(I_Q, torch.float32), _t(grad, torch.float32), cloud_hash(Q, vs), vs, vs, 0.968, T0,
                        loss='L2', loss_k=123.0).cpu().numpy()
  assert np.array_equal(plain, l2)


def test_outlier_case_on_the_device():
  from deepglobalregistration_b200 import _abi
  Sg, Q, T, T0, vs = outlier_case()
  nrm = _t(gpu_normals(Q, vs, 2 * vs, 30)[0].astype(np.float32), torch.float32)
  h = cloud_hash(Q, vs)
  l2 = _abi.icp_point_to_plane(_t(Sg, torch.float32), _t(Q, torch.float32), nrm, h, vs, 2 * vs, T0).cpu().numpy()
  tk = _abi.icp_point_to_plane(_t(Sg, torch.float32), _t(Q, torch.float32), nrm, h, vs, 2 * vs, T0, loss='Tukey',
                               loss_k=OUTLIER_TUKEY_K).cpu().numpy()
  left2, leftt = (syn.rte_rre(r[:16].reshape(4, 4), T)[0] for r in (l2, tk))
  print(f'ghost wall: L2 leaves {left2:.4f} m, Tukey {leftt:.5f} m')
  assert left2 >= OUTLIER_L2_PULLED and leftt <= OUTLIER_TUKEY_LEFT


def test_argument_checks():
  from deepglobalregistration_b200 import _abi
  P, Cs, Q, Ct, T, T0, vs = gicp_room_case()
  for loss, k in (('Tukey', 0.0), ('Huber', -1.0), ('Cauchy', float('nan')), ('GM', float('inf'))):
    with pytest.raises(_abi.DgrError, match='loss_k'):
      run_gicp(P, Cs, Q, Ct, vs, 2 * vs, T0, kernel=(loss, k))
  with pytest.raises(_abi.DgrError):
    run_gicp(P, Cs, Q, Ct, vs, 4.5 * vs, T0)
  spec, table = cloud_hash(Q, vs)
  res = torch.empty(20, dtype=torch.float64, device='cuda')
  ws = torch.empty(1 << 16, dtype=torch.float64, device='cuda')
  T12 = _t(np.eye(4)[:3], torch.float64)
  Pd, Qd, Cd = _t(P, torch.float32), _t(Q, torch.float32), _t(Ct, torch.float64)

  def gicp(loss, k, src_cov, tgt_cov):
    _abi.call('dgr_generalized_icp', _abi.ptr(Pd), src_cov, len(P), _abi.ptr(Qd), tgt_cov, _abi.ptr(spec),
              _abi.ptr(table.keys), _abi.ptr(table.vals), table.cap, 0, vs, 2 * vs, loss, k, _abi.ptr(T12), 30, 1e-6,
              1e-6, _abi.ptr(ws), _abi.ptr(res), _abi.stream())
  with pytest.raises(_abi.DgrError, match='unknown loss'):
    gicp(6, 1.0, _abi.ptr(Cd), _abi.ptr(Cd))
  with pytest.raises(_abi.DgrError, match='unknown loss'):
    gicp(-1, 1.0, _abi.ptr(Cd), _abi.ptr(Cd))
  for a, b in ((0, _abi.ptr(Cd)), (_abi.ptr(Cd), 0)):
    with pytest.raises(_abi.DgrError, match='null pointer'):
      gicp(0, 1.0, a, b)
  with pytest.raises(_abi.DgrError, match='null pointer'):
    _abi.call('dgr_icp_loss', _abi.ptr(Pd), len(P), _abi.ptr(Qd), 0, _abi.ptr(spec), _abi.ptr(table.keys),
              _abi.ptr(table.vals), table.cap, 0, vs, 2 * vs, 5, 0.1, _abi.ptr(T12), 30, 1e-6, 1e-6, _abi.ptr(ws),
              _abi.ptr(res), _abi.stream())
  nrm = _t(np.tile([0.0, 0.0, 1.0], (10, 1)), torch.float32)
  for eps in (0.0, -1e-3, float('nan'), float('inf')):
    with pytest.raises(_abi.DgrError, match='epsilon'):
      _abi.covariances_from_normals(nrm, eps)
  with pytest.raises(_abi.DgrError):
    gpu_covariances(P, vs, 4.5 * vs, 30)
  with pytest.raises(_abi.DgrError):
    gpu_covariances(P, vs, 2 * vs, 65)
  with pytest.raises(_abi.DgrError, match='loss must be one of'):
    run_gicp(P, Cs, Q, Ct, vs, 2 * vs, T0, kernel=('Welsch', 1.0))


def test_stand_in_matches_direct_calls():
  from deepglobalregistration_b200 import _abi, shims
  from deepglobalregistration_b200 import o3d_registration as reg
  o3d = shims._open3d_stub()
  R = o3d.pipelines.registration
  x0, x1, T = syn.room_pair(0, n_raw=60000)
  vs = 0.05
  P, Q = voxelise(x0, vs), voxelise(x1, vs)
  T0 = syn.random_se3(np.random.default_rng(3), 3.0, 0.03) @ T
  src, tgt = o3d.geometry.PointCloud(), o3d.geometry.PointCloud()
  src.points, tgt.points = o3d.utility.Vector3dVector(P), o3d.utility.Vector3dVector(Q)
  hyb = o3d.geometry.KDTreeSearchParamHybrid(radius=2 * vs, max_nn=30)
  src.estimate_normals(hyb)
  tgt.estimate_normals(hyb)
  crit = R.ICPConvergenceCriteria(max_iteration=30)
  # from normals, with and without a kernel
  cell, spec, table = reg._target_hash(_t(Q, torch.float64), 2 * vs)
  cs = _abi.covariances_from_normals(_t(src.normals.astype(np.float32), torch.float32), 1e-3)
  ct = _abi.covariances_from_normals(_t(tgt.normals.astype(np.float32), torch.float32), 1e-3)
  for kernel, (loss, k) in ((None, (None, 1.0)), (R.TukeyLoss(2.0), ('Tukey', 2.0))):
    r = R.registration_generalized_icp(src, tgt, 2 * vs, T0, R.TransformationEstimationForGeneralizedICP(kernel=kernel),
                                       crit)
    want = _abi.icp_generalized(_t(P, torch.float32), cs, _t(Q, torch.float32), ct, (spec, table), cell, 2 * vs,
                                T0, loss=loss, loss_k=k).cpu().numpy()
    assert np.array_equal(r.transformation, want[:16].reshape(4, 4))
    assert (r.fitness, r.inlier_rmse, len(r.correspondence_set)) == (want[16], want[17], int(want[19]))
  te, re = syn.rte_rre(r.transformation, T)
  assert te < 0.02 and re < 0.02, (te, re)
  # covariances take precedence over normals; registration_icp then runs the same thing
  cell2, spec2, table2 = reg._target_hash(_t(P, torch.float64), 2 * vs)
  src.estimate_covariances(hyb)
  tgt.estimate_covariances(hyb)
  assert src.has_covariances() and np.array_equal(src.covariances, reg.estimate_covariances(P, hyb))
  cs2 = _abi.estimate_covariances(_t(P, torch.float32), (spec2, table2), cell2, 2 * vs, 30)
  ct2 = _abi.estimate_covariances(_t(Q, torch.float32), (spec, table), cell, 2 * vs, 30)
  want = _abi.icp_generalized(_t(P, torch.float32), cs2, _t(Q, torch.float32), ct2, (spec, table), cell, 2 * vs,
                              T0).cpu().numpy()
  for r in (R.registration_generalized_icp(src, tgt, 2 * vs, T0),
            R.registration_icp(src, tgt, 2 * vs, T0, R.TransformationEstimationForGeneralizedICP(), crit)):
    assert np.array_equal(r.transformation, want[:16].reshape(4, 4))
  # registration_icp point-to-plane with a kernel, and colored ICP with one
  nrm = _t(tgt.normals.astype(np.float32), torch.float32)
  r = R.registration_icp(src, tgt, 2 * vs, T0, R.TransformationEstimationPointToPlane(R.HuberLoss(0.02)), crit)
  want = _abi.icp_point_to_plane(_t(P, torch.float32), _t(Q, torch.float32), nrm, (spec, table), cell, 2 * vs, T0,
                                 loss='Huber', loss_k=0.02).cpu().numpy()
  assert np.array_equal(r.transformation, want[:16].reshape(4, 4))
  r_l2 = R.registration_icp(src, tgt, 2 * vs, T0, R.TransformationEstimationPointToPlane(R.L2Loss()), crit)
  r_no = R.registration_icp(src, tgt, 2 * vs, T0, R.TransformationEstimationPointToPlane(), crit)
  assert np.array_equal(r_l2.transformation, r_no.transformation)
  src.colors = np.full((len(P), 3), 0.5)
  tgt.colors = np.full((len(Q), 3), 0.5)
  c_l2 = R.registration_colored_icp(src, tgt, vs, T0, R.TransformationEstimationForColoredICP(kernel=R.L2Loss()),
                                    crit)
  c_no = R.registration_colored_icp(src, tgt, vs, T0, crit, 0.968)
  assert np.array_equal(c_l2.transformation, c_no.transformation)


def test_baseline_generalized():
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.icp_baseline import ICPBaseline
  import types
  vs = 0.05
  cfg = types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=vs), clip_weight_thresh=0.05, verbose=False)
  dgr = DeepGlobalRegistration(cfg, device=torch.device('cuda:0'))
  x0, x1, T = syn.room_pair(2, n_raw=60000)
  init = syn.random_se3(np.random.default_rng(0), 3.0, 0.03) @ T
  b = ICPBaseline(dgr, method='generalized', init=init)
  T_est = b.register(x0, x1)
  te, re = syn.rte_rre(T_est, T)
  print(f'ICPBaseline(generalized): {te:.4f} m, {re:.2e} rad, {b.last_info}')
  assert b.last_branch == 'icp_generalized' and te < 0.03 and re < 0.03
  assert b.last_info['icp_fitness'] > 0.5


def test_cli_icp_generalized(tmp_path, capsys):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200 import io as dio
  torch.save(syn.make_checkpoint(0, voxel_size=0.05), tmp_path / 'ckpt.pth')
  _, xyz1, _ = syn.room_pair(2, n_raw=20000, extent=(1.8, 1.5, 1.25))
  offset = syn.random_se3(np.random.default_rng(0), 2.0, 0.02)          # cloud 0: cloud 1 a little off the identity
  xyz0 = syn.apply_se3(offset, xyz1)
  T = np.linalg.inv(offset)
  dio.write_ply(tmp_path / 'a.ply', xyz0, dtype='double')
  dio.write_ply(tmp_path / 'b.ply', xyz1, dtype='double')
  (tmp_path / 'pairs.txt').write_text(f'a.ply b.ply {" ".join(repr(float(x)) for x in T.reshape(-1))} room\n')
  ev.main(['--pair_list', str(tmp_path / 'pairs.txt'), '--weights', str(tmp_path / 'ckpt.pth'), '--method',
           'icp_generalized', '--out_dir', str(tmp_path)])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  print(summary)
  assert summary['pairs'] == 1 and summary['with_ground_truth'] == 1
  saved = np.load(next(tmp_path.glob('*-stats.npz')), allow_pickle=True)
  te, re = syn.rte_rre(saved['poses'][0], T)
  assert te < 0.03 and re < 0.03, (te, re)
