"""End-to-end and stage-isolated parity of DeepGlobalRegistration.register() against the
CPU oracle (oracle/pipeline.py) on small synthetic pairs.

Tolerances (north_star): voxel / correspondence indices bit-exact (correspondences outside
the fp64 ambiguity band), features / weights within 5e-5 relative, R,t within 1e-3 rad /
1e-3 m."""
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import pipeline as op
from oracle import registration as oreg

pytestmark = pytest.mark.gpu
EXTENT = (1.8, 1.5, 1.25)


@pytest.fixture(scope='module')
def state():
  return syn.make_checkpoint(0)


@pytest.fixture(scope='module')
def dgr(state):
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  cfg = types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False)
  d = DeepGlobalRegistration(cfg, device=torch.device('cuda'))
  assert d.use_icp is True           # reference default
  d.use_icp = False                  # these tests compare the pre-ICP pose ("tap A") unless stated
  return d


@pytest.fixture(scope='module')
def oracle_pair2(state):
  """Oracle run of the pair two tests share (seed 2), once: with ICP; the pre-ICP pose is a tap."""
  xyz0, xyz1, _ = syn.room_pair(2, n_raw=20000, extent=EXTENT)
  T_icp, taps = op.register(state, xyz0, xyz1, use_icp=True)
  return xyz0, xyz1, T_icp, taps


def _rel(got, want):
  got, want = got.detach().cpu().double(), want.detach().cpu().double()
  return float(((got - want).abs() / (1 + want.abs())).max())


def test_stage_isolated_parity(dgr, state):
  xyz0, xyz1, _ = syn.room_pair(0, n_raw=20000, extent=EXTENT)
  T_o, taps = op.register(state, xyz0, xyz1)
  with torch.no_grad():
    # stage 0: voxelisation - bit exact
    p0, c0, f0 = dgr.preprocess(xyz0, 0)
    sel0 = dgr._last_sel.cpu().numpy()
    p1, c1, f1 = dgr.preprocess(xyz1, 1)
    assert np.array_equal(sel0, taps['sel0'])
    assert np.array_equal(c0.cpu().numpy(), taps['coords0']) and np.array_equal(c1.cpu().numpy(), taps['coords1'])
    assert np.array_equal(p0.cpu().numpy(), taps['xyz0'])
    # stage 1: FCGF features
    F0 = dgr.fcgf_feature_extraction(f0, c0)
    F1 = dgr.fcgf_feature_extraction(f1, c1)
    assert _rel(F0, taps['feat0']) <= 5e-5 and _rel(F1, taps['feat1']) <= 5e-5
    # stage 2: kNN on the ORACLE's features - indices exact outside the ambiguity band
    i0, i1 = dgr.fcgf_feature_matching(taps['feat0'].cuda(), taps['feat1'].cuda())
    want, amb = oreg.feature_knn(taps['feat0'], taps['feat1'], return_ambiguous=True)
    assert i1.dtype == torch.int64 and torch.equal(i0.cpu(), torch.arange(len(want)))
    ok = (i1.cpu() == want) | amb
    assert bool(ok.all()), f'{int((~ok).sum())} kNN mismatches outside the ambiguity band'
    # stage 3/4: 6-D coords + inlier net on the ORACLE's correspondences
    from deepglobalregistration_b200 import _abi
    idx1 = torch.from_numpy(taps['idx1']).int().cuda()
    c6 = _abi.inlier_coords(c0, c1, idx1)
    assert np.array_equal(c6.cpu().numpy(), taps['coords6'])
    logit = dgr.inlier_prediction(torch.ones(len(idx1), 1, device='cuda'), c6)
    assert _rel(logit, taps['logit']) <= 5e-5
    # stage 5: registration on the ORACLE's weights
    w = taps['weights'].cuda().reshape(-1).contiguous()
    res = _abi.se3_register(p0, p1, w, idx1=idx1, quantization_size=2 * dgr.voxel_size,
                            break_threshold_ratio=1e-4).cpu().numpy()
  T = np.eye(4)
  T[:3, :3], T[:3, 3] = res[:9].reshape(3, 3), res[9:12]
  if taps['branch'] == 'procrustes':
    te, re = syn.rte_rre(T, T_o)
    assert te <= 1e-3 and re <= 1e-3, (te, re, res[12:], taps['refine'])


def test_register_known_answer_rigid_copy():
  """Cloud 1 = cloud 0 shifted by a multiple of 8 voxels - the coarsest tensor stride, so the
  strided lattices of both clouds align - with voxel = 2^-4 m so the shift is exact in
  binary: identical neighbourhoods give identical features, hence exact correspondences,
  hence the exact transform - provided the features have contrast, which a random-init
  checkpoint only has after BatchNorm calibration (util/calibrate.py)."""
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.util.calibrate import calibrate_batchnorm
  vs = 0.0625
  st = syn.make_checkpoint(4, voxel_size=vs)
  cfg = types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False)
  d = DeepGlobalRegistration(cfg)
  d.use_icp = False
  xyz0 = syn.room_scan(2, 20000, EXTENT, scene_seed=1)
  T_gt = np.eye(4)
  shift = np.array([8, -16, 24])
  T_gt[:3, 3] = vs * shift
  xyz1 = syn.apply_se3(T_gt, xyz0)
  with torch.no_grad():
    _, c0, f0 = d.preprocess(xyz0)
    calibrate_batchnorm(d.fcgf_model, ME.SparseTensor(f0, coordinates=c0, device='cuda'))
  st['state_dict'] = {k: v.detach().cpu().clone() for k, v in d.fcgf_model.state_dict().items()}
  T = d.register(xyz0, xyz1)
  assert d.last_branch == 'procrustes'
  te, re = syn.rte_rre(T, T_gt)
  assert te <= 1e-3 and re <= 1e-3, (te, re, d.last_info)
  T_o, taps = op.register(st, xyz0, xyz1)
  exact = (taps['coords1'][taps['idx1'], 1:] - taps['coords0'][:, 1:] == shift).all(1)
  assert exact.mean() > 0.99, exact.mean()
  te, re = syn.rte_rre(T, T_o)
  assert te <= 1e-3 and re <= 1e-3, (te, re)
  assert T.dtype == np.float64 and T.shape == (4, 4)


def test_register_end_to_end_vs_oracle(dgr, state, oracle_pair2):
  xyz0, xyz1, _, taps = oracle_pair2
  T = dgr.register(xyz0, xyz1)
  T_o = taps.get('T_refined', np.eye(4))          # the oracle's pose before ICP (tap A)
  assert dgr.last_branch == taps['branch']
  assert abs(dgr.last_info['wsum'] - taps['wsum']) <= 1e-3 * max(1.0, taps['wsum'])
  if taps['branch'] == 'procrustes':
    te, re = syn.rte_rre(T, T_o)
    # random-init features give ill-conditioned correspondences; the documented end-to-end
    # bar applies (1e-3 rad / 1e-3 m) and holds because every stage matches to ~1e-5.
    assert te <= 1e-3 and re <= 1e-3, (te, re, dgr.last_info, taps['refine'])


def test_register_float32_and_lidar_shape(dgr, state):
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  st = syn.make_checkpoint(3, voxel_size=0.3, feat_conv1_kernel_size=5)
  cfg = types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False)
  d = DeepGlobalRegistration(cfg)
  d.use_icp = False
  xyz0, xyz1, _ = syn.lidar_pair(0)
  xyz0, xyz1 = xyz0[::4].astype(np.float32), xyz1[::4].astype(np.float32)
  with torch.no_grad():
    p0, c0, _ = d.preprocess(xyz0)
  oc, osel = op.so.quantize_first(xyz0, 0.3)
  assert np.array_equal(c0.cpu().numpy()[:, 1:], oc)
  T = d.register(xyz0, xyz1)
  T_o, taps = op.register(st, xyz0, xyz1)
  assert d.last_branch == taps['branch']
  if taps['branch'] == 'procrustes':
    te, re = syn.rte_rre(T, T_o)
    assert te <= 1e-3 and re <= 1e-3, (te, re)


def test_checkpoint_file_boundary(tmp_path, state):
  """A checkpoint written with torch.save in the reference's layout (state_dict,
  state_dict_inlier, pickled attribute-dict config; core/trainer.py:527-549) loads through
  config.weights = <path> exactly like the in-memory dict."""
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  path = tmp_path / 'ckpt.pth'
  torch.save(state, path)
  cfg = types.SimpleNamespace(weights=str(path), clip_weight_thresh=0.05, verbose=False)
  d = DeepGlobalRegistration(cfg)
  assert d.voxel_size == state['config']['voxel_size'] and cfg.inlier_feature_type == 'ones'
  for k, v in state['state_dict'].items():
    assert torch.equal(d.fcgf_model.state_dict()[k].cpu(), v), k
  xyz0, xyz1, _ = syn.room_pair(5, n_raw=6000, extent=(1.2, 1.0, 0.8))
  T = d.register(xyz0, xyz1)
  assert T.shape == (4, 4) and np.isfinite(T).all()


@pytest.mark.parametrize('n_raw', [1, 3, 40, 300])
def test_register_tiny_clouds(dgr, state, n_raw):
  """Degenerate sizes: single voxels, fewer voxels than one 128-row tile, empty coarse
  neighbourhoods.  The weight-sum gate (>= 200) sends these to the safeguard branch (RANSAC on
  a handful of correspondences, mostly degenerate draws), which must return a rigid pose, not
  crash; every stage before it must still agree with the oracle."""
  g = np.random.default_rng(n_raw)
  xyz0 = g.uniform(0, 0.6, size=(n_raw, 3))
  xyz1 = xyz0 + 0.05
  dgr.safeguard_max_iteration = 20000
  try:
    T = dgr.register(xyz0, xyz1)
  finally:
    dgr.safeguard_max_iteration = 4000000
  T_o, taps = op.register(state, xyz0, xyz1)
  assert dgr.last_branch == taps['branch'] == 'safeguard'
  R = T[:3, :3]
  assert np.allclose(R @ R.T, np.eye(3), atol=1e-9) and abs(np.linalg.det(R) - 1) < 1e-9
  assert np.array_equal(T[3], [0, 0, 0, 1]) and dgr.last_info['ransac_inliers'] >= 1
  assert dgr.last_info['n0'] == len(taps['coords0'])
  assert abs(dgr.last_info['wsum'] - taps['wsum']) <= 1e-3 * max(1.0, taps['wsum'])


def test_preprocess_rejects_unknown_input(dgr):
  with pytest.raises(Exception, match='Unrecognized pcd type'):
    dgr.preprocess('not a point cloud')


def test_unbuilt_stages_fail_loudly(dgr):
  dgr.safeguard_method = 'fcgf_feature_matching'
  try:
    with pytest.raises(NotImplementedError):
      dgr.safeguard_registration(None, None, None, None, None, None, 0.1, 80000)
  finally:
    dgr.safeguard_method = 'correspondence'


def test_safeguard_branch_known_answer():
  """Force the weight-sum gate shut (clip threshold 1 zeroes every weight) on the rigid-copy
  pair: the safeguard's RANSAC over the (exact) correspondences, then ICP, must recover the
  shift; the oracle's safeguard on the same hypotheses agrees."""
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.util.calibrate import calibrate_batchnorm
  vs = 0.0625
  st = syn.make_checkpoint(4, voxel_size=vs)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=1.0, verbose=False))
  xyz0 = syn.room_scan(2, 20000, EXTENT, scene_seed=1)
  T_gt = np.eye(4)
  T_gt[:3, 3] = vs * np.array([8, -16, 24])
  xyz1 = syn.apply_se3(T_gt, xyz0)
  with torch.no_grad():
    _, c0, f0 = d.preprocess(xyz0)
    calibrate_batchnorm(d.fcgf_model, ME.SparseTensor(f0, coordinates=c0, device='cuda'))
  st['state_dict'] = {k: v.detach().cpu().clone() for k, v in d.fcgf_model.state_dict().items()}
  d.safeguard_max_iteration, d.safeguard_seed = 3000, 11
  for use_icp in (False, True):
    d.use_icp = use_icp
    T = d.register(xyz0, xyz1)
    assert d.last_branch == 'safeguard' and d.last_info['wsum'] == 0.0
    te, re = syn.rte_rre(T, T_gt)
    assert te <= 1e-3 and re <= 1e-3, (use_icp, te, re, d.last_info)
    assert d.last_info['ransac_fitness'] > 0.99
  T_o, taps = op.register(st, xyz0, xyz1, clip_weight_thresh=1.0, use_icp=True, safeguard_max_iteration=3000,
                          safeguard_seed=11)
  assert taps['branch'] == 'safeguard'
  te, re = syn.rte_rre(T, T_o)
  assert te <= 1e-3 and re <= 1e-3, (te, re, taps['ransac'], taps.get('icp'))
  # the public method, called the way the reference calls it (:302-311)
  with torch.no_grad():
    p0, _, _ = d.preprocess(xyz0, 0, _batch=0)
    p1, _, _ = d.preprocess(xyz1, 1, _batch=1)
  T_s = d.safeguard_registration(p0, p1, np.arange(len(taps['idx1'])), taps['idx1'], None, None, 2 * vs,
                                 num_iterations=80000)
  np.testing.assert_allclose(T_s, taps['T_ransac'], atol=1e-6)


def test_icp_kernel_vs_oracle():
  """dgr_icp (point-to-point) against the open3d restatement (oracle/icp.py): same pose to 1e-6,
  same fitness / RMSE / iteration count, from a perturbed initial pose."""
  from deepglobalregistration_b200 import _abi
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from oracle.icp import icp_point_to_point
  st = syn.make_checkpoint(0, with_inlier=True)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))
  g = np.random.default_rng(0)
  xyz0 = syn.room_scan(3, 30000, EXTENT)
  T_gt = syn.random_se3(g, 20.0, 0.3)
  xyz1 = syn.apply_se3(T_gt, syn.room_scan(4, 30000, EXTENT, scene_seed=3))
  with torch.no_grad():
    p0, c0, _ = d.preprocess(xyz0, 0, _batch=0)
    p1, c1, _ = d.preprocess(xyz1, 1, _batch=1)
  for trial, (ang, tr) in enumerate(((0.0, 0.0), (2.0, 0.03), (6.0, 0.08))):
    T_init = syn.random_se3(np.random.default_rng(10 + trial), ang, tr) @ T_gt if ang else T_gt.copy()
    res = _abi.icp_point_to_point(p0, p1, c1._dgr_manager, 0.05, 0.1, T_init, batch=1).cpu().numpy()
    T_o, info = icp_point_to_point(p0.cpu().numpy(), p1.cpu().numpy(), 0.1, T_init)
    te, re = syn.rte_rre(res[:16].reshape(4, 4), T_o)
    assert te <= 1e-5 and re <= 1e-5, (trial, te, re, res[16:], info)
    assert abs(res[16] - info['fitness']) <= 2e-4 and abs(res[17] - info['inlier_rmse']) <= 1e-5
    assert abs(int(res[18]) - info['iterations']) <= 1, (res[18], info)
  # the refined pose gets closer to the ground truth than the perturbed start
  te_i, re_i = syn.rte_rre(T_init, T_gt)
  te_f, re_f = syn.rte_rre(res[:16].reshape(4, 4), T_gt)
  assert te_f < te_i and re_f < re_i


def test_register_with_icp_vs_oracle(state, oracle_pair2):
  """Tap B: the literal return value of the reference's register() (use_icp = True)."""
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False))
  xyz0, xyz1, T_o, taps = oracle_pair2
  T = d.register(xyz0, xyz1)
  assert d.last_branch == taps['branch'] == 'procrustes'
  te, re = syn.rte_rre(T, T_o)
  assert te <= 1e-3 and re <= 1e-3, (te, re, d.last_info, taps['icp'])
  assert abs(d.last_info['icp_fitness'] - taps['icp']['fitness']) <= 5e-3
