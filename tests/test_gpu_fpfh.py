"""dgr_compute_fpfh (open3d 0.10's ComputeFPFHFeature) against oracle/fpfh.py, the open3d stand-in's
compute_fpfh_feature, and the FPFH + RANSAC / FPFH + FGR baselines against the oracle chain oracle/fpfh.py -> float64
nearest feature -> oracle/ransac_fm.py / oracle/fgr.py.  The oracle is fed the GPU's own float32 normals, so only the
FPFH stage is compared: neighbour lists and counts exactly, and every row outside the ambiguity band bit for bit."""
import importlib.util
import json
import os
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import fgr as ofg
from oracle import fpfh as ofp
from oracle import ransac_fm as orf
from oracle import registration as oreg
from test_gpu_fgr import rotation_angle
from test_gpu_icp_plane import _t, cloud_hash, voxelise
from test_gpu_ransac_fm import EXTENT, check_against_oracle

pytestmark = pytest.mark.gpu


def gpu_normals(P, cell, radius=None, max_nn=30):
  from deepglobalregistration_b200 import _abi
  radius = 2 * cell if radius is None else radius
  return _abi.estimate_normals(_t(P, torch.float32), cloud_hash(P, cell), cell, radius, max_nn)


def gpu_fpfh(P, nrm, cell, radius, max_nn, ld=33, hashed=None):
  from deepglobalregistration_b200 import _abi
  f, counts = _abi.compute_fpfh(_t(P, torch.float32), nrm, hashed or cloud_hash(P, cell), cell, radius, max_nn, ld=ld,
                                return_counts=True)
  return f.cpu().numpy(), counts.cpu().numpy()


def check_parity(name, P, cell, radius, max_nn, nrm=None):
  """GPU FPFH against the oracle on the GPU's normals -> the oracle's output (ambiguous fraction printed)."""
  nrm = gpu_normals(P, cell) if nrm is None else nrm
  f, counts = gpu_fpfh(P, nrm, cell, radius, max_nn)
  o = ofp.compute_fpfh(P, nrm.cpu().numpy().astype(np.float64), radius, max_nn)
  assert np.array_equal(counts, o['counts']), name
  ok = ~o['ambiguous']
  want = o['fpfh'].astype(np.float32)
  bad = ok & np.any(f.view(np.uint32) != want.view(np.uint32), axis=1)
  assert not bad.any(), (name, int(bad.sum()), np.flatnonzero(bad)[:5])
  print(f'\n[fpfh] {name}: n {len(P)}, reach {int(np.ceil(radius / cell))}, max_nn {max_nn}, '
        f'max count {counts.max()}, ambiguous {1 - ok.mean():.4f}')
  return o, f


def test_room_matches_the_oracle():
  P = voxelise(syn.room_pair(1, n_raw=30000, extent=EXTENT)[0], 0.05)
  o, _ = check_parity('room', P, 0.05, 0.25, 100)
  assert (o['counts'] > 100).any() and (~o['ambiguous']).mean() > 0.9


def test_noise_free_box_exercises_the_band():
  """Flat faces without noise, half the normals flipped: coplanar pairs with n2 = -n1 put alpha on the +-pi wrap."""
  P = voxelise(syn.room_scan(3, 30000, EXTENT, scene_seed=3, noise=0.0), 0.05)
  nrm = gpu_normals(P, 0.05)
  flip = torch.from_numpy(np.random.default_rng(0).random(len(P)) < 0.5).cuda()
  nrm = torch.where(flip[:, None], -nrm, nrm).contiguous()
  o, _ = check_parity('noise-free box, half the normals flipped', P, 0.05, 0.25, 100, nrm=nrm)
  assert o['ambiguous'].any()


def dense_cloud(seed, side=12, cell=0.0625):
  """Uniform points in a cube of side^3 cells, one kept per cell: about 60 % of the cells filled."""
  g = np.random.default_rng(seed)
  return voxelise(g.uniform(0.0, side * cell, size=(side ** 3, 3)), cell)


@pytest.mark.parametrize('max_nn', [2, 30, 100, 128])
@pytest.mark.parametrize('reach', [1, 2, 3, 4, 5, 6])
def test_dense_clouds_match_the_oracle(reach, max_nn):
  cell = 0.0625
  P = dense_cloud(reach * 10 + max_nn)
  radius = reach * cell if reach > 1 else 0.9 * cell
  o, _ = check_parity(f'dense reach {reach}', P, cell, radius, max_nn)
  if reach >= 2 and max_nn <= 30:
    assert (o['counts'] > max_nn).any()                 # the selection path runs


def test_isolated_points_and_padding():
  cell = 0.0625
  P = dense_cloud(7)
  far = np.array([[3.0, 3.0, 3.0], [4.0, 3.0, 3.0], [3.0, 4.0, 3.25]])
  P = np.vstack([P, far]).astype(np.float32).astype(np.float64)
  nrm = gpu_normals(P, cell)
  o, f = check_parity('isolated', P, cell, 3 * cell, 30, nrm=nrm)
  assert np.array_equal(o['counts'][-3:], [1, 1, 1]) and not f[-3:].any()
  # two calls give the same bytes; ld = 64 pads with zero columns
  f2, _ = gpu_fpfh(P, nrm, cell, 3 * cell, 30)
  f64, _ = gpu_fpfh(P, nrm, cell, 3 * cell, 30, ld=64)
  assert f.tobytes() == f2.tobytes()
  assert f64.shape == (len(P), 64) and np.array_equal(f64[:, :33], f) and not f64[:, 33:].any()


def test_padded_rows_feed_the_tensor_core_knn():
  from deepglobalregistration_b200 import _abi
  cell = 0.05
  P = voxelise(syn.room_pair(2, n_raw=20000, extent=EXTENT)[0], cell)
  Q = voxelise(syn.room_pair(2, n_raw=20000, extent=EXTENT)[1], cell)
  rows = []
  for X in (P, Q):
    nrm = gpu_normals(X, cell)
    f64 = _abi.compute_fpfh(_t(X, torch.float32), nrm, cloud_hash(X, cell), cell, 5 * cell, 100, ld=64)
    rows.append(f64)
  a, b = rows
  assert _abi.lib().dgr_knn_tc_supported(64)
  tc = _abi.knn_top1(a, b, mode='tc')
  simt = _abi.knn_top1(a[:, :33].contiguous(), b[:, :33].contiguous(), mode='simt')
  assert torch.equal(tc, simt)
  tc_r = _abi.knn_top1(b, a, mode='tc')
  assert torch.equal(tc_r, _abi.knn_top1(b[:, :33].contiguous(), a[:, :33].contiguous(), mode='simt'))


def test_bad_arguments():
  from deepglobalregistration_b200 import _abi
  cell = 0.0625
  P = dense_cloud(3)
  nrm = gpu_normals(P, cell)
  xyz, h = _t(P, torch.float32), cloud_hash(P, cell)
  for kw in (dict(radius=6.5 * cell), dict(max_nn=129), dict(max_nn=0), dict(ld=32), dict(radius=0.0)):
    args = dict(radius=3 * cell, max_nn=30, ld=33)
    args.update(kw)
    with pytest.raises(_abi.DgrError):
      _abi.compute_fpfh(xyz, nrm, h, cell, args['radius'], args['max_nn'], ld=args['ld'])
  with pytest.raises(_abi.DgrError, match='normals'):
    _abi.compute_fpfh(xyz, None, h, cell, 3 * cell, 30)
  _abi.compute_fpfh(xyz, nrm, h, cell, 6 * cell, 128)     # the largest reach and max_nn run


def test_stand_in_compute_fpfh_feature():
  from deepglobalregistration_b200 import _abi, shims
  from deepglobalregistration_b200 import o3d_registration as reg
  o3d = shims._open3d_stub()
  vs = 0.05
  P = voxelise(syn.room_pair(3, n_raw=20000, extent=EXTENT)[0], vs)
  pcd = o3d.geometry.PointCloud()
  pcd.points = o3d.utility.Vector3dVector(P)
  with pytest.raises(RuntimeError, match='normals'):
    o3d.pipelines.registration.compute_fpfh_feature(pcd, o3d.geometry.KDTreeSearchParamHybrid(radius=5 * vs, max_nn=100))
  pcd.estimate_normals(o3d.geometry.KDTreeSearchParamHybrid(radius=2 * vs, max_nn=30))
  cell, spec, table = reg._target_hash(_t(P, torch.float64), 5 * vs, max_reach=6)
  assert np.ceil(5 * vs / cell) <= 6
  want = _abi.compute_fpfh(_t(P, torch.float32), _t(pcd.normals, torch.float32), (spec, table), cell, 5 * vs,
                           100).cpu().numpy()
  for module in (o3d.pipelines.registration, o3d.registration):
    feat = module.compute_fpfh_feature(pcd, o3d.geometry.KDTreeSearchParamHybrid(radius=5 * vs, max_nn=100))
    assert isinstance(feat, reg.Feature) and feat.data.dtype == np.float64 and feat.data.shape == (33, len(P))
    assert feat.dimension() == 33 and feat.num() == len(P)
    assert np.array_equal(feat.data, want.T.astype(np.float64))
  compute = o3d.pipelines.registration.compute_fpfh_feature
  with pytest.raises(NotImplementedError):
    compute(pcd, o3d.geometry.KDTreeSearchParamKNN(30))
  with pytest.raises(NotImplementedError):
    compute(pcd, o3d.geometry.KDTreeSearchParamRadius(5 * vs))
  for bad in (dict(radius=5 * vs, max_nn=129), dict(radius=5 * vs, max_nn=0), dict(radius=0.0, max_nn=100)):
    with pytest.raises(ValueError):
      compute(pcd, o3d.geometry.KDTreeSearchParamHybrid(**bad))
  compute(pcd, o3d.geometry.KDTreeSearchParamHybrid(radius=5 * vs, max_nn=128))
  # two points in one cell at radius / 6: no one-point-per-cell hash exists
  dup = o3d.geometry.PointCloud()
  dup.points = o3d.utility.Vector3dVector(np.vstack([P, P[:1]]))
  dup.normals = np.vstack([pcd.normals, pcd.normals[:1]])
  with pytest.raises(NotImplementedError, match='radius / 6'):
    compute(dup, o3d.geometry.KDTreeSearchParamHybrid(radius=5 * vs, max_nn=100))


def _dgr(vs=0.05):
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  return DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=vs),
                                                      clip_weight_thresh=0.05, verbose=False))


def oracle_chain(d, method, xyz0, xyz1):
  """The stage inputs the baseline sees (voxelised points, GPU normals) -> oracle FPFH -> float64 nearest features.
  -> (P, Q, nn_st, nn_ts, clean): clean = no ambiguous FPFH row and no nearest feature in the top-2 gap band."""
  from deepglobalregistration_b200 import _abi
  vs = d.voxel_size
  feats, pts, clean = [], [], True
  with torch.no_grad():
    for batch, xyz in enumerate((xyz0, xyz1)):
      p, c, _ = d.preprocess(xyz, batch, _batch=batch)
      nrm = _abi.estimate_normals(p, c._dgr_manager, vs, method.normal_radius_voxels * vs, method.normal_max_nn,
                                  batch=batch)
      P = p.cpu().numpy().astype(np.float64)
      o = ofp.compute_fpfh(P, nrm.cpu().numpy().astype(np.float64), method.feature_radius_voxels * vs,
                           method.feature_max_nn)
      clean &= not o['ambiguous'].any()
      feats.append(o['fpfh'].astype(np.float32))
      pts.append(P)
  nn_st, nn_ts = orf.feature_nn(feats[0], feats[1]), orf.feature_nn(feats[1], feats[0])
  clean &= not (oreg.feature_knn(feats[0], feats[1], return_ambiguous=True)[1].any() or
                oreg.feature_knn(feats[1], feats[0], return_ambiguous=True)[1].any())
  return pts[0], pts[1], nn_st, nn_ts, clean


CHAIN_SEEDS = (1, 2, 3, 4, 5)


def test_baselines_match_the_oracle_chain():
  from deepglobalregistration_b200.core.fpfh_baseline import FPFHFastGlobal, FPFHRansac
  d = _dgr()
  d.use_icp = False
  ransac, fgr = FPFHRansac(d), FPFHFastGlobal(d)
  assert (ransac.max_iteration, ransac.max_validation, ransac.edge_ratio) == (80000, 1000, 0.0)
  vs = d.voxel_size
  checked = 0
  for seed in CHAIN_SEEDS:
    xyz0, xyz1, T_gt = syn.room_pair(seed, n_raw=20000, extent=EXTENT)
    P, Q, nn_st, nn_ts, clean = oracle_chain(d, ransac, xyz0, xyz1)
    print(f'\n[fpfh chain] seed {seed}: n {len(P)} / {len(Q)}, clean {clean}')
    if not clean:
      continue
    assert len(P) <= 10000 and len(Q) <= 10000
    T = ransac.register(xyz0, xyz1)
    i = ransac.last_info
    res = np.concatenate([T.reshape(-1), [i['ransac_fitness'], i['ransac_inlier_rmse'], i['ransac_hypothesis'],
                                          i['ransac_inliers'], i['ransac_validated'], i['ransac_drawn']]])
    check_against_oracle(res, P, Q, nn_st, 2 * vs, 80000, 1000, 0, check_dist=2 * vs)
    T = fgr.register(xyz0, xyz1)
    T_o, info = ofg.fgr(P, Q, nn_st, nn_ts, seed=0)
    i = fgr.last_info
    assert (i['fgr_mutual'], i['fgr_correspondences'], i['fgr_trials']) == (info['n_mut'], info['n_corr'],
                                                                            info['drawn'])
    te, re = np.linalg.norm(T[:3, 3] - T_o[:3, 3]), rotation_angle(T[:3, :3], T_o[:3, :3])
    assert te <= 1e-8 and re <= 1e-8, (seed, te, re)
    checked += 1
  assert checked >= 1


# room pairs (n_raw 40000, voxel 0.05 m) on which the CPU oracle chain (oracle normals -> oracle/fpfh.py -> float64
# nearest features -> oracle/ransac_fm.py and oracle/fgr.py, no ICP) meets the 0.3 m / 15 deg criterion with both
# searches
ACCURACY_SEEDS = (0, 1, 2, 3, 4)


@pytest.mark.parametrize('seed', ACCURACY_SEEDS)
def test_baselines_register_room_pairs(seed):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200.core.fpfh_baseline import FPFHFastGlobal, FPFHRansac
  d = _dgr()
  d.use_icp = True
  xyz0, xyz1, T_gt = syn.room_pair(seed, n_raw=40000, extent=EXTENT)
  for cls in (FPFHRansac, FPFHFastGlobal):
    method = cls(d)
    T = method.register(xyz0, xyz1)
    ok, rte, rre = ev.rte_rre(T, T_gt, 0.3, 15.0)
    print(f'\n[fpfh accuracy] {method.label}, seed {seed}: RTE {rte:.4f} m, RRE {rre:.3f} deg')
    assert ok == 1.0, (method.label, seed, rte, rre, method.last_info)
    assert 'icp_fitness' in method.last_info


def test_evaluate_fpfh_methods_on_a_pair_list(tmp_path, capsys):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200 import io as dio
  torch.save(syn.make_checkpoint(0), tmp_path / 'ckpt.pth')
  xyz0, xyz1, T_gt = syn.room_pair(2, n_raw=20000, extent=EXTENT)
  dio.write_ply(tmp_path / 'a.ply', xyz0, dtype='double')
  dio.write_ply(tmp_path / 'b.ply', xyz1, dtype='double')
  (tmp_path / 'pairs.txt').write_text(f'a.ply b.ply {" ".join(repr(float(x)) for x in T_gt.reshape(-1))} room\n'
                                      'a.ply b.ply\n')
  for method, stem, name in (('fpfh_ransac', 'fpfh-ransac-b200', 'FPFH + RANSAC'),
                             ('fpfh_fgr', 'fpfh-fgr-b200', 'FPFH + FGR')):
    ev.main(['--pair_list', str(tmp_path / 'pairs.txt'), '--weights', str(tmp_path / 'ckpt.pth'), '--out_dir',
             str(tmp_path), '--method', method, '--ransac_max_iteration', '20000', '--ransac_max_validation', '300'])
    summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert summary['pairs'] == 2 and summary['with_ground_truth'] == 1 and 'recall' in summary
    saved = np.load(tmp_path / f'{stem}-stats.npz', allow_pickle=True)
    assert list(saved['names']) == [name] and saved['stats'].shape == (1, 2, 5)
    for T in saved['poses']:
      assert np.allclose(T[:3, :3] @ T[:3, :3].T, np.eye(3), atol=1e-9) and np.array_equal(T[3], [0, 0, 0, 1])


def test_dgr_pair_size_time():
  """Per-pass times at the DGR pair size (tools/fpfh_bench.py); prints, asserts nothing about speed."""
  path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools', 'fpfh_bench.py')
  spec = importlib.util.spec_from_file_location('fpfh_bench', path)
  bench = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(bench)
  out = bench.measure(reps=3)
  print(f'\n[fpfh timing] {json.dumps(out)}')
  assert out['n0'] == 51381 and out['n1'] == 39881, out
