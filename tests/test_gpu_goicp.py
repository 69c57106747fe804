"""dgr_goicp (Go-ICP) against oracle/goicp.py: the distance transform bit for bit, the restricted-domain searches
step for step, the full rotation domain where ICP from the identity fails, trimming, determinism, caps, argument
checks, the baseline and the evaluation entry point."""
import json
import math
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import goicp as og
from oracle import icp as oicp
from test_oracle_goicp import goicp_case

pytestmark = pytest.mark.gpu

FIELDS = og.RESULT


def _t(a):
  return torch.as_tensor(np.asarray(a, np.float32)).cuda().contiguous()


def run(src, tgt, **kw):
  from deepglobalregistration_b200 import _abi
  res = _abi.goicp(_t(src), _t(tgt), **kw).cpu().numpy()
  return res[:16].reshape(4, 4), dict(zip(FIELDS, res[16:29]))


def test_distance_transform_matches_the_oracle():
  from deepglobalregistration_b200 import _abi
  g = np.random.default_rng(0)
  clouds = [g.uniform(-1, 1, (5000, 3)), np.array([[0.2, -0.1, 0.3]]),
            np.array([[1.0, -1.0, 1.0], [-1.0, 1.0, 0.2], [0.0, 0.0, -1.0], [0.5, 0.5, 0.5]])]
  for y in clouds:
    y32 = y.astype(np.float32)
    for G, e in ((64, 2.0), (48, 1.5), (16, 1.0)):
      grid, s = _abi.goicp_distance_transform(_t(y32), G, e, src=_t(y32[:1024]))
      _, Y32, _, _, s_o = og.normalise(y32[:1024], y32)
      assert s == s_o
      assert np.array_equal(grid.cpu().numpy(), og.DistanceTransform(Y32, G, e).grid), (len(y), G, e)


@pytest.mark.parametrize('seed', [1, 2])
def test_restricted_domain_matches_the_oracle(seed):
  src, tgt, T_gt, rv = goicp_case(seed)
  hw = math.pi / 4
  kw = dict(dt_size=64, rot_min=rv - hw, rot_width=2 * hw, cubes_per_round=8)
  T, info = run(src, tgt, **kw)
  T_o, info_o = og.goicp(src, tgt, **kw)
  for k in ('rounds', 'children', 'translation_cubes', 'icp_runs', 'inner_overflows', 'converged', 'K',
            'pool_high_water', 'host_reads'):
    assert info[k] == info_o[k], (k, info, info_o)
  for k in ('E', 'lb_min', 'eps', 'scale'):
    assert abs(info[k] - info_o[k]) <= 1e-9 * abs(info_o[k]), (k, info[k], info_o[k])
  assert np.abs(T - T_o).max() <= 1e-6
  assert info['converged'] == 1 and info['E'] - info['lb_min'] < info['eps']
  te, re = syn.rte_rre(T, T_gt)
  assert re < math.radians(3) and te < 0.02 * 3.6, (te, re)                 # 64 cells of 18 cm


def full_case(seed, angle_deg):
  x = syn.room_scan(seed, 60000, (3.6, 3.0, 2.5), scene_seed=seed)
  y = syn.room_scan(seed + 50, 60000, (3.6, 3.0, 2.5), scene_seed=seed)
  g = np.random.default_rng(seed)
  axis = g.normal(size=3)
  axis /= np.linalg.norm(axis)
  T = syn.random_se3(g, 0.0, 0.3)
  from scipy.spatial.transform import Rotation
  T[:3, :3] = Rotation.from_rotvec(axis * math.radians(angle_deg)).as_matrix()
  src = x[np.arange(500) * len(x) // 500]
  tgt = syn.apply_se3(T, y[g.choice(len(y), 8000, replace=False)])
  return src.astype(np.float32), tgt.astype(np.float32), T


@pytest.mark.parametrize('seed,angle', [(3, 120.0), (4, 160.0)])
def test_full_rotation_domain_finds_the_global_optimum(seed, angle):
  src, tgt, T_gt = full_case(seed, angle)
  T_icp, _ = oicp.icp_point_to_point(src, tgt, 0.25)
  assert syn.rte_rre(T_icp, T_gt)[1] > math.radians(10)                      # ICP from the identity fails
  T, info = run(src, tgt, dt_size=128)
  te, re = syn.rte_rre(T, T_gt)
  print(f'\n[goicp] full domain, {angle} deg: {info}')
  assert info['converged'] == 1 and info['E'] - info['lb_min'] < info['eps'], info
  assert re < math.radians(2) and te < 0.02 * 3.6, (te, re, info)


def test_trimmed_partial_overlap():
  """rho = 0.3 against a target cropped to 70 % of the room, on a rotation domain of half-width pi/4 around the
  truth: the pose is recovered within 40 rounds (the certificate needs more), LB_min <= E* throughout."""
  src, tgt, T_gt, rv = goicp_case(1, n_s=160)
  back = syn.apply_se3(np.linalg.inv(T_gt), tgt)
  tgt = tgt[back[:, 0] > np.quantile(back[:, 0], 0.3)]
  hw = math.pi / 4
  T, info = run(src, tgt, trim_fraction=0.3, dt_size=64, rot_min=rv - hw, rot_width=2 * hw, cubes_per_round=8,
                max_rounds=40)
  te, re = syn.rte_rre(T, T_gt)
  print(f'\n[goicp] trimmed: {info}')
  assert info['K'] == 112 and info['lb_min'] <= info['E'] and info['rounds'] <= 40
  assert re < math.radians(2) and te < 0.02 * 3.6, (te, re, info)


def test_deterministic_and_caps():
  src, tgt, _, rv = goicp_case(2)
  hw = math.pi / 4
  kw = dict(dt_size=64, rot_min=rv - hw, rot_width=2 * hw, cubes_per_round=8)
  from deepglobalregistration_b200 import _abi
  a = _abi.goicp(_t(src), _t(tgt), **kw).cpu().numpy()
  b = _abi.goicp(_t(src), _t(tgt), **kw).cpu().numpy()
  assert np.array_equal(a, b)
  _, info = run(src, tgt, max_rounds=1, **kw)
  assert info['converged'] == 0 and info['rounds'] == 1 and info['lb_min'] <= info['E']
  _, info = run(src, tgt, max_rotation_cubes=64, **kw)
  assert info['converged'] == 0 and info['lb_min'] <= info['E'] and info['pool_high_water'] <= 64
  for trim in (0.0, 0.3):
    _, info = run(src, tgt, trim_fraction=trim, **kw)
    assert info['inner_overflows'] >= 0 and info['host_reads'] == info['rounds'] + 1


def test_bad_arguments_raise():
  from deepglobalregistration_b200 import _abi
  src, tgt, _, _ = goicp_case(1, n_s=64, n_t=200)
  big = np.zeros((1025, 3), np.float32)
  bad = [dict(src=big), dict(dt_size=15), dict(dt_size=513), dict(trim_fraction=1.0), dict(trim_fraction=-0.1),
         dict(mse_thresh=0.0), dict(rot_width=0.0), dict(trans_width=-1.0), dict(dt_expand=0.0),
         dict(cubes_per_round=0), dict(cubes_per_round=16, max_rotation_cubes=127)]
  for kw in bad:
    s = kw.pop('src', src)
    with pytest.raises(_abi.DgrError):
      _abi.goicp(_t(s), _t(tgt), **kw)
  with pytest.raises(_abi.DgrError):
    _abi.goicp(_t(src), _t(np.zeros((0, 3))))


def _dgr():
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  st = syn.make_checkpoint(4, voxel_size=0.0625)
  return DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))


def test_baseline_recovers_a_room_pair():
  from deepglobalregistration_b200.core.goicp import GoICPBaseline
  xyz0, xyz1, T_gt = syn.room_pair(3, n_raw=60_000)
  b = GoICPBaseline(_dgr())
  T = b.register(xyz0, xyz1)
  te, re = syn.rte_rre(T, T_gt)
  print(f'\n[goicp] baseline: {b.last_info}')
  assert b.last_branch == 'goicp' and b.last_info['n_data'] == 1000
  assert re < math.radians(3) and te < 0.1, (te, re, b.last_info)


def test_evaluate_goicp_on_a_pair_list(tmp_path, capsys):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200 import io as dio
  state = syn.make_checkpoint(0)
  torch.save(state, tmp_path / 'ckpt.pth')
  lines = []
  for k in range(2):
    xyz0, xyz1, T_gt = syn.room_pair(k, n_raw=30_000)
    np.savez(tmp_path / f'a{k}.npz', pcd=xyz0)
    dio.write_ply(tmp_path / f'b{k}.ply', xyz1, dtype='double')
    lines.append(f'a{k}.npz b{k}.ply {" ".join(repr(float(x)) for x in T_gt.reshape(-1))} room')
  (tmp_path / 'pairs.txt').write_text('\n'.join(lines) + '\n')
  ev.main(['--pair_list', str(tmp_path / 'pairs.txt'), '--weights', str(tmp_path / 'ckpt.pth'), '--out_dir',
           str(tmp_path), '--method', 'goicp', '--goicp_n_data', '500'])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  assert summary['pairs'] == 2 and summary['with_ground_truth'] == 2
  saved = np.load(tmp_path / 'goicp-b200-stats.npz', allow_pickle=True)
  assert list(saved['names']) == ['Go-ICP'] and saved['stats'].shape == (1, 2, 5)
