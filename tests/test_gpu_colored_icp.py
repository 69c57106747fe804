"""dgr_color_gradient and dgr_colored_icp (open3d's colour gradient and colored ICP) against oracle/colored_icp.py,
the open3d stand-in's registration_colored_icp, and multi-scale colored ICP refinement in multiway registration.
Neighbour counts are compared exactly (both sides evaluate d^2 with the same rounding); gradients and poses to
round-off, since the sums run in a different order on the GPU."""
import json

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import synthetic as syn
from oracle import colored_icp as oc
from test_gpu_fgr import rotation_angle
from test_gpu_icp_plane import _t, cloud_hash, gpu_normals, run_plane
from test_oracle_colored_icp import WALL_COLORED_LEFT, WALL_P2PLANE_LEFT, WALL_VOXEL, wall_case

pytestmark = pytest.mark.gpu

PIVOT_EXCLUDE = 1e-6      # gradients whose smallest Cholesky pivot is below this share of the diagonal are not compared


def coloured_fragment(k, vs):
  """Fragment k of the coloured room (float32-representable, first point per cell of `vs`) and its intensities."""
  clouds, cols, _ = syn.room_fragments(0, n_frag=6, n_raw=60000, colours=True)
  x32 = np.asarray(clouds[k], np.float32).astype(np.float64)
  _, first = np.unique(np.floor(x32 / vs).astype(np.int64), axis=0, return_index=True)
  first = np.sort(first)
  return x32[first], oc.intensity(cols[k][first]).astype(np.float32)


def gpu_gradient(P, nrm, inten, cell, radius, max_nn, hashed=None):
  from deepglobalregistration_b200 import _abi
  g, c = _abi.color_gradient(_t(P, torch.float32), _t(nrm, torch.float32), _t(inten, torch.float32),
                             hashed or cloud_hash(P, cell), cell, radius, max_nn, return_counts=True)
  return g.cpu().numpy().astype(np.float64), c.cpu().numpy()


def run_colored(P, I_P, Q, nrm, I_Q, grad, vs, max_dist, T_init, lam=oc.LAMBDA_GEOMETRIC, max_iter=30, hashed=None):
  from deepglobalregistration_b200 import _abi
  return _abi.icp_colored(_t(P, torch.float32), _t(I_P, torch.float32), _t(Q, torch.float32), _t(nrm, torch.float32),
                          _t(I_Q, torch.float32), _t(grad, torch.float32), hashed or cloud_hash(Q, vs), vs, max_dist,
                          lam, T_init, max_iter).cpu().numpy()


@pytest.mark.parametrize('ratio', [2, 4])
def test_gradient_matches_the_oracle(ratio):
  vs = 0.05
  P, inten = coloured_fragment(0, vs)
  radius = ratio * vs
  nrm, _ = gpu_normals(P, vs, radius, 30)
  nrm32 = nrm.astype(np.float32)
  g, counts = gpu_gradient(P, nrm32, inten, vs, radius, 30)
  g_o, c_o, pivot = oc.color_gradient(P, nrm32, inten, radius, 30)
  assert np.array_equal(counts, c_o)
  assert ratio == 2 or (counts > 30).any()                               # max_nn truncation active at ratio 4
  ok = pivot > PIVOT_EXCLUDE
  zero = np.minimum(counts, 30) < 4
  assert np.array_equal(g[zero], np.zeros((zero.sum(), 3)))
  scale = np.maximum(np.linalg.norm(g_o, axis=1), 1e-3)
  err = np.linalg.norm(g - g_o.astype(np.float32), axis=1) / scale
  print(f'ratio {ratio}: {len(P)} points, {int((~ok & ~zero).sum())} excluded by pivot, {int(zero.sum())} with < 4 '
        f'neighbours, max relative error {err[ok].max():.3g}')
  # float32 output: compare the oracle's value rounded to float32 at a relative 1e-9 of the fp64 quantities, plus one
  # float32 rounding of the result
  assert np.all(err[ok] <= 1e-9 + 2.0 ** -23), np.sort(err[ok])[-5:]
  assert ok.mean() > 0.9
  g2, c2 = gpu_gradient(P, nrm32, inten, vs, radius, 30)
  assert np.array_equal(g, g2) and np.array_equal(counts, c2)


def colored_case(seed=0, vs=0.05):
  """Fragments 0 and 1 of the coloured room, the GPU's target normals and gradients at radius 2 vs, and a start a
  few degrees / cm off the true relative pose."""
  _, _, poses = syn.room_fragments(0, n_frag=6, n_raw=60000, colours=True)
  P, I_P = coloured_fragment(0, vs)
  Q, I_Q = coloured_fragment(1, vs)
  T_gt = np.linalg.inv(poses[1]) @ poses[0]
  T_init = syn.random_se3(np.random.default_rng(seed), 3.0, 0.03) @ T_gt
  nrm = gpu_normals(Q, vs, 2 * vs, 30)[0].astype(np.float32)
  grad = gpu_gradient(Q, nrm, I_Q, vs, 2 * vs, 30)[0].astype(np.float32)
  return P, I_P, Q, I_Q, nrm, grad, T_init, T_gt, vs


def test_colored_icp_matches_the_oracle():
  P, I_P, Q, I_Q, nrm, grad, T_init, T_gt, vs = colored_case()
  for max_iter in (30, 3):
    res = run_colored(P, I_P, Q, nrm, I_Q, grad, vs, vs, T_init, max_iter=max_iter)
    T_o, info = oc.colored_icp(P, I_P, Q, nrm, I_Q, grad, vs, T_init, max_iter=max_iter)
    assert (int(res[18]), int(res[19])) == (info['iterations'], info['n_corr']), (res[16:], info)
    assert abs(res[16] - info['fitness']) <= 1e-9 and abs(res[17] - info['inlier_rmse']) <= 1e-9
    T = res[:16].reshape(4, 4)
    assert np.array_equal(T[3], [0, 0, 0, 1]) and np.all(np.isfinite(T))
    assert np.linalg.norm(T[:3, 3] - T_o[:3, 3]) <= 1e-7 and rotation_angle(T[:3, :3], T_o[:3, :3]) <= 1e-7
  te, re = syn.rte_rre(run_colored(P, I_P, Q, nrm, I_Q, grad, vs, vs, T_init)[:16].reshape(4, 4), T_gt)
  assert te < 0.02 and re < 0.02, (te, re)
  hashed = cloud_hash(Q, vs)
  a = run_colored(P, I_P, Q, nrm, I_Q, grad, vs, vs, T_init, hashed=hashed)
  b = run_colored(P, I_P, Q, nrm, I_Q, grad, vs, vs, T_init, hashed=hashed)
  assert np.array_equal(a, b)


def test_lambda_one_is_point_to_plane():
  P, I_P, Q, I_Q, nrm, grad, T_init, _, vs = colored_case(1)
  c = run_colored(P, I_P, Q, nrm, I_Q, grad, vs, 2 * vs, T_init, lam=1.0)
  p = run_plane(P, Q, nrm, vs, 2 * vs, T_init)
  assert (int(c[18]), int(c[19])) == (int(p[18]), int(p[19]))
  assert np.abs(c[:16] - p[:16]).max() <= 1e-12 and c[16] == p[16]


def test_sliding_wall():
  P, I_P, Q, I_Q, nrm_o, T0 = wall_case()
  vs = WALL_VOXEL
  nrm = gpu_normals(Q, vs, 2 * vs, 30)[0].astype(np.float32)
  grad = gpu_gradient(Q, nrm, I_Q, vs, 2 * vs, 30)[0].astype(np.float32)
  p = run_plane(P, Q, nrm, vs, vs, T0)
  c = run_colored(P, I_P, Q, nrm, I_Q, grad, vs, vs, T0)
  left_p, left_c = np.linalg.norm(p[3:12:4]), np.linalg.norm(c[3:12:4])
  print(f'sliding wall: point-to-plane leaves {left_p:.4f} m, colored ICP {left_c:.4f} m')
  assert left_p >= WALL_P2PLANE_LEFT and left_c <= WALL_COLORED_LEFT


def test_argument_checks():
  from deepglobalregistration_b200 import _abi
  P, I_P, Q, I_Q, nrm, grad, T_init, _, vs = colored_case()
  for lam, md in ((1.5, vs), (-0.1, vs), (0.9, 4.5 * vs)):
    with pytest.raises(_abi.DgrError):
      run_colored(P, I_P, Q, nrm, I_Q, grad, vs, md, T_init, lam=lam)
  spec, table = cloud_hash(Q, vs)
  res = torch.empty(20, dtype=torch.float64, device='cuda')
  ws = torch.empty(1 << 16, dtype=torch.float64, device='cuda')
  T12 = _t(np.eye(4)[:3], torch.float64)
  Qd = _t(Q, torch.float32)
  with pytest.raises(_abi.DgrError, match='null pointer'):
    _abi.call('dgr_colored_icp', _abi.ptr(_t(P, torch.float32)), 0, len(P), _abi.ptr(Qd), _abi.ptr(Qd), _abi.ptr(Qd),
              _abi.ptr(Qd), _abi.ptr(spec), _abi.ptr(table.keys), _abi.ptr(table.vals), table.cap, 0, vs, vs, 0.9,
              _abi.ptr(T12), 30, 1e-6, 1e-6, _abi.ptr(ws), _abi.ptr(res), _abi.stream())
  with pytest.raises(_abi.DgrError):
    gpu_gradient(Q, nrm, I_Q, vs, 4.5 * vs, 30)
  with pytest.raises(_abi.DgrError):
    gpu_gradient(Q, nrm, I_Q, vs, 2 * vs, 65)


def test_stand_in_both_forms():
  from deepglobalregistration_b200 import _abi, shims
  from deepglobalregistration_b200 import o3d_registration as reg
  o3d = shims._open3d_stub()
  vs = 0.05
  P, I_P, Q, I_Q, _, _, T_init, T_gt, _ = colored_case(2)
  src, tgt = o3d.geometry.PointCloud(), o3d.geometry.PointCloud()
  src.points, tgt.points = o3d.utility.Vector3dVector(P), o3d.utility.Vector3dVector(Q)
  src.colors = np.repeat(I_P.astype(np.float64)[:, None], 3, axis=1)
  tgt.colors = np.repeat(I_Q.astype(np.float64)[:, None], 3, axis=1)
  tgt.estimate_normals(o3d.geometry.KDTreeSearchParamHybrid(radius=2 * vs, max_nn=30))
  crit = o3d.registration.ICPConvergenceCriteria(relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30)
  r010 = o3d.registration.registration_colored_icp(src, tgt, vs, T_init, crit, 0.968)
  r012 = o3d.pipelines.registration.registration_colored_icp(
      src, tgt, vs, T_init, o3d.pipelines.registration.TransformationEstimationForColoredICP(), crit)
  # the same thing through _abi directly, bit for bit
  cell, spec, table = reg._target_hash(_t(Q, torch.float64), 2 * vs)
  assert cell == vs
  nrm = _t(tgt.normals.astype(np.float32), torch.float32)
  i_t = _t(reg.intensity(tgt.colors), torch.float32)
  grad = _abi.color_gradient(_t(Q, torch.float32), nrm, i_t, (spec, table), cell, 2 * vs, 30)
  want = _abi.icp_colored(_t(P, torch.float32), _t(reg.intensity(src.colors), torch.float32), _t(Q, torch.float32),
                          nrm, i_t, grad, (spec, table), cell, vs, 0.968, T_init).cpu().numpy()
  for r in (r010, r012):
    assert np.array_equal(r.transformation, want[:16].reshape(4, 4))
    assert (r.fitness, r.inlier_rmse, len(r.correspondence_set)) == (want[16], want[17], int(want[19]))
  te, re = syn.rte_rre(r010.transformation, T_gt)
  assert te < 0.02 and re < 0.02, (te, re)
  # a cloud no admissible cell hashes: the voxel-downsample hint
  dense = o3d.geometry.PointCloud()
  dense.points = o3d.utility.Vector3dVector(np.concatenate([Q, Q + 1e-4]))
  dense.colors = np.full((2 * len(Q), 3), 0.5)
  dense.normals = np.tile([0.0, 0.0, 1.0], (2 * len(Q), 1))
  with pytest.raises(NotImplementedError, match='voxel-downsample'):
    reg.registration_colored_icp(src, dense, vs, T_init)


class _StubMethod:
  """A pairwise method that returns the ground truth perturbed by a seeded few degrees and centimetres, drawn in call
  order (so two runs over the same pairs get the same poses).  Fragments are told apart by their first point."""

  def __init__(self, clouds, gt, vs, seed=0):
    self.voxel_size = vs
    self.rng = np.random.default_rng(seed)
    self.index = {np.asarray(c, np.float64)[0].tobytes(): k for k, c in enumerate(clouds)}
    self.gt = gt

  def register(self, a, b):
    i, j = (self.index[np.asarray(c, np.float64)[0].tobytes()] for c in (a, b))
    return syn.random_se3(self.rng, 2.0, 0.02) @ np.linalg.inv(self.gt[j]) @ self.gt[i]


def _pose_error(T, T_ref):
  return np.linalg.norm(T[:3, 3] - T_ref[:3, 3]) + rotation_angle(T[:3, :3], T_ref[:3, :3])


def test_multiway_refinement():
  from deepglobalregistration_b200.core.multiway import MultiwayRegistration, absolute_trajectory_error
  clouds, cols, gt = syn.room_fragments(0, n_frag=6, colours=True)
  pcds = []
  for c, col in zip(clouds, cols):
    p = dio.PointCloud(c)
    p.colors = col
    pcds.append(p)
  vs = 0.05
  poses0, rep0 = MultiwayRegistration(_StubMethod(clouds, gt, vs)).register_sequence(clouds)
  poses, rep = MultiwayRegistration(_StubMethod(clouds, gt, vs), refine='colored_icp').register_sequence(pcds)
  assert np.array_equal(rep['pairwise_poses'], rep0['pairwise_poses'])
  kept = [e for e in rep['edges'] if e['kept']]
  assert rep['kept'] == rep0['kept'] and len(kept) >= 6 and 'refine' in rep['seconds']
  for e in kept:
    T_ref = np.linalg.inv(gt[e['t']]) @ gt[e['s']]
    before, after = _pose_error(e['T_pairwise'], T_ref), _pose_error(e['T'], T_ref)
    print(f'edge ({e["s"]}, {e["t"]}): error {before:.4f} -> {after:.4f}, fitness {e["refine_fitness"]:.3f}')
    assert after < before, (e['s'], e['t'], before, after, e['refine_fitness'])
  ate0, ate = absolute_trajectory_error(poses0, gt), absolute_trajectory_error(poses, gt)
  print(f'ATE {ate:.4f} m refined, {ate0:.4f} m without; refinement {rep["seconds"]["refine"]:.3f} s for '
        f'{len(kept)} edges')
  assert ate < ate0
  # refine=None: today's output, bit for bit (the same stub draws)
  again, rep_again = MultiwayRegistration(_StubMethod(clouds, gt, vs)).register_sequence(clouds)
  assert np.array_equal(again, poses0)
  assert all(np.array_equal(a['T'], b['T']) and np.array_equal(a['info'], b['info'])
             for a, b in zip(rep_again['edges'], rep0['edges']))


def test_cli_refine(tmp_path, capsys):
  from deepglobalregistration_b200 import multiway as cli
  clouds, cols, gt = syn.room_fragments(1, n_frag=4, n_raw=60000, colours=True)
  lst = tmp_path / 'frags.txt'
  for k, (c, col) in enumerate(zip(clouds, cols)):
    c8 = np.round(col * 255).astype(np.uint8)
    dio.write_ply(tmp_path / f'f{k}.ply', c, dtype='double', red=c8[:, 0], green=c8[:, 1], blue=c8[:, 2])
  lst.write_text(''.join(f'f{k}.ply\n' for k in range(4)))
  dio.write_trajectory(str(tmp_path / 'traj.log'), [([k, k, 4], P) for k, P in enumerate(gt)])
  torch.save(syn.make_checkpoint(0, voxel_size=0.05), tmp_path / 'ckpt.pth')
  cli.main(['--fragment_list', str(lst), '--gt_trajectory', str(tmp_path / 'traj.log'), '--weights',
            str(tmp_path / 'ckpt.pth'), '--method', 'fpfh_fgr', '--refine', 'colored_icp', '--out_dir',
            str(tmp_path / 'out')])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  print(summary)
  assert summary['refine'] == 'colored_icp' and 'refine' in summary['seconds']
  back = dio.read_trajectory(summary['trajectory'])
  assert [cp.metadata for cp in back] == [[k, k, 4] for k in range(4)]
  assert summary['ate'] >= 0.0
