"""Multiway registration end to end (core/multiway.py, python -m deepglobalregistration_b200.multiway): a known answer
through DGR with an injected wrong loop closure, partial-overlap fragments through FPFH + FGR, and the CLI."""
import json
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import synthetic as syn
from deepglobalregistration_b200.core.multiway import (MultiwayRegistration, absolute_trajectory_error, odometry_chain,
                                                       select_edges)

pytestmark = pytest.mark.gpu

EXTENT = (1.8, 1.5, 1.25)
ROOM_ATE_BOUND = 0.02     # measured 0.0137 m (odometry chain 0.0167 m) on an H100


def _calibrated_dgr(vs):
  """The BatchNorm-calibrated random-init DGR of test_gpu_pipeline.py::test_safeguard_branch_known_answer, with the
  calibrated statistics written back into the checkpoint."""
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.util.calibrate import calibrate_batchnorm
  st = syn.make_checkpoint(4, voxel_size=vs)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))
  xyz0 = syn.room_scan(2, 20000, EXTENT, scene_seed=1)
  with torch.no_grad():
    _, c0, f0 = d.preprocess(xyz0)
    calibrate_batchnorm(d.fcgf_model, ME.SparseTensor(f0, coordinates=c0, device='cuda'))
  st['state_dict'] = {k: v.detach().cpu().clone() for k, v in d.fcgf_model.state_dict().items()}
  return d, xyz0


def test_known_answer_through_dgr_with_a_wrong_loop_closure():
  vs = 0.0625
  d, xyz0 = _calibrated_dgr(vs)
  shifts = [vs * np.array(m) for m in ([0, 0, 0], [8, 0, 0], [8, -16, 0], [0, -16, 24], [-8, 8, 16])]
  clouds = [xyz0 + s for s in shifts]
  gt = np.stack([np.eye(4)] * 5)
  for k, s in enumerate(shifts):
    gt[k, :3, 3] = shifts[0] - s                       # fragment k into fragment 0's frame
  mw = MultiwayRegistration(d)
  assert mw.voxel_size == vs and mw.info_radius == 2 * vs
  pairs, X = mw.pairwise(clouds)
  for (i, j), T in zip(pairs, X):                      # the batched pairwise path sees the calibrated network
    te, re = syn.rte_rre(T, np.linalg.inv(gt[j]) @ gt[i])
    assert te <= 1e-3 and re <= 1e-3, (i, j, te, re)
  edges, n_points = mw.edges(clouds, pairs, X)
  kept = select_edges(edges, n_points, mw.overlap_thresh)
  assert len(kept) == 10                               # full overlap: every loop closure is kept
  wrong = dict(kept[1])                                # (0, 2) with a grossly wrong pose
  W = np.eye(4)
  W[:3, :3] = syn.random_se3(np.random.default_rng(0), 60.0, 0.0)[:3, :3]
  W[:3, 3] = [1.5, 0.0, 0.0]
  wrong['T'] = W @ wrong['T']
  graph = kept + [wrong]
  poses, alive, lp, stats = mw.optimise(5, graph)
  print(f'line process {np.round(lp, 4).tolist()}, stats {stats}')
  assert not alive[-1] and alive[:-1].all() and lp[-1] < 0.25
  for k in range(5):
    te, re = syn.rte_rre(poses[k], gt[k])
    assert te <= 1e-3 and re <= 1e-3, (k, te, re)


def _fpfh_fgr(vs=0.05):
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.fpfh_baseline import FPFHFastGlobal
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=vs),
                                                   clip_weight_thresh=0.05, verbose=False))
  d.use_icp = True
  return FPFHFastGlobal(d)


def test_partial_overlap_room_through_fpfh_fgr():
  clouds, gt = syn.room_fragments(0, n_frag=6)
  mw = MultiwayRegistration(_fpfh_fgr())
  poses, report = mw.register_sequence(clouds)
  ate = absolute_trajectory_error(poses, gt)
  ate_chain = absolute_trajectory_error(odometry_chain(len(clouds), report['edges']), gt)
  print(f'ATE {ate:.4f} m (odometry chain {ate_chain:.4f} m); kept {report["kept"]}, pruned {report["pruned"]}, '
        f'loop candidates {report["loop_candidates"]}, seconds {report["seconds"]}, optimiser {report["optimiser"]}')
  assert report['odometry'] == 5 and report['loop_candidates'] == 10
  assert ate < ROOM_ATE_BOUND and ate <= ate_chain + 1e-9


def test_cli_writes_a_trajectory_and_a_summary(tmp_path, capsys):
  from deepglobalregistration_b200 import multiway as cli
  clouds, gt = syn.room_fragments(1, n_frag=4)
  frag = tmp_path / 'scene'
  frag.mkdir()
  for k, c in enumerate(clouds):
    dio.write_ply(frag / f'cloud_bin_{k}.ply', c, dtype='double')
  (tmp_path / 'scene-evaluation').mkdir()
  dio.write_trajectory(str(tmp_path / 'scene-evaluation' / 'gt.log'),
                       [([i, j, 4], np.linalg.inv(gt[i]) @ gt[j])     # fragment j in fragment i's frame
                        for i in range(4) for j in range(i + 1, 4)])
  torch.save(syn.make_checkpoint(0, voxel_size=0.05), tmp_path / 'ckpt.pth')
  cli.main(['--fragments_dir', str(frag), '--weights', str(tmp_path / 'ckpt.pth'), '--method', 'fpfh_fgr',
            '--out_dir', str(tmp_path / 'out')])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  print(summary)
  assert summary['fragments'] == 4 and summary['pairs'] == 6 and summary['gt_pairs'] == 6
  assert 'recall_synchronised' in summary and 'recall_pairwise' in summary
  back = dio.read_trajectory(summary['trajectory'])
  assert [cp.metadata for cp in back] == [[k, k, 4] for k in range(4)]
  assert np.allclose(back[0].pose, np.eye(4))
  lst = tmp_path / 'frags.txt'
  lst.write_text(''.join(f'scene/cloud_bin_{k}.ply\n' for k in range(4)))
  dio.write_trajectory(str(tmp_path / 'traj.log'), [([k, k, 4], P) for k, P in enumerate(gt)])
  cli.main(['--fragment_list', str(lst), '--gt_trajectory', str(tmp_path / 'traj.log'), '--weights',
            str(tmp_path / 'ckpt.pth'), '--method', 'fpfh_fgr', '--out_dir', str(tmp_path / 'out2')])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  assert summary['ate'] >= 0.0 and summary['ate_odometry'] >= 0.0
