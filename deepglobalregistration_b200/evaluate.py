"""Pair-list evaluation - the caller side of register() (SURVEY.md §8f rank 4): what the
reference's scripts/test_3dmatch.py:93-162 and scripts/test_kitti.py:57-112 do, sharded over the
GPUs of one box (sharding.py; pairs are independent, one all-gather of the results at the end).

    torchrun --nproc-per-node 8 -m deepglobalregistration_b200.evaluate \\
        --threed_match_dir /data/threedmatch_test --weights ckpt.pth --out_dir out
    python -m deepglobalregistration_b200.evaluate --pair_list pairs.txt --weights ckpt.pth

Pair sources:
* a 3DMatch test tree: ``<root>/<scene>/cloud_bin_<i>.ply`` and ``<root>/<scene>-evaluation/gt.log``
  (dataloader/threedmatch_loader.py:167-196); gt.log holds the pose of fragment j in fragment i's
  frame, so the pose register(cloud_i, cloud_j) must return is its inverse (scripts/test_3dmatch.py:107);
* a KITTI odometry tree: ``<root>/dataset/sequences/<dd>/velodyne/<tttttt>.bin`` and
  ``<root>/dataset/poses/<dd>.txt``; pairs = frames at least 10 m apart chosen the way
  dataloader/kitti_loader.py:229-279 chooses them, ground truth from the odometry poses and the
  velodyne-to-camera calibration (:66-78, :147-148).  The reference additionally polishes that pose
  with a 200-iteration ICP and caches it (:139-160); that refinement is NOT applied here, so RTE / RRE
  carry the odometry's own error (a few cm) - fine for the 0.6 m / 5 deg success criterion;
* a pair list: one pair per line, ``file0 file1 [16 numbers = row-major 4x4 mapping file0 into file1's
  frame] [group]``, any format io.read_points understands (KITTI .bin, .npz, .ply ...).

Output: ``stats`` [n_pairs, 5] = (success, RTE m, RRE deg, seconds, group id) - the row layout of the
reference's ``*-stats_*.npz`` - plus the poses."""
import argparse
import math
import os

import numpy as np

from . import io as dio
from . import sharding


def rte_rre(T_pred, T_gt, rte_thresh, rre_thresh, eps=1e-16):
  """(success, RTE [m], RRE [deg]) with the reference's evaluation criterion
  (scripts/test_3dmatch.py:38-46): identical arithmetic, so success counts are comparable."""
  if T_pred is None:
    return np.array([0, np.inf, np.inf])
  rte = float(np.linalg.norm(T_pred[:3, 3] - T_gt[:3, 3]))
  c = (np.trace(T_pred[:3, :3].T @ T_gt[:3, :3]) - 1) / 2
  rre = math.degrees(math.acos(min(max(c, -1 + eps), 1 - eps)))
  return np.array([float(rte < rte_thresh and rre < rre_thresh), rte, rre])


class Pair:
  __slots__ = ('file0', 'file1', 'T_gt', 'group')

  def __init__(self, file0, file1, T_gt=None, group=''):
    self.file0, self.file1, self.T_gt, self.group = file0, file1, T_gt, group


def threedmatch_pairs(root, scenes=None, ext='.ply'):
  """Every (i, j) of every scene's gt.log."""
  if scenes is None:
    scenes = sorted(d[:-len('-evaluation')] for d in os.listdir(root) if d.endswith('-evaluation'))
  pairs = []
  for scene in scenes:
    log = os.path.join(root, scene + '-evaluation', 'gt.log')
    if not os.path.exists(log):
      raise FileNotFoundError(log)
    for cp in dio.read_trajectory(log):
      i, j = cp.metadata[0], cp.metadata[1]
      pairs.append(Pair(os.path.join(root, scene, f'cloud_bin_{i}{ext}'),
                        os.path.join(root, scene, f'cloud_bin_{j}{ext}'), np.linalg.inv(cp.pose), scene))
  return pairs


# velodyne -> camera-0 calibration the reference hard-codes (dataloader/kitti_loader.py:66-78)
KITTI_VELO2CAM = np.array([
    [7.533745e-03, -9.999714e-01, -6.166020e-04, -4.069766e-03],
    [1.480249e-02, 7.280733e-04, -9.998902e-01, -7.631618e-02],
    [9.998621e-01, 7.523790e-03, 1.480755e-02, -2.717806e-01],
    [0.0, 0.0, 0.0, 1.0]])
KITTI_TEST_DRIVES = (8, 9, 10)                  # dataloader/split/test_kitti.txt
KITTI_SKIPPED = {(8, 15, 58)}                   # "problematic sequence", dataloader/kitti_loader.py:275-279


def kitti_poses(root, drive):
  """[n_frames, 4, 4] camera-0 poses of a drive (poses/<dd>.txt: 12 numbers per line)."""
  odo = np.loadtxt(os.path.join(root, 'dataset', 'poses', f'{drive:02d}.txt'), ndmin=2)
  P = np.tile(np.eye(4), (len(odo), 1, 1))
  P[:, :3, :] = odo.reshape(-1, 3, 4)
  return P


def kitti_gt_pose(P0, P1):
  """Pose mapping the velodyne frame of scan 0 into that of scan 1: V^-1 P1^-1 P0 V - what the
  reference computes (in transposed form) at dataloader/kitti_loader.py:147-148."""
  V = KITTI_VELO2CAM
  return np.linalg.inv(V) @ np.linalg.inv(P1) @ P0 @ V


def kitti_pairs(root, drives=KITTI_TEST_DRIVES, min_dist=10.0):
  """The test pairs of KITTINMPairDataset (dataloader/kitti_loader.py:229-279): walk each drive,
  pair the current frame with the frame just before the first one (within 100 frames) that is
  more than `min_dist` metres away, continue after the partner."""
  pairs = []
  for drive in drives:
    vel = os.path.join(root, 'dataset', 'sequences', f'{drive:02d}', 'velodyne')
    frames = sorted(int(f[:-4]) for f in os.listdir(vel) if f.endswith('.bin'))
    if not frames:
      raise FileNotFoundError(f'no scans under {vel}')
    have = set(frames)
    P = kitti_poses(root, drive)
    pos = P[:, :3, 3]
    cur = frames[0]
    while cur in have:
      far = np.flatnonzero(np.linalg.norm(pos[cur:cur + 100] - pos[cur], axis=1) > min_dist)
      if len(far) == 0:
        cur += 1
        continue
      nxt = int(far[0]) + cur - 1
      if nxt not in have:
        cur += 1                                   # (the reference would spin here; frames are contiguous in KITTI)
        continue
      if (drive, cur, nxt) not in KITTI_SKIPPED:
        pairs.append(Pair(os.path.join(vel, f'{cur:06d}.bin'), os.path.join(vel, f'{nxt:06d}.bin'),
                          kitti_gt_pose(P[cur], P[nxt]), f'drive{drive:02d}'))
      cur = nxt + 1
  return pairs


def read_pair_list(path):
  base = os.path.dirname(os.path.abspath(path))
  pairs = []
  with open(path) as fh:
    for ln, line in enumerate(fh, 1):
      tok = line.split('#')[0].split()
      if not tok:
        continue
      if len(tok) not in (2, 3, 18, 19):
        raise ValueError(f'{path}:{ln}: expected "file0 file1 [16 numbers] [group]"')
      T = np.array(tok[2:18], dtype=np.float64).reshape(4, 4) if len(tok) >= 18 else None
      group = tok[-1] if len(tok) in (3, 19) else ''
      f0, f1 = (t if os.path.isabs(t) else os.path.join(base, t) for t in tok[:2])
      pairs.append(Pair(f0, f1, T, group))
  return pairs


def evaluate(method, pairs, rte_thresh=0.3, rre_thresh=15.0, log=None, device=None):
  """Register every pair (this rank's share; results gathered on all ranks).  `device`: where the
  gather buffer lives - a CUDA device under an NCCL process group (NCCL has no CPU backend), None for
  gloo / a single process.
  -> dict(stats [n, 5], poses [n, 4, 4], branch [n], groups [names])."""
  groups = sorted({p.group for p in pairs})
  rows = sharding.register_pairs(method, [(p.file0, p.file1) for p in pairs], device=device).numpy().astype(np.float64)
  n = len(pairs)
  stats = np.zeros((n, 5))
  poses = rows[:, :16].reshape(n, 4, 4)
  for k, p in enumerate(pairs):
    if p.T_gt is not None:
      stats[k, :3] = rte_rre(poses[k], p.T_gt, rte_thresh, rre_thresh)
    else:
      stats[k, :3] = (np.nan, np.nan, np.nan)
    stats[k, 3] = rows[k, 19] / 1e3
    stats[k, 4] = groups.index(p.group)
    if log is not None and p.T_gt is not None and stats[k, 0] == 0:
      log(f'pair {k} ({os.path.basename(p.file0)}, {os.path.basename(p.file1)}) failed: '
          f'RTE {stats[k, 1]:.3f} m, RRE {stats[k, 2]:.2f} deg')
  return dict(stats=stats, poses=poses, branch=rows[:, 18], groups=groups)


def summarize(result):
  """The numbers the reference prints (scripts/test_3dmatch.py:49-63,148-160): overall means, means
  over the successful pairs, per-group recall and the average of the per-group recalls."""
  stats = result['stats']
  have = ~np.isnan(stats[:, 0])
  s = stats[have]
  out = dict(pairs=int(len(stats)), with_ground_truth=int(have.sum()), seconds_per_pair=float(stats[:, 3].mean()) if len(stats) else 0.0)
  if len(s):
    ok = s[:, 0] > 0
    out.update(recall=float(ok.mean()), rte_all=float(s[:, 1].mean()), rre_all=float(s[:, 2].mean()),
               rte_success=float(s[ok, 1].mean()) if ok.any() else float('nan'),
               rre_success=float(s[ok, 2].mean()) if ok.any() else float('nan'))
    per = {}
    for g, name in enumerate(result['groups']):
      m = s[:, 4] == g
      if m.any():
        per[name] = float(s[m, 0].mean())
    out.update(recall_per_group=per, recall_group_average=float(np.mean(list(per.values()))))
  return out


def main(argv=None):
  import json

  import torch
  import torch.distributed as dist
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  src = ap.add_mutually_exclusive_group(required=True)
  src.add_argument('--threed_match_dir', help='3DMatch test tree (scene folders + <scene>-evaluation/gt.log)')
  src.add_argument('--kitti_dir', help='KITTI odometry root (contains dataset/sequences, dataset/poses); '
                   'use --success_rte_thresh 0.6 --success_rre_thresh 5 (scripts/test_kitti.py:33-34)')
  src.add_argument('--pair_list', help='text file: file0 file1 [16 numbers] [group] per line')
  ap.add_argument('--weights', required=True)
  ap.add_argument('--clip_weight_thresh', type=float, default=0.05)
  ap.add_argument('--success_rte_thresh', type=float, default=0.3, help='m (config.py:127; KITTI: 0.6)')
  ap.add_argument('--success_rre_thresh', type=float, default=15.0, help='deg (config.py:128; KITTI: 5)')
  ap.add_argument('--no_icp', action='store_true')
  ap.add_argument('--method', choices=('dgr', 'fcgf_ransac', 'fcgf_fgr', 'icp_point_to_point', 'icp_point_to_plane',
                                       'goicp', 'super4pcs', 'pointnetlk'),
                  default='dgr',
                  help='dgr: DeepGlobalRegistration.register; fcgf_ransac: the FCGF + RANSAC baseline on the same '
                  'checkpoint (core/fcgf_ransac.py); fcgf_fgr: FCGF + Fast Global Registration with open3d\'s '
                  'default options (core/fcgf_fgr.py); icp_point_to_point / icp_point_to_plane: ICP from the identity '
                  'on the checkpoint\'s voxelisation (core/icp_baseline.py); goicp: globally optimal Go-ICP on the same '
                  'voxelisation (core/goicp.py); super4pcs: 4-point congruent sets on the same voxelisation '
                  '(core/super4pcs.py); pointnetlk: PointNetLK on the same voxelisation with the network of '
                  '--pointnetlk_weights (core/pointnetlk.py)')
  ap.add_argument('--ransac_max_iteration', type=int, default=80000, help='fcgf_ransac: hypotheses drawn at most')
  ap.add_argument('--ransac_max_validation', type=int, default=1000,
                  help='fcgf_ransac: hypotheses scored (the ones that pass the checkers first)')
  ap.add_argument('--ransac_edge_ratio', type=float, default=0.0,
                  help='fcgf_ransac: edge-length checker similarity threshold (open3d uses 0.9); 0 = off')
  ap.add_argument('--icp_max_correspondence_distance', type=float, default=None,
                  help='icp_*: correspondence radius in metres (default 2 voxels, at most 4)')
  ap.add_argument('--icp_max_iteration', type=int, default=30, help='icp_*: ICP updates at most')
  ap.add_argument('--goicp_mse_thresh', type=float, default=1e-3,
                  help='goicp: stop when E* - LB < mse_thresh K (normalised units)')
  ap.add_argument('--goicp_trim_fraction', type=float, default=0.0, help='goicp: share of source points left out')
  ap.add_argument('--goicp_n_data', type=int, default=1000, help='goicp: source points searched (at most 1024)')
  ap.add_argument('--super4pcs_overlap', type=float, default=0.5,
                  help='super4pcs: expected overlap; bases span at most overlap x the source diameter')
  ap.add_argument('--super4pcs_delta', type=float, default=None,
                  help='super4pcs: congruence and LCP tolerance in metres (default 2 voxels)')
  ap.add_argument('--super4pcs_sample_size', type=int, default=512,
                  help='super4pcs: source points (at most 1024); the target sample is twice as many (at most 4096)')
  ap.add_argument('--super4pcs_max_bases', type=int, default=256, help='super4pcs: bases tried at most')
  ap.add_argument('--pointnetlk_weights', default=None,
                  help='pointnetlk: PointNet_features state dict (required: a random network is no baseline)')
  ap.add_argument('--pointnetlk_max_iter', type=int, default=10, help='pointnetlk: Lucas-Kanade steps at most')
  ap.add_argument('--out_dir', default='.')
  args = ap.parse_args(argv)
  if args.method == 'pointnetlk' and not args.pointnetlk_weights:
    ap.error('--method pointnetlk needs --pointnetlk_weights')

  world = int(os.environ.get('WORLD_SIZE', '1'))
  local = int(os.environ.get('LOCAL_RANK', '0'))
  torch.cuda.set_device(local)
  if world > 1:
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
  rank = dist.get_rank() if world > 1 else 0
  from .core.deep_global_registration import DeepGlobalRegistration
  cfg = argparse.Namespace(weights=args.weights, clip_weight_thresh=args.clip_weight_thresh, verbose=False)
  dgr = DeepGlobalRegistration(cfg, device=torch.device('cuda', local))
  dgr.use_icp = not args.no_icp
  method = dgr
  if args.method == 'fcgf_ransac':
    from .core.fcgf_ransac import FCGFRansac
    method = FCGFRansac(dgr)
    method.max_iteration, method.max_validation = args.ransac_max_iteration, args.ransac_max_validation
    method.edge_ratio = args.ransac_edge_ratio
  elif args.method == 'fcgf_fgr':
    from .core.fcgf_fgr import FCGFFastGlobal
    method = FCGFFastGlobal(dgr)
  elif args.method in ('icp_point_to_point', 'icp_point_to_plane'):
    from .core.icp_baseline import ICPBaseline
    method = ICPBaseline(dgr, args.method[len('icp_'):], args.icp_max_correspondence_distance, args.icp_max_iteration)
  elif args.method == 'goicp':
    from .core.goicp import GoICPBaseline
    method = GoICPBaseline(dgr, args.goicp_mse_thresh, args.goicp_trim_fraction, args.goicp_n_data)
  elif args.method == 'super4pcs':
    from .core.super4pcs import Super4PCSBaseline
    method = Super4PCSBaseline(dgr, overlap=args.super4pcs_overlap, delta=args.super4pcs_delta,
                               sample_size=args.super4pcs_sample_size, max_bases=args.super4pcs_max_bases)
  elif args.method == 'pointnetlk':
    from .core.pointnetlk import PointNetLKBaseline
    method = PointNetLKBaseline(dgr, args.pointnetlk_weights, max_iter=args.pointnetlk_max_iter)
  if args.threed_match_dir:
    pairs = threedmatch_pairs(args.threed_match_dir)
  elif args.kitti_dir:
    pairs = kitti_pairs(args.kitti_dir)
  else:
    pairs = read_pair_list(args.pair_list)
  # the output directory is settled BEFORE hours of registration: created if missing; when that is
  # impossible fall back to the current directory as the reference does (scripts/test_3dmatch.py:135-137)
  out_dir = args.out_dir
  if rank == 0:
    try:
      os.makedirs(out_dir, exist_ok=True)
    except OSError as e:
      print(f'cannot create {out_dir!r} ({e}); saving to the current directory')
      out_dir = '.'
  result = evaluate(method, pairs, args.success_rte_thresh, args.success_rre_thresh,
                    log=print if rank == 0 else None, device=torch.device('cuda', local))
  if rank == 0:
    summary = summarize(result)
    print(json.dumps(dict(summary, world_size=world)))          # the summary first: a failing save loses nothing
    stem, name = {'dgr': ('dgr-b200', 'DGR'), 'fcgf_ransac': ('fcgf-ransac-b200', 'RANSAC'),
                  'fcgf_fgr': ('fcgf-fgr-b200', 'FGR'), 'icp_point_to_point': ('icp-p2p-b200', 'ICP (Point-to-point)'),
                  'icp_point_to_plane': ('icp-p2plane-b200', 'ICP (Point-to-plane)'),
                  'goicp': ('goicp-b200', 'Go-ICP'), 'super4pcs': ('super4pcs-b200', 'Super4PCS'),
                  'pointnetlk': ('pointnetlk-b200', 'PointNetLK')}[args.method]
    out = os.path.join(out_dir, f'{stem}-stats.npz')
    np.savez(out, stats=result['stats'][None], names=[name], poses=result['poses'], groups=result['groups'])
    print(json.dumps(dict(summary, world_size=world, saved=out)))
  if world > 1:
    dist.destroy_process_group()


if __name__ == '__main__':
  main()
