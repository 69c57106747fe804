"""Multiway registration of a fragment sequence (core/multiway.py) from the command line, with any pairwise method of
evaluate.py (the same flags).

    python -m deepglobalregistration_b200.multiway --fragments_dir /data/3dmatch/7-scenes-redkitchen \\
        --method dgr --weights ckpt.pth --out_dir out
    torchrun --nproc-per-node 8 -m deepglobalregistration_b200.multiway --fragment_list frags.txt \\
        --gt_trajectory gt.log --method fpfh_fgr --weights ckpt.pth

Fragments:
* ``--fragments_dir D``: ``D/cloud_bin_<i>.ply`` in index order (the 3DMatch layout).  When ``D-evaluation/gt.log``
  exists, the summary gives the pairwise recall of the synchronised poses (P_j^-1 P_i) on gt.log's pairs next to the
  recall of the raw pairwise poses on the same pairs (evaluate.rte_rre, --success_rte_thresh / --success_rre_thresh);
* ``--fragment_list F``: one fragment file per line (relative to F's directory), any format io.read_points reads;
  ``--gt_trajectory LOG`` (one pose per fragment, in order) adds the ATE: the RMS translation error after expressing
  both trajectories relative to fragment 0, next to the ATE of the odometry chain.

``--refine colored_icp`` refines every kept edge by multi-scale colored ICP before the optimisation (open3d's
refine_registration); the fragments then need colours (PLY red / green / blue).

Output: the trajectory (metadata ``k k N`` and fragment k's pose in fragment 0's frame) written with
io.write_trajectory, and one JSON summary line."""
import argparse
import json
import os
import re

import numpy as np

from . import evaluate as ev
from . import io as dio
from .core.multiway import MultiwayRegistration, absolute_trajectory_error, odometry_chain


def fragments_in_dir(root):
  files = [f for f in os.listdir(root) if re.fullmatch(r'cloud_bin_\d+\.ply', f)]
  if not files:
    raise FileNotFoundError(f'no cloud_bin_<i>.ply under {root}')
  return [os.path.join(root, f) for f in sorted(files, key=lambda f: int(f[len('cloud_bin_'):-4]))]


def read_fragment_list(path):
  base = os.path.dirname(os.path.abspath(path))
  out = []
  with open(path) as fh:
    for line in fh:
      tok = line.split('#')[0].strip()
      if tok:
        out.append(tok if os.path.isabs(tok) else os.path.join(base, tok))
  return out


def pair_recall(poses, pairwise, gt_pairs, rte_thresh, rre_thresh):
  """(recall of the synchronised poses, recall of the raw pairwise poses) on gt pairs [(i, j, T_gt mapping i into
  j)]; pairwise: {(i, j): X} for i < j."""
  sync, raw = [], []
  for i, j, T_gt in gt_pairs:
    sync.append(ev.rte_rre(np.linalg.inv(poses[j]) @ poses[i], T_gt, rte_thresh, rre_thresh)[0])
    X = pairwise[(i, j)] if i < j else np.linalg.inv(pairwise[(j, i)])
    raw.append(ev.rte_rre(X, T_gt, rte_thresh, rre_thresh)[0])
  return float(np.mean(sync)) if sync else float('nan'), float(np.mean(raw)) if raw else float('nan')


def main(argv=None):
  import torch
  import torch.distributed as dist
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  src = ap.add_mutually_exclusive_group(required=True)
  src.add_argument('--fragments_dir', help='cloud_bin_<i>.ply files (3DMatch layout)')
  src.add_argument('--fragment_list', help='text file: one fragment file per line')
  ap.add_argument('--gt_trajectory', default=None, help='with --fragment_list: ground-truth poses, one per fragment')
  ev.add_method_arguments(ap)
  ap.add_argument('--overlap_thresh', type=float, default=0.3,
                  help='loop closures kept when Lambda[5, 5] / min(n_i, n_j) reaches it')
  ap.add_argument('--info_radius_voxels', type=float, default=2.0, help='information-matrix radius in voxels')
  ap.add_argument('--refine', choices=['colored_icp'], default=None,
                  help='refine every kept edge by multi-scale colored ICP (needs coloured fragments)')
  ap.add_argument('--out_dir', default='.')
  args = ap.parse_args(argv)
  ev.check_method_arguments(ap, args)
  if args.gt_trajectory and not args.fragment_list:
    ap.error('--gt_trajectory goes with --fragment_list (--fragments_dir reads <dir>-evaluation/gt.log)')

  world = int(os.environ.get('WORLD_SIZE', '1'))
  local = int(os.environ.get('LOCAL_RANK', '0'))
  torch.cuda.set_device(local)
  if world > 1:
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
  rank = dist.get_rank() if world > 1 else 0
  device = torch.device('cuda', local)
  method = ev.build_method(args, device)
  if args.fragments_dir:
    files = fragments_in_dir(args.fragments_dir)
  else:
    files = read_fragment_list(args.fragment_list)
  mw = MultiwayRegistration(method, overlap_thresh=args.overlap_thresh, info_radius_voxels=args.info_radius_voxels,
                            refine=args.refine)
  poses, report = mw.register_sequence(files, device=device)
  if rank == 0:
    n = len(files)
    edges = report['edges']
    summary = dict(fragments=n, pairs=report['pairs'], odometry_edges=report['odometry'],
                   loop_candidates=report['loop_candidates'], kept_edges=report['kept'], pruned=report['pruned'],
                   seconds={k: round(v, 4) for k, v in report['seconds'].items()},
                   iterations=[report['optimiser'].get('iterations'), report['optimiser'].get('iterations_pruned')],
                   method=args.method, world_size=world)
    if args.refine:
      summary['refine'] = args.refine
    pairwise = {(e['s'], e['t']): e['T'] for e in edges}
    if args.fragments_dir:
      log = os.path.normpath(args.fragments_dir) + '-evaluation/gt.log'
      if os.path.exists(log):
        gt = [(cp.metadata[0], cp.metadata[1], np.linalg.inv(cp.pose)) for cp in dio.read_trajectory(log)
              if cp.metadata[0] < n and cp.metadata[1] < n]
        summary['recall_synchronised'], summary['recall_pairwise'] = pair_recall(
            poses, pairwise, gt, args.success_rte_thresh, args.success_rre_thresh)
        summary['gt_pairs'] = len(gt)
    if args.gt_trajectory:
      G = np.stack([cp.pose for cp in dio.read_trajectory(args.gt_trajectory)])
      if len(G) != n:
        raise ValueError(f'{args.gt_trajectory}: {len(G)} poses for {n} fragments')
      summary['ate'] = absolute_trajectory_error(poses, G)
      summary['ate_odometry'] = absolute_trajectory_error(odometry_chain(n, edges), G)
    os.makedirs(args.out_dir, exist_ok=True)
    out = os.path.join(args.out_dir, f'multiway-{args.method}-b200.log')
    dio.write_trajectory(out, [([k, k, n], P) for k, P in enumerate(poses)])
    summary['trajectory'] = out
    print(json.dumps(summary))
  if world > 1:
    dist.destroy_process_group()


if __name__ == '__main__':
  main()
