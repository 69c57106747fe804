"""Time generalized ICP and the robust losses on the GPU, at two sizes: room_pair(0) voxelised at 0.05 m and a
KITTI-shape lidar_pair(0) voxelised at 0.3 m (sensors 3 m apart), each second cloud started 3 degrees / 3 cm (room)
or 2 degrees / 0.3 m (LiDAR) off the truth.  Per size, with CUDA events (medians over --reps): the covariance pass
(dgr_estimate_covariances, radius 2 voxels, max_nn 30) on the target, the from-normals pass
(dgr_covariances_from_normals, epsilon 1e-3), one dgr_generalized_icp call on covariances from both clouds' normals
(30 iterations at most, max_dist 2 voxels), and point-to-plane ICP with and without TukeyLoss(k = 1 voxel).  The
card's name and power limit are read in the same run.  One JSON line.

    python tools/gicp_bench.py [--reps 10]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from tools.fpfh_bench import card, median_ms  # noqa: E402


def cases():
  """(name, xyz0, xyz1, T_init, voxel) of the two sizes."""
  x0, x1, T = syn.room_pair(0)
  yield 'room_0.05', x0, x1, syn.random_se3(np.random.default_rng(0), 3.0, 0.03) @ T, 0.05
  x0, x1, T = syn.lidar_pair(0, advance=3.0)
  yield 'lidar_0.3', x0, x1, syn.random_se3(np.random.default_rng(0), 2.0, 0.3) @ T, 0.3


def run(reps):
  dev = torch.device('cuda')
  _abi.refresh_stream()
  out = dict(card=card(), reps=reps, sizes={})
  for name, x0, x1, T0, vs in cases():
    clouds = []
    for x in (x0, x1):
      x32 = np.asarray(x, np.float32).astype(np.float64)
      _, first = np.unique(np.floor(x32 / vs).astype(np.int64), axis=0, return_index=True)
      p = x32[np.sort(first)]
      raw, spec, table, _, _, n = _abi.voxelise(torch.from_numpy(np.ascontiguousarray(p)).to(dev), vs)
      assert n == len(p)
      clouds.append((torch.from_numpy(p).to(dev, torch.float32).contiguous(), (spec, table)))
    (P, hP), (Q, hQ) = clouds
    nP = _abi.estimate_normals(P, hP, vs, 2 * vs, 30)
    nQ = _abi.estimate_normals(Q, hQ, vs, 2 * vs, 30)
    cP, cQ = _abi.covariances_from_normals(nP), _abi.covariances_from_normals(nQ)
    T12 = torch.from_numpy(np.ascontiguousarray(T0[:3])).to(dev)
    res = {}
    r = dict(n_src=len(P), n_tgt=len(Q))
    r['covariances_ms'] = median_ms(lambda: _abi.estimate_covariances(Q, hQ, vs, 2 * vs, 30), reps)
    r['from_normals_ms'] = median_ms(lambda: _abi.covariances_from_normals(nQ), reps)

    def gicp():
      res['gicp'] = _abi.icp_generalized(P, cP, Q, cQ, hQ, vs, 2 * vs, T12)

    def plane():
      res['plane'] = _abi.icp_point_to_plane(P, Q, nQ, hQ, vs, 2 * vs, T12)

    def tukey():
      res['tukey'] = _abi.icp_point_to_plane(P, Q, nQ, hQ, vs, 2 * vs, T12, loss='Tukey', loss_k=vs)

    r['gicp_ms'] = median_ms(gicp, reps)
    r['plane_ms'] = median_ms(plane, reps)
    r['plane_tukey_ms'] = median_ms(tukey, reps)
    for k, v in res.items():
      h = v.cpu().numpy()
      r[f'{k}_iterations'] = int(h[18])
      r[f'{k}_fitness'] = float(h[16])
    out['sizes'][name] = r
  return out


def main(argv=None):
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--reps', type=int, default=10)
  args = ap.parse_args(argv)
  print(json.dumps(run(args.reps)))


if __name__ == '__main__':
  main()
