"""Time colored ICP (open3d's registration_colored_icp) on the GPU: dgr_color_gradient of the target and one
dgr_colored_icp call (30 iterations at most, max_distance = the voxel, gradient radius 2 voxels, max_nn 30) on a
room_pair(0)-sized coloured pair (250k raw points per cloud, the second cloud resampled and moved 3 degrees / 3 cm) at
voxels 0.05, 0.025 and 0.0125 m, with CUDA events (medians); the fp64 oracle on the same inputs at the scales in
--oracle_voxels; and multiway registration of a 6-fragment coloured room through FPFH + FGR with refine='colored_icp'
(the pairwise stage and the refinement stage, host clocks around synchronised work).  The card's name and power limit
are read in the same run.  One JSON line.

Bytes model of the gradient pass (per point; the probe reads each of the (2 reach + 1)^3 hash slots' 8-byte key and
4-byte value, every in-radius neighbour's 12-byte point and 4-byte intensity, the point's own point, normal and
intensity, and writes a 12-byte gradient and a 4-byte count):  125 * 12 + 16 * nbrs + 28 + 16 at reach 2.

    python tools/colored_icp_bench.py [--reps 5] [--oracle_voxels 0.05]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import io as dio  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from deepglobalregistration_b200.o3d_registration import intensity  # noqa: E402
from tools.fpfh_bench import card, median_ms  # noqa: E402

VOXELS = (0.05, 0.025, 0.0125)
HBM_BYTES_PER_S = 3.35e12                 # H100 SXM data sheet


def coloured_pair():
  """(xyz0, rgb0, xyz1, rgb1, T mapping 0 into 1): room_pair(0)'s scene and sizes, with _face_colour colours."""
  x0, c0 = syn.room_scan(0, scene_seed=0, colours=True)
  x1, c1 = syn.room_scan(1, scene_seed=0, colours=True)
  T = syn.random_se3(np.random.default_rng(7), 3.0, 0.03)
  return x0, c0 / 255.0, syn.apply_se3(T, x1), c1 / 255.0, T


def first_per_cell(x, cell):
  x32 = np.asarray(x, np.float32).astype(np.float64)
  _, first = np.unique(np.floor(x32 / cell).astype(np.int64), axis=0, return_index=True)
  return np.sort(first)


def scale_case(pair, vs):
  x0, c0, x1, c1, _ = pair
  i0, i1 = first_per_cell(x0, vs), first_per_cell(x1, vs)
  P, Q = x0[i0].astype(np.float32).astype(np.float64), x1[i1].astype(np.float32).astype(np.float64)
  return P, intensity(c0[i0]), Q, intensity(c1[i1])


def bench_scale(pair, vs, reps, oracle):
  P, I_P, Q, I_Q = scale_case(pair, vs)
  dev = torch.device('cuda')
  _, spec, table, _, _, n = _abi.voxelise(torch.from_numpy(Q).to(dev), vs)
  assert n == len(Q)
  hashed = (spec, table)
  src, tgt = torch.from_numpy(P).float().to(dev), torch.from_numpy(Q).float().to(dev)
  i_s, i_t = torch.from_numpy(I_P).to(dev), torch.from_numpy(I_Q).to(dev)
  nrm, counts = _abi.estimate_normals(tgt, hashed, vs, 2 * vs, 30, return_counts=True)
  grad = _abi.color_gradient(tgt, nrm, i_t, hashed, vs, 2 * vs, 30)
  T0 = torch.from_numpy(np.eye(4)[:3].copy()).to(dev)
  out = {}
  out['gradient_ms'] = median_ms(lambda: _abi.color_gradient(tgt, nrm, i_t, hashed, vs, 2 * vs, 30), reps)
  res = [None]

  def icp():
    res[0] = _abi.icp_colored(src, i_s, tgt, nrm, i_t, grad, hashed, vs, vs, 0.968, T0)
  out['icp_ms'] = median_ms(icp, reps)
  r = res[0].cpu().numpy()
  nb = np.minimum(counts.cpu().numpy(), 30).astype(np.float64)
  bytes_model = float(len(Q) * (125 * 12 + 28 + 16) + 16 * nb.sum())
  out.update(voxel=vs, n_src=len(P), n_tgt=len(Q), mean_neighbours=float(nb.mean()), icp_iterations=int(r[18]),
             fitness=float(r[16]), te_rre=[float(v) for v in syn.rte_rre(r[:16].reshape(4, 4), pair[4])],
             gradient_bytes_model=bytes_model,
             gradient_share_of_hbm=bytes_model / (out['gradient_ms'] * 1e-3) / HBM_BYTES_PER_S)
  if oracle:
    from oracle import colored_icp as oc
    n_np, g_np = nrm.cpu().numpy().astype(np.float64), grad.cpu().numpy().astype(np.float64)
    t = time.perf_counter()
    oc.color_gradient(Q, n_np, I_Q, 2 * vs, 30)
    out['oracle_gradient_s'] = time.perf_counter() - t
    t = time.perf_counter()
    oc.colored_icp(P, I_P, Q, n_np, I_Q, g_np, vs, np.eye(4))
    out['oracle_icp_s'] = time.perf_counter() - t
  return out


def bench_multiway():
  import types
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.fpfh_baseline import FPFHFastGlobal
  from deepglobalregistration_b200.core.multiway import MultiwayRegistration
  clouds, cols, _ = syn.room_fragments(0, n_frag=6, colours=True)
  pcds = []
  for c, col in zip(clouds, cols):
    p = dio.PointCloud(c)
    p.colors = col
    pcds.append(p)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=0.05),
                                                   clip_weight_thresh=0.05, verbose=False))
  d.use_icp = True
  mw = MultiwayRegistration(FPFHFastGlobal(d), refine='colored_icp')
  mw.register_sequence(pcds)                              # warm-up
  torch.cuda.synchronize()
  _, rep = mw.register_sequence(pcds)
  sec = rep['seconds']
  return dict(fragments=6, kept_edges=rep['kept'], pairwise_s=sec['pairwise'], refine_s=sec['refine'],
              information_s=sec['information'], optimise_s=sec['optimise'], total_s=sec['total'])


def main(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--reps', type=int, default=5)
  ap.add_argument('--oracle_voxels', type=float, nargs='*', default=[0.05])
  args = ap.parse_args(argv)
  _abi.require_device('cuda')
  _abi.refresh_stream()
  pair = coloured_pair()
  scales = [bench_scale(pair, vs, args.reps, vs in args.oracle_voxels) for vs in VOXELS]
  print(json.dumps(dict(card=card(), scales=scales, multiway=bench_multiway())))


if __name__ == '__main__':
  main()
