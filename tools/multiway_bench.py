"""Time the multiway-registration kernels on the GPU, and the CPU oracle on the same inputs:
  * dgr_information_matrix on the bench pair syn.room_pair(0) (voxel 0.05 m, radius 2 voxels), with its bytes model
    and its share of the H100's 3.35 TB/s;
  * dgr_pose_graph_optimize at N = 60 / E = 1770 (every pair, 20 % of the loop closures wrong) and at N = 256.
Prints the card's name and power limit, then one JSON line.

    python tools/multiway_bench.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from deepglobalregistration_b200.core.multiway import odometry_chain  # noqa: E402
from oracle import pose_graph as pg  # noqa: E402


def card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  return out or torch.cuda.get_device_name()


def gpu_ms(fn, reps):
  fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


def graph(seed, n, n_loops, n_wrong):
  g = syn.pose_graph(seed, n, n_loops, noise=0.005, n_wrong=n_wrong)
  g['start'] = odometry_chain(n, [dict(s=int(s), t=int(t), T=T) for (s, t), T in zip(g['ends'], g['T'])])
  return g


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  args = ap.parse_args()
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  out = dict(card=card())
  vs = 0.05
  xyz0, xyz1, T = syn.room_pair(0)
  x0 = torch.from_numpy(xyz0).to(dev)
  x1 = torch.from_numpy(xyz1).to(dev)
  _, _, _, sel0, _, n0 = _abi.voxelise(x0, vs)
  src = x0[sel0.long()].float().contiguous()
  _, spec, table, sel1, _, n1 = _abi.voxelise(x1, vs)
  tgt = x1[sel1.long()].float().contiguous()
  ms = gpu_ms(lambda: _abi.information_matrix(src, tgt, (spec, table), vs, 2 * vs, T), args.reps)
  lam = _abi.information_matrix(src, tgt, (spec, table), vs, 2 * vs, T).cpu().numpy()
  # bytes model: source points once, 125 probes of 8-byte keys + 4-byte values per point (reach 2), the matched
  # candidates' target rows (12 B each) - an upper bound on the distinct-line traffic is the table plus both clouds
  table_bytes = table.cap * 12
  model = n0 * 12 + table_bytes + n1 * 12
  t0 = time.perf_counter()
  pg.information_matrix(src.cpu().numpy(), tgt.cpu().numpy(), T, 2 * vs)
  cpu_info = time.perf_counter() - t0
  out['information'] = dict(n_src=n0, n_tgt=n1, correspondences=int(lam[36]), ms=round(ms, 4),
                            bytes_model=int(model), share_of_3_35TBs=round(model / (ms * 1e-3) / 3.35e12, 4),
                            oracle_s=round(cpu_info, 3))
  for name, (n, n_loops, n_wrong) in {'n60_e1770': (60, 1770 - 59, (1770 - 59) // 5),
                                      'n256': (256, 300, 30)}.items():
    g = graph(1, n, n_loops, n_wrong)
    conf = np.ones(len(g['ends']))
    run = lambda: _abi.pose_graph_optimize(g['start'], g['ends'], g['T'], g['info'], g['uncertain'], conf,
                                           reference_node=0)
    run()
    reps = max(1, args.reps // (10 if n > 100 else 1))
    t0 = time.perf_counter()
    for _ in range(reps):
      P, kept, lp, st = run()
    gpu_s = (time.perf_counter() - t0) / reps
    t0 = time.perf_counter()
    Po, ko, lo, so = pg.global_optimization(g['start'], g['ends'], g['T'], g['info'], g['uncertain'],
                                            option=dict(reference_node=0))
    cpu_s = time.perf_counter() - t0
    out[name] = dict(nodes=n, edges=len(g['ends']), wrong=int(g['wrong'].sum()), pruned=st['pruned'],
                     iterations=[st['iterations'], st['iterations_pruned']], factorisations=st['factorisations'],
                     ms=round(gpu_s * 1e3, 3), ms_per_factorisation_and_solve=round(gpu_s * 1e3 / st['factorisations'], 4),
                     oracle_s=round(cpu_s, 3), max_pose_diff_vs_oracle=float(np.abs(P - Po).max()),
                     same_pruned_set=bool(np.array_equal(kept, ko)))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
