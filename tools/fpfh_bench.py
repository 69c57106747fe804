"""Time FPFH + RANSAC / FPFH + FGR on the bench's full-size pair syn.room_pair(0) (voxel 0.05 m, about 51k / 40k voxels):
the three FPFH passes (neighbours, SPFH, FPFH; per-kernel device times from torch.profiler, summed over both clouds),
the whole dgr_compute_fpfh call of both clouds, both kNN directions on the 64-column rows, and the RANSAC and FGR
searches with the baselines' settings (CUDA events, medians), with the card's name and power limit read in the same
run.  One JSON line.

    python tools/fpfh_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402

PASSES = (('neighbours', 'fpfh_neighbour_kernel'), ('spfh', 'fpfh_spfh_kernel'), ('fpfh', 'fpfh_kernel'))


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return out or f'{torch.cuda.get_device_name()}, power limit unknown'


def median_ms(fn, reps):
  fn()
  torch.cuda.synchronize()
  ms = []
  for _ in range(reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    fn()
    ev[1].record()
    torch.cuda.synchronize()
    ms.append(ev[0].elapsed_time(ev[1]))
  return float(np.median(ms))


def pass_ms(fn, reps):
  """Median per call of each FPFH kernel's summed device time (torch.profiler)."""
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  per = {name: [] for name, _ in PASSES}
  for _ in range(reps):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      fn()
      torch.cuda.synchronize()
    for name, kernel in PASSES:
      us = sum(e.device_time_total for e in prof.key_averages() if kernel in e.key)
      per[name].append(us / 1e3)
  return {name: float(np.median(v)) for name, v in per.items()}


def measure(reps=5):
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.fpfh_baseline import FPFHFastGlobal, FPFHRansac
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=0.05),
                                                     clip_weight_thresh=0.05, verbose=False))
  xyz0, xyz1, _ = syn.room_pair(0)
  name = card()
  ransac, fgr = FPFHRansac(dgr), FPFHFastGlobal(dgr)
  vs = dgr.voxel_size
  with torch.no_grad():
    p0, c0, _ = dgr.preprocess(xyz0, 0, _batch=0)
    p1, c1, _ = dgr.preprocess(xyz1, 1, _batch=1)
    clouds = []
    for batch, (p, c) in enumerate(((p0, c0), (p1, c1))):
      m = c._dgr_manager
      nrm = _abi.estimate_normals(p, m, vs, ransac.normal_radius_voxels * vs, ransac.normal_max_nn, batch=batch)
      clouds.append((p, nrm, m, batch))

    def fpfh_both():
      return [_abi.compute_fpfh(p, nrm, m, vs, ransac.feature_radius_voxels * vs, ransac.feature_max_nn, batch=b,
                                ld=ransac.feature_ld) for p, nrm, m, b in clouds]
    f0, f1 = fpfh_both()
    out = dict(card=name, n0=len(p0), n1=len(p1), voxel=vs, radius_voxels=ransac.feature_radius_voxels,
               max_nn=ransac.feature_max_nn)
    out.update({f'{k}_ms': round(v, 3) for k, v in pass_ms(fpfh_both, reps).items()})
    out['fpfh_call_both_ms'] = round(median_ms(fpfh_both, reps), 3)
    out['normals_both_ms'] = round(median_ms(lambda: [_abi.estimate_normals(
        p, m, vs, ransac.normal_radius_voxels * vs, ransac.normal_max_nn, batch=b) for p, _, m, b in clouds], reps), 3)
    out['knn_01_ms'] = round(median_ms(lambda: _abi.knn_top1(f0, f1), reps), 3)
    out['knn_10_ms'] = round(median_ms(lambda: _abi.knn_top1(f1, f0), reps), 3)
    m1 = c1._dgr_manager
    out['ransac_search_incl_knn_ms'] = round(median_ms(lambda: ransac._search(p0, p1, f0, f1, m1), reps), 3)
    out['fgr_search_incl_both_knn_ms'] = round(median_ms(lambda: fgr._search(p0, p1, f0, f1, m1), reps), 3)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=5)
  args = ap.parse_args()
  print(json.dumps(measure(args.reps)), flush=True)


if __name__ == '__main__':
  main()
