"""Time GoICPBaseline (Go-ICP) on the bench's full-size pair syn.room_pair(0) at the defaults (n_data 1000, G 300),
with and without trimming, for a few cubes_per_round: CUDA-event times of the distance transform and of the whole
search, rounds, cubes and distance-transform gathers per second, convergence and the final gap, with the card's
name and power limit read in the same run.  One JSON line per run.

    python tools/goicp_bench.py [--B 16 64 256] [--trim 0 0.3]
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


def card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  return out or torch.cuda.get_device_name()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[16, 64, 256])
  ap.add_argument('--trim', type=float, nargs='+', default=[0.0, 0.3])
  ap.add_argument('--dt_size', type=int, default=300)
  args = ap.parse_args()
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.goicp import GoICPBaseline
  st = syn.make_checkpoint(0, voxel_size=0.05)
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))
  xyz0, xyz1, T_gt = syn.room_pair(0)
  name = card()
  with torch.no_grad():
    p0, _, _ = dgr.preprocess(xyz0, 0, _batch=0)
    p1, _, _ = dgr.preprocess(xyz1, 1, _batch=1)
  src = p0[torch.arange(1000, device=p0.device) * len(p0) // 1000].float().contiguous()
  tgt = p1.float().contiguous()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  _abi.goicp_distance_transform(tgt, args.dt_size, 2.0, src)          # warm-up
  ev[0].record()
  _abi.goicp_distance_transform(tgt, args.dt_size, 2.0, src)
  ev[1].record()
  torch.cuda.synchronize()
  dt_ms = ev[0].elapsed_time(ev[1])
  for trim in args.trim:
    for B in args.B:
      b = GoICPBaseline(dgr, trim_fraction=trim, dt_size=args.dt_size, cubes_per_round=B)
      ev[0].record()
      T = b.register(xyz0, xyz1)
      ev[1].record()
      torch.cuda.synchronize()
      ms = ev[0].elapsed_time(ev[1])
      i = b.last_info
      te, re = syn.rte_rre(T, T_gt)
      gathers = i['translation_cubes'] * len(src)
      print(json.dumps(dict(card=name, n_s=len(src), n_t=len(tgt), G=args.dt_size, trim=trim, B=B,
                            dt_build_ms=round(dt_ms, 3), register_ms=round(ms, 1), rounds=int(i['rounds']),
                            children=int(i['children']), translation_cubes=int(i['translation_cubes']),
                            cubes_per_s=i['translation_cubes'] / ms * 1e3, dt_gathers_per_s=gathers / ms * 1e3,
                            icp_runs=int(i['icp_runs']), inner_overflows=int(i['inner_overflows']),
                            converged=int(i['converged']), gap=i['E'] - i['lb_min'], eps=i['eps'],
                            pool_high_water=int(i['pool_high_water']), rte_m=te, rre_deg=float(np.degrees(re)))),
            flush=True)


if __name__ == '__main__':
  main()
