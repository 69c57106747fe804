"""Time Super4PCS on the bench's full-size pair syn.room_pair(0) (voxel 0.05 m): CUDA-event times of the
distance-transform build and of one round of B bases, the round's kernel time per phase (base selection, pairs, join,
fit + prefilter, selection + full LCP; torch.profiler), and the whole call at the defaults, with candidates per base,
the recovery error, and the card's name and power limit read in the same run.  One JSON line per setting.

    python tools/super4pcs_bench.py [--B 16 64] [--sample 256 512 1024]
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


def timed(fn, reps=3):
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  fn()
  best = float('inf')
  for _ in range(reps):
    ev[0].record()
    out = fn()
    ev[1].record()
    torch.cuda.synchronize()
    best = min(best, ev[0].elapsed_time(ev[1]))
  return best, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, nargs='+', default=[16, 64])
  ap.add_argument('--sample', type=int, nargs='+', default=[256, 512, 1024])
  args = ap.parse_args()
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.super4pcs import Super4PCSBaseline
  st = syn.make_checkpoint(0, voxel_size=0.05)
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))
  xyz0, xyz1, T_gt = syn.room_pair(0)
  name = card()
  with torch.no_grad():
    p0, _, _ = dgr.preprocess(xyz0, 0, _batch=0)
    p1, _, _ = dgr.preprocess(xyz1, 1, _batch=1)
  tgt = p1.float().contiguous()
  dt_ms, _ = timed(lambda: _abi.goicp_distance_transform(tgt, 300, 2.0, tgt[:1024]))
  for n in args.sample:
    src = p0[torch.arange(n, device=p0.device) * len(p0) // n].float().contiguous()
    nq = min(4096, 2 * n)
    for B in args.B:
      kw = dict(n_sample_tgt=nq, delta=0.1, max_bases=B, bases_per_round=B, terminate_fraction=1.0)
      one_ms, res = timed(lambda: _abi.super4pcs(src, tgt, return_log=True, **kw))
      log = res[1].cpu().numpy()
      phase = {}
      with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _abi.super4pcs(src, tgt, **kw)
        torch.cuda.synchronize()
      for e in prof.key_averages():
        k = e.key
        group = ('dt' if 'dt_' in k or 'normalise' in k or 'stats' in k else 'base' if 's4_base' in k else
                 'pairs' if 's4_pair' in k else 'join' if 's4_hash' in k or 's4_join' in k else
                 'fit_prefilter' if 's4_fit' in k else 'verify' if 's4_select' in k or 's4_lcp' in k else None)
        if group:
          phase[group] = phase.get(group, 0.0) + getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0)) / 1e3
      v = log[log[:, 4] == 1]
      print(json.dumps(dict(card=name, n_s=n, n_q=nq, n_t=len(tgt), B=B, dt_build_ms=round(dt_ms, 3),
                            round_ms=round(one_ms, 2), round_minus_dt_ms=round(one_ms - dt_ms, 2),
                            valid_bases=len(v), s1_mean=float(v[:, 5].mean()) if len(v) else 0.0,
                            candidates_mean=float(v[:, 7].mean()) if len(v) else 0.0,
                            candidates_dropped_mean=float(v[:, 8].mean()) if len(v) else 0.0,
                            best_lcp_fraction=float(res[0][16]),
                            phase_ms={k: round(v, 3) for k, v in phase.items()})), flush=True)
    b = Super4PCSBaseline(dgr, sample_size=n)
    ms, T = timed(lambda: b.register(xyz0, xyz1), reps=2)
    te, re = syn.rte_rre(T, T_gt)
    i = b.last_info
    print(json.dumps(dict(card=name, n_s=n, n_q=b.n_sample_tgt, defaults=True, register_ms=round(ms, 1),
                          rounds=int(i['rounds']), bases=int(i['bases']), valid_bases=int(i['valid_bases']),
                          candidates=int(i['candidates']), candidates_dropped=int(i['candidates_dropped']),
                          pairs_dropped=int(i['pairs_dropped']), lcp_fraction=i['lcp_fraction'], rte_m=te,
                          rre_deg=float(np.degrees(re)))), flush=True)


if __name__ == '__main__':
  main()
