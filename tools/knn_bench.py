"""Feature kNN timings on the GPU.

    python tools/knn_bench.py [--out DIR] [--features FILE]

1. `_abi.knn_top1` (tensor-core path) on random unit features at 51 381 x 39 881 x 32 (the bench pair's size),
   100k x 100k x 32 and 50k x 50k x 64: CUDA events around 5 calls after 3 warm-up calls.
2. The same shapes, tensor-core against fp32 ('simt') kernel, with a check that both return the same bits.
3. Per kernel: torch.profiler (CUDA activities) times of every kNN kernel, so pass 1 and pass 2 (the second
   template argument of the sweep kernel) are reported separately.
4. The bench pair's own features: syn.room_pair(0, 250k raw points) through DeepGlobalRegistration.register with
   the seed-0 checkpoint, the executor's feature tap split at last_info['n0'].  Time of the search on them, and
   the number of pass-2 candidates per row (mean, max), counted here from float64 distances with the kernel's
   bound: column j is a candidate of row i when d2(i, j) <= min_j d2(i, j) + 4 E_i,
   E_i = knn_error_bound(|a_i|, max_j |b_j|) (csrc/knn_tc.cu).
With --out, idx1 of the bench features is written to DIR/knn_bench_idx1.npy.  The FCGF features of two runs can
differ in their last bits (the convolution accumulates with atomics), so to compare two builds on the same
features pass --features FILE: the first run saves them there and later runs load them.
"""
import argparse
import collections
import json
import os
import re
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from deepglobalregistration_b200 import _abi

SHAPES = ((51381, 39881, 32), (100000, 100000, 32), (50000, 50000, 64))


def timed(fn, warm=3, reps=5):
  for _ in range(warm):
    out = fn()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    out = fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps, out


def kernel_times(fn, reps=5):
  """{kernel name: mean ms per call} of the kNN kernels fn launches."""
  fn()
  torch.cuda.synchronize()
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
  out = collections.defaultdict(float)
  for ev in prof.events():
    if ev.device_type.name == 'CUDA' and 'knn' in ev.name:
      m = re.search(r'(knn\w*)(<[^>]*>)?', ev.name)
      out[m.group(1) + (m.group(2) or '')] += ev.device_time / 1e3 / reps
  return dict(out)


def sweep_split(kt):
  """(pass-1 ms, pass-2 ms, other kNN kernels ms) from kernel_times."""
  p = [0.0, 0.0, 0.0]
  for name, ms in kt.items():
    m = re.search(r'<\d+,\s*([12])>', name)
    p[int(m.group(1)) - 1 if m else 2] += ms
  return p


def error_bound(na, nb):
  return (0.0009765625 * 1.25 + 4e-5) * na * nb + 1e-6 * (na + nb) ** 2 + 1e-7


def candidates_per_row(F0, F1, chunk=2048):
  a, b = F0.double(), F1.double()
  nb2 = (b * b).sum(1)
  nbmax = nb2.max().sqrt()
  counts = []
  for s in range(0, a.shape[0], chunk):
    x = a[s:s + chunk]
    na2 = (x * x).sum(1)
    d2 = (na2[:, None] + nb2[None, :] - 2.0 * x @ b.T).clamp_min(0.0)
    thr = d2.min(1).values + 4.0 * error_bound(na2.sqrt(), nbmax)
    counts.append((d2 <= thr[:, None]).sum(1))
  c = torch.cat(counts).double()
  return float(c.mean()), int(c.max())


def bench_features():
  from deepglobalregistration_b200 import synthetic as syn
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  state = syn.make_checkpoint(0)
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False),
                               device=torch.device('cuda:0'))
  dgr.use_icp = False
  xyz0, xyz1, _ = syn.room_pair(0, n_raw=250_000)
  dgr.register(xyz0, xyz1)
  torch.cuda.synchronize()
  ctx, n0 = dgr._last_ctx, dgr.last_info['n0']
  F = ctx.tap('features')
  return F[:n0].contiguous(), F[n0:].contiguous(), ctx.tap('idx1').clone()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--features', default=None)
  args = ap.parse_args()
  res = {'device': torch.cuda.get_device_name(0)}
  torch.manual_seed(0)
  feats = {s: tuple(torch.nn.functional.normalize(torch.randn(n, s[2], device='cuda'), dim=1) for n in s[:2])
           for s in SHAPES}
  for (n0, n1, c), (F0, F1) in feats.items():
    ms, idx = timed(lambda: _abi.knn_top1(F0, F1))
    p1, p2, other = sweep_split(kernel_times(lambda: _abi.knn_top1(F0, F1)))
    key = f'{n0}x{n1}x{c}'
    res[key] = {'ms': ms, 'pass1_ms': p1, 'pass2_ms': p2, 'other_knn_kernels_ms': other}
    print(f'knn {key}: {ms:.3f} ms (pass 1 {p1:.3f}, pass 2 {p2:.3f}, other {other:.3f})  '
          f'{n0 * n1 * c / ms / 1e9:.2f} T pair-terms/s  checksum {int(idx.long().sum())}', flush=True)
  print('--- tc vs simt')
  for (n0, n1, c), (F0, F1) in feats.items():
    got = {m: timed(lambda: _abi.knn_top1(F0, F1, return_distance=True, mode=m), warm=2) for m in ('tc', 'simt')}
    same = all(torch.equal(a, b) for a, b in zip(got['tc'][1], got['simt'][1]))
    for m, (ms, _) in got.items():
      print(f'{m:5s} knn {n0}x{n1}x{c}: {ms:.3f} ms', flush=True)
    print(f'      tc == simt bit for bit: {same}', flush=True)
    res[f'{n0}x{n1}x{c}']['simt_ms'], res[f'{n0}x{n1}x{c}']['tc_equals_simt'] = got['simt'][0], same
  print('--- bench pair features')
  if args.features and os.path.exists(args.features):
    F0, F1 = (t.cuda() for t in torch.load(args.features))
    idx_exec = None
  else:
    F0, F1, idx_exec = bench_features()
    if args.features:
      torch.save((F0.cpu(), F1.cpu()), args.features)
  ms, idx = timed(lambda: _abi.knn_top1(F0, F1))
  p1, p2, other = sweep_split(kernel_times(lambda: _abi.knn_top1(F0, F1)))
  mean_c, max_c = candidates_per_row(F0, F1)
  res['bench_pair'] = {'n0': F0.shape[0], 'n1': F1.shape[0], 'c': F0.shape[1], 'ms': ms, 'pass1_ms': p1,
                       'pass2_ms': p2, 'other_knn_kernels_ms': other, 'candidates_mean': mean_c,
                       'candidates_max': max_c, 'equals_executor_idx1': None if idx_exec is None else bool(torch.equal(idx, idx_exec)),
                       'idx1_checksum': int(idx.long().sum())}
  print(json.dumps(res['bench_pair']), flush=True)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    np.save(os.path.join(args.out, 'knn_bench_idx1.npy'), idx.cpu().numpy())
    with open(os.path.join(args.out, 'knn_bench.json'), 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
