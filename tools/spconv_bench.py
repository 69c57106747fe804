"""Tensor-core sparse-convolution timings, launch shape by launch shape, on the bench pair's kernel maps.

    python tools/spconv_bench.py [--lib OTHER/libdgr_b200.so] [--out DIR] [--reps N]

Registers syn.room_pair(0, 250k raw points) once with the seed-0 checkpoint, takes the executor's 3-D and 6-D
coordinate taps and rebuilds, through me/coords.py, the kernel maps of the two ResUNetBN2C passes (strides 1 / 2 / 4
/ 8, the stride-2 maps and their transposes).  Every distinct (D, map, cin, cout) the networks launch on the tensor
cores - 3xFP16 where cout >= 128 and cin % 64 == 0, 3xTF32 elsewhere, as the executor chooses - is timed with CUDA
events over `reps` launches after warm-up, on random non-negative activations (the kernel's time does not depend
on the values).  Printed per shape: pairs, tiles, ms, the algorithmic bytes and FLOPs of exec.cu::run_conv
(P (cin + cout) 4 + 8 P + K_nonempty cin cout 4 bytes, 2 P cin cout FLOP) and what share of the data-sheet peaks
(3.35 TB/s HBM3, 989 TFLOP/s dense FP16 / 495 TF32, H100 SXM at 700 W) they amount to; the card's name, power limit
and SM clock as nvidia-smi reports them head the table.

--lib loads a second build of the library through ctypes and alternates the two builds launch by launch on the
same buffers in this process (the C ABI and the packed weight layouts are the same), so `ms_other` and the ratio
come from one run.
"""
import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from deepglobalregistration_b200 import _abi

HBM_PEAK, F16_PEAK, TF32_PEAK = 3.35e12, 989e12, 495e12
C_ENC, C_TR = (32, 64, 128, 256), (64, 64, 64, 128)          # ResUNetBN2C


def bench_coords():
  from deepglobalregistration_b200 import synthetic as syn
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0), clip_weight_thresh=0.05,
                                                     verbose=False), device=torch.device('cuda:0'))
  dgr.use_icp = False
  xyz0, xyz1, _ = syn.room_pair(0, n_raw=250_000)
  dgr.register(xyz0, xyz1)
  torch.cuda.synchronize()
  ctx = dgr._last_ctx
  return {3: ctx.tap('coords').clone(), 6: ctx.tap('coords6').clone()}


def network_launches(coords):
  """[(map name, km, cin, cout)] of one ResUNetBN2C forward over `coords`, tensor-core layers only."""
  from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey
  man = CoordinateManager(coords.contiguous())
  key, same, down, up = CoordinateMapKey(1), [], [], []
  for level in range(4):
    same.append(man.kernel_map(key, 1, 3)[1])
    if level < 3:
      nxt, km = man.kernel_map(key, 2, 3)
      down.append(km)
      up.append(man.transpose_kernel_map(nxt, 2, 3)[1])
      key = nxt
  out = []
  for l in range(4):
    s = 1 << l
    if l > 0:
      out.append((f's{s >> 1}->{s}', down[l - 1], C_ENC[l - 1], C_ENC[l]))
    out += [(f's{s}', same[l], C_ENC[l], C_ENC[l])] * 2
  tr_in = (None, C_ENC[1] + C_TR[2], C_ENC[2] + C_TR[3], C_ENC[3])
  for l in (3, 2, 1):
    s = 1 << l
    out.append((f's{s}->{s >> 1}', up[l - 1], tr_in[l], C_TR[l]))
    out += [(f's{s >> 1}', same[l - 1], C_TR[l], C_TR[l])] * 2
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--lib', default=None, help='a second libdgr_b200.so to alternate with')
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=20)
  args = ap.parse_args()
  _abi.require_device('cuda')
  card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                        capture_output=True, text=True).stdout.strip()
  print(f'card: {card}', flush=True)
  other = _abi.bind(args.lib, ('dgr_spconv_tc_fwd', 'dgr_spconv_tc_f16_fwd', 'dgr_last_error')) if args.lib else None
  res = {'card': card, 'other_lib': args.lib, 'rows': []}
  seen = {}
  for D, coords in bench_coords().items():
    for name, km, cin, cout in network_launches(coords):
      if (D, name, cin, cout) in seen:
        seen[(D, name, cin, cout)]['launches_per_pair'] += 1
        continue
      f16 = cout >= 128 and cin % 64 == 0
      g = torch.Generator(device='cuda').manual_seed(cin + cout)
      feat = torch.rand(km.n_in, cin, device='cuda', generator=g)
      W = (torch.rand(km.K, cin, cout, device='cuda', generator=g) - 0.5) / cin
      outb = torch.zeros(km.n_out, cout, device='cuda')
      head = [_abi.ptr(feat), cin, None, cout, _abi.ptr(km.in_idx), _abi.ptr(km.out_idx), _abi.ptr(km.kofs),
              _abi.ptr(km.tile_k), _abi.ptr(km.tile_start), km.n_tiles, _abi.TILE_ROWS]
      if f16:
        packed = torch.empty(4 * km.K * cin * cout, dtype=torch.uint8, device='cuda')
        wscale, amax = torch.empty(2, device='cuda'), torch.empty(1, device='cuda')
        _abi.call('dgr_pack_weight_f16', _abi.ptr(W), km.K, cin, cout, _abi.ptr(packed), _abi.ptr(wscale), _abi.stream())
        _abi.call('dgr_absmax_f32', _abi.ptr(feat), feat.numel(), _abi.ptr(amax), _abi.stream())
        fn, tail = 'dgr_spconv_tc_f16_fwd', [_abi.ptr(amax), _abi.ptr(wscale), _abi.ptr(outb), _abi.stream()]
      else:
        packed = _abi.pack_weight_tf32(W, km.K, cin, cout)
        fn, tail = 'dgr_spconv_tc_fwd', [3, _abi.ptr(outb), _abi.stream()]
      head[2] = _abi.ptr(packed)
      del W

      def this():
        _abi.call(fn, *head, *tail)

      def that():
        if getattr(other, fn)(*head, *tail) != 0:
          raise RuntimeError(other.dgr_last_error().decode())

      builds = [this] + ([that] if other else [])
      for launch in builds * 3:
        launch()
      ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
            for _ in builds]
      for r in range(args.reps):                   # alternate the builds launch by launch
        for b, launch in enumerate(builds):
          ev[b][r][0].record()
          launch()
          ev[b][r][1].record()
      torch.cuda.synchronize()
      ms = [sorted(e0.elapsed_time(e1) for e0, e1 in evs)[len(evs) // 2] for evs in ev]
      nonempty = int((km.kofs_host[1:] > km.kofs_host[:-1]).sum())
      P = int(km.n_pairs)
      by, fl = P * (cin + cout) * 4.0 + 8.0 * P + nonempty * cin * cout * 4.0, 2.0 * P * cin * cout
      row = {'D': D, 'map': name, 'cin': cin, 'cout': cout, 'mode': '3xfp16' if f16 else '3xtf32', 'K': km.K, 'P': P,
             'n_tiles': int(km.n_tiles), 'launches_per_pair': 1, 'ms': ms[0], 'GB': by / 1e9, 'GFLOP': fl / 1e9,
             'share_hbm_peak': by / (ms[0] * 1e-3) / HBM_PEAK,
             'share_tensor_peak': fl / (ms[0] * 1e-3) / (F16_PEAK if f16 else TF32_PEAK)}
      if other:
        row['ms_other'], row['other_over_this'] = ms[1], ms[1] / ms[0]
      seen[(D, name, cin, cout)] = row
      res['rows'].append(row)
      print(json.dumps(row), flush=True)
      del feat, outb, packed
  tot = sum(r['ms'] * r['launches_per_pair'] for r in res['rows'])
  line = f'sum over one pair: {tot:.3f} ms'
  if other:
    tot_o = sum(r['ms_other'] * r['launches_per_pair'] for r in res['rows'])
    line += f', other build {tot_o:.3f} ms ({tot_o / tot:.3f}x)'
    res['sum_ms_other'] = tot_o
  res['sum_ms'] = tot
  print(line, flush=True)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'spconv_bench.json'), 'w') as fh:
      json.dump(res, fh, indent=1)


if __name__ == '__main__':
  main()
