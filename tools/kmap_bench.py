"""GPU time of every kernel-map launch of the bench pair's coordinate phase (syn.room_pair(0, 250k raw points)):
the FCGF network's 3-D maps (3^3 at strides 1..8, the 7^3 conv1 map, the three stride-2 down maps) and the inlier
network's 6-D maps on the fixture's correspondences (tests/golden/fullsize_config2.npz idx1), built as the native
executor builds them (coarse levels from the stride-1 rows, the level-0 Bloom filter size everywhere).

Every probe is timed in the general mode (every offset probed per output row) and, when the library has
dgr_kmap_probe_mode, in the mode the executor picks for the map; the two must give identical masks, counts and
pair lists.  `*_ms` is the median of `reps` calls bracketed by CUDA events, `probe_dev_ms_*` the mean device time
of the kernels and memsets of one call (torch.profiler).
Usage: python tools/kmap_bench.py [reps] [out.json]"""
import json
import os
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from deepglobalregistration_b200 import _abi
from deepglobalregistration_b200 import synthetic as syn
from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
from deepglobalregistration_b200.me.coords import CoordinateManager, kernel_offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
out_json = sys.argv[2] if len(sys.argv) > 2 else None
HAS_MODES = 'dgr_kmap_probe_mode' in _abi.DECLARATIONS
P, C = _abi.ptr, _abi.call


def device_ms(fn):
  """Mean device time of one call: the kernels and memsets it enqueues, from torch.profiler's CUDA activities.
  For launches of a few microseconds the event time above is the host's enqueue time as much as the GPU's."""
  fn()
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
  us = sum(e.time_range.elapsed_us() for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
  return us / 1000.0 / reps


def median_ms(fn):
  fn()
  ts = []
  for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
  return float(np.median(ts))


def bench_map(man, words, lin, lout, ks):
  """-> row of the table for the map from level lin to level lout (level l: tensor stride 2^l)."""
  s_in, s_out = 1 << lin, 1 << lout
  m_in, m_out = man._map(s_in), man._map(s_out)
  D, dev = man.D, man.device
  offs = kernel_offsets(ks, D, s_in, dev)
  K, ncols, n_out = offs.shape[0], D + 1, m_out.n
  W = _abi.lib().dgr_kmap_mask_words(n_out)
  use_bloom = K > 27
  bloom = torch.empty(words, dtype=torch.int32, device=dev) if use_bloom else None
  if use_bloom:
    C('dgr_bloom2_build', P(m_in.table.keys), m_in.table.cap, P(bloom), words, _abi.stream())
  nw = words if use_bloom else 0
  tab = (P(m_in.table.keys), P(m_in.table.vals), m_in.table.cap)

  def buffers():
    return (torch.empty(K * W, dtype=torch.int32, device=dev),
            torch.empty(_abi.lib().dgr_kmap_cnt_elems(K, n_out), dtype=torch.int32, device=dev),
            torch.empty(K + 2, dtype=torch.int32, device=dev), torch.empty(5, dtype=torch.int32, device=dev))

  def general(b):
    C('dgr_kmap_probe', P(m_out.coords), n_out, None, ncols, P(man.spec), *tab, P(bloom), nw, P(offs), K, P(b[0]),
      P(b[1]), P(b[2]), P(b[3]), _abi.stream())

  mode = _abi.kmap_mode(s_in, s_out, ks) if HAS_MODES else None

  def moded(b):
    down = mode == _abi.KMAP_DOWN       # reads no filter
    C('dgr_kmap_probe_mode', mode, P(m_out.coords), n_out, None, ncols, P(man.spec), *tab, P(None if down else bloom),
      0 if down else nw, P(offs), K,
      P(m_in.coords), m_in.n, None, s_in, P(m_out.table.keys), P(m_out.table.vals), m_out.table.cap, P(b[0]),
      P(b[1]), P(b[2]), P(b[3]), _abi.stream())

  runs = [('general', general)] + ([('mode', moded)] if mode is not None else [])
  row = {'D': D, 'map': f's{s_in}->s{s_out} k{ks}', 'K': K, 'rows_out': n_out, 'rows_in': m_in.n}
  first = None
  for name, fn in runs:
    b = buffers()
    row[f'probe_ms_{name}'] = median_ms(lambda: fn(b))
    row[f'probe_dev_ms_{name}'] = device_ms(lambda: fn(b))
    fn(b)
    meta = b[3].cpu().tolist()
    Pn, n_tiles = meta[0], meta[1]
    ii = torch.empty(max(Pn, 1), dtype=torch.int32, device=dev)
    jj = torch.empty(max(Pn, 1), dtype=torch.int32, device=dev)
    tk = torch.empty(max(n_tiles, 1), dtype=torch.int32, device=dev)
    ts = torch.empty(max(n_tiles, 1), dtype=torch.int32, device=dev)

    def fill():
      C('dgr_kmap_fill', P(b[0]), P(b[1]), K, n_out, P(m_out.coords), ncols, P(man.spec), *tab, P(offs), P(ii), P(jj),
        _abi.stream())

    def tiles():
      C('dgr_kernel_map_tiles', P(b[2]), K, _abi.TILE_ROWS, n_tiles, 0, P(tk), P(ts), _abi.stream())

    if name == 'general':
      row['pairs'], row['probes_general'] = Pn, K * n_out
      row['fill_ms'] = median_ms(fill) if Pn else 0.0
      row['tiles_ms'] = median_ms(tiles) if Pn else 0.0
    fill(); tiles()
    torch.cuda.synchronize()
    got = [b[0], b[1], b[2], b[3], ii[:Pn], jj[:Pn], tk[:n_tiles], ts[:n_tiles]]
    if first is None:
      first = got
    else:
      row['identical'] = all(torch.equal(a, c) for a, c in zip(first, got))
      row['mode'] = mode
  return row


def main():
  assert torch.cuda.is_available(), 'kmap_bench times GPU launches: no CUDA device'
  gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'fullsize_config2.npz'))
  state = syn.make_checkpoint(0)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False))
  xyz0, xyz1, _ = syn.room_pair(0, n_raw=250_000)
  with torch.no_grad():
    _, c0, _ = d.preprocess(xyz0, 0, _batch=0)
    _, c1, _ = d.preprocess(xyz1, 1, _batch=1)
  idx1 = torch.from_numpy(gold['idx1']).cuda()
  nets = [('fcgf', torch.cat((c0, c1), 0).contiguous(), 7),
          ('inlier', _abi.inlier_coords(c0, c1, idx1).contiguous(), 3)]
  rows = []
  for net, coords, conv1 in nets:
    man = CoordinateManager(coords, assume_unique=True)
    words = _abi.lib().dgr_bloom2_words(coords.shape[0])
    maps = [(l, l, 3) for l in range(4)] + [(l, l + 1, 3) for l in range(3)]
    if conv1 != 3:
      maps.append((0, 0, conv1))
    for lin, lout, ks in maps:
      r = bench_map(man, words, lin, lout, ks)
      r['net'] = net
      rows.append(r)
      print(json.dumps(r), flush=True)
  for D in (3, 6):
    sel = [r for r in rows if r['D'] == D]
    tot = {k: round(sum(r.get(k, 0.0) for r in sel), 4)
           for k in ('probe_ms_general', 'probe_ms_mode', 'probe_dev_ms_general', 'probe_dev_ms_mode', 'fill_ms', 'tiles_ms')}
    print(json.dumps({'D': D, 'totals': tot}), flush=True)
  ok = all(r.get('identical', True) for r in rows)
  print('KMAP_BENCH', torch.cuda.get_device_name(), 'IDENTICAL' if ok else 'DIFFERENT', flush=True)
  if out_json:
    with open(out_json, 'w') as fh:
      json.dump({'device': torch.cuda.get_device_name(), 'reps': reps, 'rows': rows}, fh, indent=1)
  sys.exit(0 if ok else 1)


if __name__ == '__main__':
  main()
