"""The pipelined tensor-core sparse convolution over runs of tiles, against fp64 and against itself.

A CTA of spconv_tc_kernel works through a run of consecutive tiles with a producer warpgroup running ahead of two
consumer warpgroups through a two-stage ring whose position carries across tile boundaries.  The launcher picks the
run length from the tile count (one tile per CTA until the grid covers the device twice, then up to
spconv_ring::kMaxRun), so the maps here are built to given tile counts: single tiles, counts around each change of
run length, and counts where every CTA wraps the ring many times.  Buckets keep the sizes of test_gpu_conv_fp64
(tile edges, partial last tiles, empty offsets), so runs straddle offsets, and on the paired list the padding tiles
fall on the first, a middle and the last position of a run.  Criterion: oracle/precision.py.
"""
import numpy as np
import pytest
import torch

from oracle import precision as pr
from test_gpu_conv_fp64 import SIZES, _buckets, _check, _data, _f16, _kmap, _refs, _tc, abi  # noqa: F401

pytestmark = pytest.mark.gpu

N_ROWS = 3000
MAX_RUN, MIN_WAVES = 8, 2                # spconv_ring::kMaxRun, kMinWaves
TILES_PER_PASS = sum((s + 127) // 128 for s in SIZES)


def _sizes_for(n_tiles):
  """Bucket sizes, cycling through SIZES, whose plain tile list has exactly n_tiles tiles."""
  sizes, left, i = [], n_tiles, 0
  while left > 0:
    s = SIZES[i % len(SIZES)]
    i += 1
    tiles = (s + 127) // 128
    if tiles > left:
      s, tiles = left * 128 - 5, left       # a partial last tile
    sizes.append(s)
    left -= tiles
  return sizes + [0]                        # an empty last offset


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _run_both(abi, mode, feat, W, b, kms, case):
  refs = _refs(feat, W, b, N_ROWS)
  if mode == 'f16':
    floor = pr.f16_floor(feat, W, b, N_ROWS)
    for name, km in kms:
      _check('3xfp16', f'{case} {name}', _f16(abi, feat, W, km), *refs, floor)
  else:
    fd, Wt = feat.cuda(), abi.pack_weight_tf32(W.cuda(), len(b), W.shape[1], W.shape[2])
    for name, km in kms:
      _check('3xtf32', f'{case} {name}', _tc(abi, fd, Wt, km, 3), *refs)


@pytest.mark.parametrize('mode,cin,cout', [('tf32', 32, 32), ('tf32', 96, 48), ('f16', 64, 128), ('f16', 192, 256)])
def test_tile_counts(abi, mode, cin, cout):
  """1, kMaxRun - 1, kMaxRun, kMaxRun + 1 tiles; tile counts one below, at and above the launches where the run
  length becomes 2, 3 and kMaxRun (for one and for two resident CTAs per SM); and, at the narrower shapes, more than
  3 * kMaxRun * SMs tiles, where every CTA of a full wave goes round the ring at least four times."""
  sms = _sms()
  counts = [1, MAX_RUN - 1, MAX_RUN, MAX_RUN + 1]
  if cin * cout <= 64 * 128:
    for resident in (sms, 2 * sms):
      for run in (2, 3, MAX_RUN):
        counts += [MIN_WAVES * resident * run - 1, MIN_WAVES * resident * run, MIN_WAVES * resident * run + 1]
    counts.append(4 * MAX_RUN * sms + 3)
  else:
    counts += [MIN_WAVES * sms * run + d for run, d in ((2, -1), (2, 0), (2, 1), (3, 1))]
  for n_tiles in sorted(set(counts)):
    sizes = _sizes_for(n_tiles)
    b = _buckets(sizes, N_ROWS, N_ROWS, seed=n_tiles)
    km, kp = _kmap(abi, b, N_ROWS, N_ROWS, False), _kmap(abi, b, N_ROWS, N_ROWS, True)
    assert km.n_tiles == n_tiles and kp.n_tiles > n_tiles
    feat, W = _data(N_ROWS, cin, len(b), cout, seed=n_tiles + cin)
    _run_both(abi, mode, feat, W, b, (('plain', km), ('paired', kp)), f'{cin}->{cout} tiles{n_tiles}')


@pytest.fixture(scope='module')
def medium(abi):
  """(buckets, plain km, paired km): 26 passes over SIZES, ~1300 tiles - runs of 2 to 5 tiles on a 132-SM device."""
  b = _buckets(list(SIZES) * 26, N_ROWS, N_ROWS, seed=2)
  return b, _kmap(abi, b, N_ROWS, N_ROWS, False), _kmap(abi, b, N_ROWS, N_ROWS, True)


@pytest.mark.parametrize('mode,cin', [('f16', 64), ('f16', 128), ('f16', 192), ('f16', 256),
                                      ('tf32', 32), ('tf32', 64), ('tf32', 96), ('tf32', 128)])
def test_chunks_and_widths(abi, medium, mode, cin):
  """1, 2, 3 and 4 chunks per tile (odd counts leave the ring at a different stage for every other tile) at every
  accumulator width, one of them padded, on the plain and the paired list."""
  b, km, kp = medium
  for cout in (32, 96, 128, 256) if mode == 'f16' else (32, 48, 128, 256):
    feat, W = _data(N_ROWS, cin, len(b), cout, seed=cin * 1000 + cout + 3)
    _run_both(abi, mode, feat, W, b, (('plain', km), ('paired', kp)), f'{cin}->{cout}')


@pytest.mark.parametrize('mode,cin,cout', [('f16', 192, 256), ('f16', 64, 128), ('tf32', 96, 64), ('tf32', 32, 256)])
def test_run_equals_single_tile_launches(abi, mode, cin, cout):
  """Carry-over across tiles.  Every pair has its own out row, so each output is one red onto zero and nothing
  reorders: one launch over the whole tile list must equal, bit for bit, the list evaluated one tile per launch."""
  g = np.random.default_rng(5)
  sizes = list(SIZES) * 26
  P = sum(sizes)
  rows = g.permutation(P)
  b, at = [], 0
  for s in sizes:
    b.append((g.choice(N_ROWS, s, replace=False).astype(np.int64), np.sort(rows[at:at + s])))
    at += s
  feat, W = _data(N_ROWS, cin, len(b), cout, seed=cin + cout)
  fd, Wd = feat.cuda(), W.cuda().contiguous()
  if mode == 'f16':
    packed = torch.empty(4 * len(b) * cin * cout, dtype=torch.uint8, device='cuda')
    wscale, amax = torch.empty(2, device='cuda'), torch.empty(1, device='cuda')
    abi.call('dgr_pack_weight_f16', abi.ptr(Wd), len(b), cin, cout, abi.ptr(packed), abi.ptr(wscale), abi.stream())
    abi.call('dgr_absmax_f32', abi.ptr(fd), fd.numel(), abi.ptr(amax), abi.stream())
  else:
    packed = abi.pack_weight_tf32(Wd, len(b), cin, cout)

  def launch(km, first, n_tiles, out):
    head = (abi.ptr(fd), cin, abi.ptr(packed), cout, abi.ptr(km.in_idx), abi.ptr(km.out_idx), abi.ptr(km.kofs),
            abi.ptr(km.tile_k[first:]), abi.ptr(km.tile_start[first:]), n_tiles, abi.TILE_ROWS)
    if mode == 'f16':
      abi.call('dgr_spconv_tc_f16_fwd', *head, abi.ptr(amax), abi.ptr(wscale), abi.ptr(out), abi.stream())
    else:
      abi.call('dgr_spconv_tc_fwd', *head, 3, abi.ptr(out), abi.stream())

  for pair in (False, True):
    km = _kmap(abi, b, N_ROWS, P, pair)
    assert km.n_tiles >= TILES_PER_PASS * 26
    whole, single = torch.zeros(P, cout, device='cuda'), torch.zeros(P, cout, device='cuda')
    launch(km, 0, km.n_tiles, whole)
    for t in range(km.n_tiles):
      launch(km, t, 1, single)
    assert bool(whole.any()) and torch.equal(whole, single), f'{mode} {cin}->{cout} paired {pair}'
