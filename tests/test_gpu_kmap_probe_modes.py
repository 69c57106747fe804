"""The probe modes of dgr_kmap_probe_mode against the general-offset probe (every offset probed for every output
row): same-stride maps probe half the offsets and mirror the rest, kernel-3 down maps are enumerated from their
input rows.  Both must give the same bit masks, block counts, bucket offsets, meta block, pair lists and work lists,
bit for bit (the atomics are OR and integer adds)."""
import os
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


def _cloud(D, n, ext, seed):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-ext, ext, size=(n, D)), axis=0)
  c = c[g.permutation(len(c))]
  b = g.integers(0, 2, size=(len(c), 1))
  return np.concatenate([b, c], 1).astype(np.int32)


def _with_junk(rows, extra, seed):
  """rows followed by `extra` rows inside the coordinate range that the device count must hide."""
  if extra == 0:
    return rows
  g = np.random.default_rng(seed)
  junk = rows[torch.from_numpy(g.integers(0, len(rows), size=extra)).cuda()].clone()
  junk[:, 1:] += torch.from_numpy(g.integers(-1, 2, size=(extra, rows.shape[1] - 1)).astype(np.int32)).cuda()
  return torch.cat([rows, junk]).contiguous()


def _build(abi, mode, man, s_in, s_out, ks, extra=0, n_dev_override=None):
  """Kernel map from stride s_in to s_out of `man` in probe mode `mode` -> every array phase 1 and 2 write."""
  from deepglobalregistration_b200.me.coords import kernel_offsets
  P_, C_ = abi.ptr, abi.call
  m_in, m_out = man._map(s_in), man._map(s_out)
  D, dev = man.D, man.device
  offs = kernel_offsets(ks, D, s_in, dev)
  K, ncols = offs.shape[0], D + 1
  n_out, n_in = m_out.n, m_in.n
  if n_dev_override is not None:
    n_out = n_in = n_dev_override
  out_rows = _with_junk(m_out.coords, extra, 1)
  in_rows = _with_junk(m_in.coords, extra, 2)
  n_out_max, n_in_max = out_rows.shape[0], in_rows.shape[0]
  padded = extra > 0 or n_dev_override is not None
  n_out_dev = torch.tensor([n_out], dtype=torch.int32, device=dev) if padded else None
  n_in_dev = torch.tensor([n_in], dtype=torch.int32, device=dev) if padded else None
  W = abi.lib().dgr_kmap_mask_words(n_out_max)
  bits = torch.full((K * W,), -1, dtype=torch.int32, device=dev)        # poisoned: every word must be written
  cnt = torch.full((abi.lib().dgr_kmap_cnt_elems(K, n_out_max),), -1, dtype=torch.int32, device=dev)
  kofs = torch.full((K + 2,), -1, dtype=torch.int32, device=dev)
  meta = torch.full((5,), -1, dtype=torch.int32, device=dev)
  down = mode == abi.KMAP_DOWN
  bloom, n_words = None, 0
  if K > 27 and not down:
    n_words = abi.lib().dgr_bloom2_words(n_in_max)
    bloom = torch.empty(n_words, dtype=torch.int32, device=dev)
    C_('dgr_bloom2_build', P_(m_in.table.keys), m_in.table.cap, P_(bloom), n_words, abi.stream())
  tab = (P_(m_in.table.keys), P_(m_in.table.vals), m_in.table.cap)
  C_('dgr_kmap_probe_mode', mode, P_(out_rows), n_out_max, P_(n_out_dev), ncols, P_(man.spec), *tab, P_(bloom), n_words,
     P_(offs), K, P_(in_rows if down else None), n_in_max if down else 0, P_(n_in_dev if down else None),
     s_in if down else 0, P_(m_out.table.keys if down else None), P_(m_out.table.vals if down else None),
     m_out.table.cap if down else 0, P_(bits), P_(cnt), P_(kofs), P_(meta), abi.stream())
  m = meta.cpu().tolist()
  P, n_tiles = m[0], m[1]
  in_idx = torch.full((max(P, 1),), -1, dtype=torch.int32, device=dev)
  out_idx = torch.full((max(P, 1),), -1, dtype=torch.int32, device=dev)
  tile_k = torch.full((max(n_tiles, 1),), -1, dtype=torch.int32, device=dev)
  tile_start = torch.full((max(n_tiles, 1),), -1, dtype=torch.int32, device=dev)
  if P > 0:
    C_('dgr_kmap_fill', P_(bits), P_(cnt), K, n_out_max, P_(out_rows), ncols, P_(man.spec), *tab, P_(offs), P_(in_idx),
       P_(out_idx), abi.stream())
    C_('dgr_kernel_map_tiles', P_(kofs), K, abi.TILE_ROWS, n_tiles, 0, P_(tile_k), P_(tile_start), abi.stream())
  torch.cuda.synchronize()
  return dict(bits=bits, cnt=cnt, kofs=kofs, meta=meta, in_idx=in_idx, out_idx=out_idx, tile_k=tile_k,
              tile_start=tile_start)


def _check(abi, man, s_in, s_out, ks, **kw):
  mode = abi.kmap_mode(s_in, s_out, ks)
  assert mode != abi.KMAP_GENERAL
  want = _build(abi, abi.KMAP_GENERAL, man, s_in, s_out, ks, **kw)
  got = _build(abi, mode, man, s_in, s_out, ks, **kw)
  for k in want:
    assert torch.equal(got[k], want[k]), (k, man.D, s_in, s_out, ks, kw)
  return int(want['meta'][0])


def _manager(coords):
  from deepglobalregistration_b200.me.coords import CoordinateManager
  ct = coords if torch.is_tensor(coords) else torch.from_numpy(coords).cuda().contiguous()
  return CoordinateManager(ct, assume_unique=True)


MAPS = [(1, 1, 3), (2, 2, 3), (4, 4, 3), (8, 8, 3), (1, 2, 3), (2, 4, 3), (4, 8, 3)]


def test_bench_pair_maps(abi):
  """Every map of the bench pair's two networks: the FCGF network (3-D, 7^3 conv1) on the voxelised pair and the
  6-D inlier network on the full-size fixture's correspondences."""
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  gold = np.load(os.path.join(GOLD, 'fullsize_config2.npz'))
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0), clip_weight_thresh=0.05,
                                                   verbose=False))
  xyz0, xyz1, _ = syn.room_pair(0, n_raw=250_000)
  with torch.no_grad():
    _, c0, _ = d.preprocess(xyz0, 0, _batch=0)
    _, c1, _ = d.preprocess(xyz1, 1, _batch=1)
  fcgf = _manager(torch.cat((c0, c1), 0).contiguous())
  for s_in, s_out, ks in MAPS + [(1, 1, 7)]:
    assert _check(abi, fcgf, s_in, s_out, ks) > 0
  inlier = _manager(abi.inlier_coords(c0, c1, torch.from_numpy(gold['idx1']).cuda()).contiguous())
  for s_in, s_out, ks in MAPS:
    assert _check(abi, inlier, s_in, s_out, ks) > 0


@pytest.mark.parametrize('D,n,ext', [(3, 6000, 12), (6, 4000, 3)])
def test_negative_coordinates_and_device_counts(abi, D, n, ext):
  man = _manager(_cloud(D, n, ext, seed=D))
  for s_in, s_out, ks in MAPS + ([(1, 1, 5)] if D == 3 else []):
    for extra in (0, 900):                   # n_out_dev (and n_in_dev) below the row bounds
      assert _check(abi, man, s_in, s_out, ks, extra=extra) > 0


@pytest.mark.parametrize('D', [3, 6])
@pytest.mark.parametrize('corner', [1, -1])
def test_row_with_every_parent(abi, D, corner):
  """A stride-1 row odd on every axis (+1 or -1: floor parity) with all 2^D parents present at stride 2."""
  par = np.array(np.meshgrid(*[[corner - 1, corner + 1]] * D, indexing='ij')).reshape(D, -1).T
  rows = np.concatenate([np.full((1, D), corner), par], 0)
  man = _manager(np.concatenate([np.zeros((len(rows), 1)), rows], 1).astype(np.int32))
  assert man._map(2).n == 2 ** D
  _check(abi, man, 1, 1, 3)
  # the odd row reaches all 2^D parents, every even row only itself
  assert _check(abi, man, 1, 2, 3) == 2 * 2 ** D
  got = _build(abi, abi.kmap_mode(1, 2, 3), man, 1, 2, 3)
  assert int((got['in_idx'] == 0).sum()) == 2 ** D


@pytest.mark.parametrize('D', [3, 6])
def test_single_row_and_empty_levels(abi, D):
  man = _manager(np.concatenate([[[0]], np.full((1, D), -3)], 1).astype(np.int32))
  for s_in, s_out, ks in MAPS:
    assert _check(abi, man, s_in, s_out, ks) == 1
  man = _manager(_cloud(D, 500, 4, seed=11))
  for s_in, s_out, ks in MAPS:
    assert _check(abi, man, s_in, s_out, ks, extra=64, n_dev_override=0) == 0


def test_operator_path_uses_the_modes(abi):
  """me/coords.py builds its same-stride and down maps in the new modes; the pair lists equal the general probe's."""
  man = _manager(_cloud(3, 5000, 10, seed=4))
  from deepglobalregistration_b200.me.coords import CoordinateMapKey
  for s_in, conv_stride in ((1, 1), (1, 2), (2, 2)):
    _, km = man.kernel_map(CoordinateMapKey(s_in), conv_stride, 3)
    want = _build(abi, abi.KMAP_GENERAL, man, s_in, s_in * conv_stride, 3)
    assert np.array_equal(km.kofs_host, want['kofs'][:28].cpu().numpy())
    assert torch.equal(km.in_idx[:km.n_pairs], want['in_idx'][:km.n_pairs])
    assert torch.equal(km.out_idx[:km.n_pairs], want['out_idx'][:km.n_pairs])
