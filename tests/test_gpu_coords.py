"""GPU parity of the integer coordinate kernels against the oracle: bit-exact."""
import numpy as np
import pytest
import torch

from oracle import sparse_ops as so

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


def _cloud(seed, n, scale=3.0, dtype=np.float64):
  g = np.random.default_rng(seed)
  return (g.normal(size=(n, 3)) * scale).astype(dtype)


def _quantize_gpu(abi, xyz, voxel):
  return abi.voxelise(torch.from_numpy(xyz).cuda(), voxel)


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
@pytest.mark.parametrize('n,voxel', [(5000, 0.25), (200000, 0.05), (1, 0.1), (37, 5.0)])
def test_quantize_first_bit_exact(abi, dtype, n, voxel):
  xyz = _cloud(n, n, dtype=dtype)
  coords, spec, table, sel, inv, m = _quantize_gpu(abi, xyz, voxel)
  want_c, want_sel = so.quantize_first(xyz, voxel)
  assert m == len(want_sel)
  assert np.array_equal(sel.cpu().numpy(), want_sel)
  got_c = abi.gather_rows_i32(coords, sel, m).cpu().numpy()
  assert np.array_equal(got_c[:, 1:], want_c) and (got_c[:, 0] == 0).all()
  # inverse: every raw row maps to the representative of its voxel
  inv = inv.cpu().numpy()[:n]
  raw = np.floor(xyz / voxel).astype(np.int32)
  assert np.array_equal(raw, want_c[inv])
  # the table now maps a voxel to its row in the deduplicated cloud
  found = abi.hash_find(torch.from_numpy(got_c).cuda(), spec, table).cpu().numpy()
  assert np.array_equal(found, np.arange(m))


def test_quantize_voxel_boundaries_float64(abi):
  # points that sit exactly on / next to voxel faces: division must be IEEE double division
  v = 0.05
  base = np.arange(-40, 40, dtype=np.float64)[:, None] * v
  xyz = np.concatenate([np.repeat(base, 3, 1), np.repeat(np.nextafter(base, -np.inf), 3, 1),
                        np.repeat(np.nextafter(base, np.inf), 3, 1)])
  d = torch.from_numpy(xyz).cuda()
  coords, _ = abi.quantize_points(d, v)
  assert np.array_equal(coords.cpu().numpy()[:, 1:], np.floor(xyz / v).astype(np.int32))
  x32 = xyz.astype(np.float32)
  coords32, _ = abi.quantize_points(torch.from_numpy(x32).cuda(), v)
  assert np.array_equal(coords32.cpu().numpy()[:, 1:], np.floor(x32 / v).astype(np.int32))


def test_duplicates_all_same_voxel(abi):
  xyz = np.full((1000, 3), 0.01)
  _, _, _, sel, inv, m = _quantize_gpu(abi, xyz, 0.05)
  assert m == 1 and sel.cpu().tolist() == [0] and (inv.cpu().numpy()[:1000] == 0).all()


def test_hash_find_misses(abi):
  xyz = _cloud(3, 4000)
  coords, spec, table, sel, _, m = _quantize_gpu(abi, xyz, 0.2)
  kept = abi.gather_rows_i32(coords, sel, m).cpu().numpy()
  probe = kept.copy()
  probe[:, 1] += 1
  want = so.kernel_map(kept, kept, np.array([[1, 0, 0]]))[0]
  exp = np.full(m, -1)
  exp[want[1]] = want[0]
  got = abi.hash_find(torch.from_numpy(probe).cuda(), spec, table).cpu().numpy()
  assert np.array_equal(got, exp)
  far = np.array([[0, 10 ** 6, 0, 0], [5, 0, 0, 0]], np.int32)     # outside the packed range
  assert abi.hash_find(torch.from_numpy(far).cuda(), spec, table).cpu().tolist() == [-1, -1]


def _manager(abi, coords_np):
  from deepglobalregistration_b200.me.coords import CoordinateManager
  return CoordinateManager(torch.from_numpy(coords_np).cuda())


@pytest.mark.parametrize('D', [3, 6])
def test_strided_and_coarse_maps_bit_exact(abi, D):
  from deepglobalregistration_b200.me.coords import CoordinateMapKey
  g = np.random.default_rng(D)
  c = np.unique(g.integers(-40, 40, size=(6000, D)), axis=0)
  c = c[g.permutation(len(c))]
  coords = np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)
  man = _manager(abi, coords)                   # one map per _map() call
  # all three levels from one call, as the executor builds them (dgr_coarse_maps)
  multi, tables, n_out = abi.coarse_maps(man.coordinates(CoordinateMapKey(1)), man.spec, [2, 4, 8])
  n_out = n_out.cpu().tolist()
  cur = coords
  for l, s in enumerate((2, 4, 8)):
    want, _ = so.stride_coords(cur, s)
    for got, table in ((man.coordinates(CoordinateMapKey(s)), man._maps[s].table), (multi[l, :n_out[l]], tables[l])):
      assert np.array_equal(got.cpu().numpy(), want), f'stride {s}'
      # the table maps every coarse coordinate to its row
      rows = abi.hash_find(torch.from_numpy(want).cuda(), man.spec, table).cpu().numpy()
      assert np.array_equal(rows, np.arange(len(want))), f'stride {s}'
    cur = want


def _check_kmap(km, buckets):
  kofs = km.kofs_host
  ii, jj = km.in_idx.cpu().numpy(), km.out_idx.cpu().numpy()
  assert km.n_pairs == sum(len(b[0]) for b in buckets)
  for kap, (wi, wj) in enumerate(buckets):
    a, b = kofs[kap], kofs[kap + 1]
    assert np.array_equal(jj[a:b], wj), f'kappa {kap} out rows'
    assert np.array_equal(ii[a:b], wi), f'kappa {kap} in rows'
  # work list covers every pair exactly once
  tk, ts = km.tile_k.cpu().numpy()[:km.n_tiles], km.tile_start.cpu().numpy()[:km.n_tiles]
  covered = np.zeros(max(km.n_pairs, 1), np.int32)
  for k, s in zip(tk, ts):
    e = min(s + 128, kofs[k + 1])
    assert kofs[k] <= s < e
    covered[s:e] += 1
  assert (covered[:km.n_pairs] == 1).all()
  if km.nbr is not None:
    # the dense neighbour table kept for the conv1 table kernel: nbr[kappa, j] = i of every pair, otherwise -1
    want = np.full((len(buckets), km.n_out), -1, np.int32)
    for kap, (wi, wj) in enumerate(buckets):
      want[kap, wj] = wi
    assert np.array_equal(km.nbr.cpu().numpy(), want)


@pytest.mark.parametrize('D,ks', [(3, 3), (3, 5), (3, 7), (6, 3)])
def test_kernel_maps_bit_exact(abi, D, ks):
  from deepglobalregistration_b200.me.coords import CoordinateMapKey
  g = np.random.default_rng(10 * D + ks)
  span = 14 if D == 3 else 3
  c = np.unique(g.integers(-span, span, size=(3000, D)), axis=0)
  c = c[g.permutation(len(c))]
  coords = np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)
  man = _manager(abi, coords)
  _, km = man.kernel_map(CoordinateMapKey(1), 1, ks)
  assert (km.nbr is not None) == (D == 3 and ks > 3)
  _check_kmap(km, so.kernel_map(coords, coords, so.kernel_offsets(ks, D, 1)))
  if ks == 3:
    # stride-2 map and its transposed use, then the 3^D map on the coarse level
    key2, kd = man.kernel_map(CoordinateMapKey(1), 2, 3)
    coarse, _ = so.stride_coords(coords, 2)
    down = so.kernel_map(coords, coarse, so.kernel_offsets(3, D, 1))
    _check_kmap(kd, down)
    _, kt = man.transpose_kernel_map(key2, 2, 3)
    assert torch.equal(kt.in_idx, kd.out_idx) and torch.equal(kt.out_idx, kd.in_idx)
    _, k2 = man.kernel_map(key2, 1, 3)
    _check_kmap(k2, so.kernel_map(coarse, coarse, so.kernel_offsets(3, D, 2)))


def test_duplicate_coordinates_rejected(abi):
  c = np.array([[0, 1, 2, 3], [0, 1, 2, 3]], np.int32)
  with pytest.raises(ValueError):
    _manager(abi, c)


def test_empty_inputs(abi):
  d = torch.zeros(0, 3, dtype=torch.float64, device='cuda')
  _, _, _, sel, _, n = abi.voxelise(d, 0.05)
  assert n == 0 and sel.numel() == 0
