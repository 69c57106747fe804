"""The fused pair executor's voxelisation (dgr_pair_register: what register(), register_batch() and bench.py run)
against fp64 / exact-integer references evaluated on exactly the rows the kernels read.

The executor keys every point as floor(x / voxel) in the input dtype, keeps the first point of each voxel, and hands
its ICP refine (and the safeguard's ICP) float32 rows searched through that table with cell = voxel and radius
2 voxel.  Every row must lie in the cell it is keyed under (DESIGN.md §3): the rows are checked against
`rows_in_cells`, against what preprocess() returns for the same input, and through the search itself.  Non-finite
coordinates and key extents beyond 63 packed bits are refused, and a refused pair leaves its context usable.

All clouds stay far below the coordinate magnitude where a cell holds no float32 value (|x| 2^-23 ~ cell / 4): no
float32 row can agree with its key there, and this file does not test such clouds."""
import math
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import pose_graph as opg
from oracle import sparse_ops as so
from oracle.icp import icp_point_to_point
from test_abi_and_host import ordered
from test_gpu_hash_search_edges import rows_in_cells, snapped_cloud, straddling_pairs

pytestmark = pytest.mark.gpu

VOXELS = (0.025, 0.05, 0.0625, 0.3)
DTYPES = ((np.float64, np.float64), (np.float32, np.float32), (np.float64, np.float32), (np.float32, np.float64))
NOT_FINITE = 'coordinates are not finite, or their extent does not fit a 63-bit packed key'
EXTENT = 'extent does not fit a 63-bit packed key'

_DGR = {}


def dgr(vs):
  """One DeepGlobalRegistration per voxel size (random-init checkpoint), ICP on."""
  if vs not in _DGR:
    from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
    _DGR[vs] = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=vs),
                                                            clip_weight_thresh=0.05, verbose=False))
  return _DGR[vs]


def on(x, side):
  """x as a host array or as a CUDA tensor of the same dtype."""
  return x if side == 'host' else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def run_pair(d, x0, x1, ctx=None, clip=0.05, use_icp=True):
  """-> (result block float64 [64], context) of one dgr_pair_register."""
  from deepglobalregistration_b200 import native
  fcgf, inl = d.native_networks()
  ctx = d.native_context(0) if ctx is None else ctx
  res = native.pair_register(ctx, fcgf, inl, x0, x1, d.voxel_size, clip, use_icp)
  return res, ctx


def taps(ctx):
  return {k: ctx.tap(k).cpu().numpy() for k in ('coords', 'sel', 'xyz', 'features')}


def check_rows(res, ctx, x0, x1, vs):
  """The integer taps against the oracle's voxelisation, and the rows against rows_in_cells on the kept points and
  their keys.  -> (taps, n0, number of coordinates that moved off x.float())."""
  n0, n1 = int(res[40]), int(res[41])
  t = taps(ctx)
  coords, sel, xyz = t['coords'], t['sel'], t['xyz']
  c0, s0 = so.quantize_first(x0, vs)
  c1, s1 = so.quantize_first(x1, vs)
  assert (n0, n1) == (len(s0), len(s1)) and coords.shape == (n0 + n1, 4)
  assert not coords[:n0, 0].any() and (coords[n0:, 0] == 1).all()
  assert np.array_equal(coords[:n0, 1:], c0) and np.array_equal(coords[n0:, 1:], c1)
  assert np.array_equal(sel[:n0], s0) and np.array_equal(sel[n0:], s1 + len(x0))
  xs = np.concatenate([x0[s0].astype(np.float64), x1[s1].astype(np.float64)])
  keys = coords[:, 1:].astype(np.float64)
  assert xyz.tobytes() == rows_in_cells(xs, vs, keys).tobytes()
  x32 = xs.astype(np.float32)
  moved = np.abs(ordered(xyz) - ordered(x32))
  assert moved.max() <= 2, moved.max()
  agree = np.floor(x32.astype(np.float64) / vs) == keys
  assert xyz[agree].tobytes() == x32[agree].tobytes()
  return t, n0, int((moved > 0).sum())


def pair_table(coords):
  """(spec, table) of the pair's rows rebuilt from the tapped coords (distinct rows: table value = row)."""
  from deepglobalregistration_b200 import _abi
  c = torch.from_numpy(coords).cuda().contiguous()
  spec = _abi.keyspec_build(_abi.coords_minmax(c), 4)
  table, _, _, cnt = _abi.unique_first(c, spec)
  assert _abi.read_count(cnt) == len(coords)
  return spec, table


def check_search(t, n0, vs):
  """The executor's search on its own rows (cloud 0 onto cloud 1 through the pair's table at cell = voxel, radius
  2 voxel, from the identity): correspondence count, fitness and RMSE of a zero-iteration ICP, and the information
  matrix - whose sums of target rows pin which rows were chosen - against the brute-force fp64 nearest within the
  radius.  -> the reference's correspondence count."""
  from deepglobalregistration_b200 import _abi
  xyz = t['xyz']
  spec, table = pair_table(t['coords'])
  src, tgt = xyz[:n0], xyz[n0:]
  radius = 2 * vs
  j = opg.nearest_within(src.astype(np.float64), tgt.astype(np.float64), radius)
  m = j >= 0
  n = int(m.sum())
  d2 = ((src[m].astype(np.float64) - tgt[j[m]].astype(np.float64)) ** 2).sum(1)
  dsrc, dxyz = torch.from_numpy(src).cuda(), torch.from_numpy(xyz).cuda()
  res = _abi.icp_point_to_point(dsrc, dxyz, (spec, table), vs, radius, np.eye(4), max_iter=0, batch=1).cpu().numpy()
  assert int(res[19]) == n and res[16] == n / len(src), (res[16:], n)
  rmse = math.sqrt(d2.sum() / n) if n else 0.0
  assert abs(res[17] - rmse) <= 1e-12 * max(rmse, 1e-30), (res[17], rmse)
  info = _abi.information_matrix(dsrc, dxyz, (spec, table), vs, radius, np.eye(4), batch=1).cpu().numpy()
  L, n_o = opg.information_matrix(src, tgt, np.eye(4), radius)
  assert int(info[36]) == n_o == n
  assert np.allclose(info[:36].reshape(6, 6), L, rtol=1e-12, atol=1e-9)
  return n


def inputs(vs):
  """(name, cloud 0, cloud 1) float64: straddling (p, q, s) triples (p in cloud 0; q, s in cloud 1) and pairs of
  boundary-snapped clouds at offsets 0, -100 m and +1000 m."""
  out = []
  t = straddling_pairs(vs, 2)
  if len(t):
    out.append(('triples', t[:, 0].copy(), t[:, 1:].reshape(-1, 3).copy()))
  for k, off in enumerate((0.0, -100.0, 1000.0)):
    out.append((f'snapped {off}', snapped_cloud(10 + k, vs, off), snapped_cloud(20 + k, vs, off)))
  return out


@pytest.mark.parametrize('vs', VOXELS)
def test_executor_rows_agree_with_their_keys(vs):
  """For every input, dtype pair (including both mixed instantiations of the compaction) and input side, the search
  on the executor's rows equals the fp64 reference, the taps equal the oracle's voxelisation, and the rows equal
  rows_in_cells and preprocess()'s rows bit for bit."""
  d = dgr(vs)
  moved = 0
  for name, a, b in inputs(vs):
    for t0, t1 in DTYPES:
      x0, x1 = a.astype(t0), b.astype(t1)
      for side in ('host', 'cuda'):
        res, ctx = run_pair(d, on(x0, side), on(x1, side))
        if side == 'cuda':
          check_search(taps(ctx), int(res[40]), vs)
        t, n0, mv = check_rows(res, ctx, x0, x1, vs)
        moved += mv
        with torch.no_grad():
          p0, _, _ = d.preprocess(on(x0, side), 0, _batch=0)
          p1, _, _ = d.preprocess(on(x1, side), 1, _batch=1)
        assert t['xyz'][:n0].tobytes() == p0.cpu().numpy().tobytes(), (name, t0, t1, side)
        assert t['xyz'][n0:].tobytes() == p1.cpu().numpy().tobytes(), (name, t0, t1, side)
  assert moved > 0            # the inputs do straddle: x.float() alone would put rows in the wrong cells


def snap_to_boundaries(x, cell, frac, seed):
  """A fraction of x's coordinates moved to within 2 float32 ulps (plus a sub-ulp float64 part) of the nearest cell
  boundary."""
  g = np.random.default_rng(seed)
  b = np.round(x / cell) * cell
  ulp = np.spacing(np.abs(b).astype(np.float32) + np.float32(cell)).astype(np.float64)
  snap = b + (g.integers(-2, 3, x.shape) + g.uniform(-0.5, 0.5, x.shape)) * ulp
  return np.where(g.random(x.shape) < frac, snap, x)


def check_icp(icp, T_init, xyz, n0, vs):
  """An ICP result block (pose 16, fitness, RMSE, iterations) against oracle/icp.py on the executor's rows from
  T_init, at test_icp_kernel_vs_oracle's bars.  T_init's rotation is a float32 one widened, orthonormal only to float32
  rounding, which rte_rre's arccos turns into up to ~1e-4 rad between identical poses: the rotation is compared
  entry by entry instead."""
  T_o, info = icp_point_to_point(xyz[:n0], xyz[n0:], 2 * vs, T_init)
  T = icp[:16].reshape(4, 4)
  te = float(np.linalg.norm(T[:3, 3] - T_o[:3, 3]))
  dr = float(np.abs(T[:3, :3] - T_o[:3, :3]).max())
  assert te <= 1e-5 and dr <= 1e-5, (te, dr, icp[16:20], info)
  assert abs(icp[16] - info['fitness']) <= 2e-4 and abs(icp[17] - info['inlier_rmse']) <= 1e-5, (icp[16:20], info)
  assert abs(int(icp[18]) - info['iterations']) <= 1, (icp[18], info)
  assert info['n_corr'] > 0.3 * n0


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_executor_icp_vs_oracle(dtype):
  """The ICP refine from the Procrustes pose in the result block, and the safeguard's ICP (forced by a clip of
  1.0, which zeroes every weight) from its RANSAC pose, against the oracle on the tapped rows of a room pair with
  30 % of its coordinates at cell boundaries."""
  from deepglobalregistration_b200 import native
  vs = 0.05
  d = dgr(vs)
  a, b, _ = syn.room_pair(2, n_raw=20000, extent=(1.8, 1.5, 1.25))
  x0 = snap_to_boundaries(a, vs, 0.3, 1).astype(dtype)
  x1 = snap_to_boundaries(b, vs, 0.3, 2).astype(dtype)
  res, ctx = run_pair(d, x0, x1)
  t, n0, moved = check_rows(res, ctx, x0, x1, vs)
  assert moved > 0
  T12 = np.eye(4)
  T12[:3, :3], T12[:3, 3] = res[:9].reshape(3, 3), res[9:12]
  check_icp(res[17:37], T12, t['xyz'], n0, vs)
  res, ctx = run_pair(d, x0, x1, clip=1.0)
  assert res[16] < max(200, 0.05 * n0)                   # register() would take the safeguard branch
  sg = native.pair_safeguard(ctx, 2 * vs, 200000, 0, True)
  check_icp(sg[20:40], sg[:16].reshape(4, 4), taps(ctx)['xyz'], n0, vs)


# ---------------------------------------------------------------------------------------------------------------------
# non-finite and out-of-range input
# ---------------------------------------------------------------------------------------------------------------------
def nan_cases(vs):
  """(name, cloud) float64 clouds each holding one non-finite coordinate: in a row that would be kept, and behind an
  earlier point of the voxel a conversion sending NaN to 0 would put it in (so that only a check over every raw
  point, not over the kept ones, refuses it)."""
  base = syn.room_scan(5, 400, (0.8, 0.6, 0.5)) + 0.3
  out = []
  for v in (math.nan, math.inf, -math.inf):
    x = base.copy()
    x[37, 1] = v
    out.append((f'{v} kept', x))
  x = base.copy()
  x[5] = [x[5, 0], x[5, 1], 0.5 * vs]                   # cell (cx, cy, 0)
  x[200] = [x[5, 0], x[5, 1], math.nan]                 # cell (cx, cy, NaN): cell 0 without the refusal
  out.append(('nan behind an earlier point', x))
  return out


def test_non_finite_input_is_refused():
  """NaN and +-inf in either cloud, float32 and float64, host arrays and CUDA tensors: register() and
  preprocess() raise DgrError; the context then registers the next pair as a fresh one does."""
  from deepglobalregistration_b200 import _abi
  vs = 0.05
  d = dgr(vs)
  good = syn.room_scan(6, 400, (0.8, 0.6, 0.5)) + 0.3
  for name, bad in nan_cases(vs):
    for dt in (np.float64, np.float32):
      for side in ('host', 'cuda'):
        for pair in ((bad, good), (good, bad)):
          with pytest.raises(_abi.DgrError, match=NOT_FINITE):
            d.register(on(pair[0].astype(dt), side), on(pair[1].astype(dt), side))
        with pytest.raises(_abi.DgrError, match=NOT_FINITE):
          d.preprocess(on(bad.astype(dt), side))
  check_same_as_fresh(d, good, good[::-1] + 0.01)


def test_cells_at_the_key_edges():
  """float64 input at voxel 1.0 - cells INT_MIN + 32 and INT_MAX - 32 (the key margin is 32 cells) are accepted
  by voxelise with their exact cells; one cell beyond either edge is refused."""
  from deepglobalregistration_b200 import _abi
  lo, hi = -2 ** 31 + 32, 2 ** 31 - 1 - 32
  for cell, ok in ((lo, True), (hi, True), (lo - 1, False), (hi + 1, False)):
    x = np.array([[cell + 0.5, 0.25, -3.5], [0.5, 0.5, 0.5]])
    d = torch.from_numpy(x).cuda()
    if ok:
      raw, _, _, sel, _, n = _abi.voxelise(d, 1.0)
      assert n == 2 and raw[:, 1:].cpu().numpy().tolist() == [[cell, 0, -4], [0, 0, 0]]
    else:
      with pytest.raises(_abi.DgrError, match=NOT_FINITE):
        _abi.voxelise(d, 1.0)


def bits(span):
  """Packed bits of a spatial column spanning `span` cells (32 margin cells on either side)."""
  return max(1, math.ceil(math.log2(span + 65)))


def span_of(b):
  """The largest span that packs into b bits."""
  return 2 ** b - 65


def test_3d_key_extent_boundary():
  """_abi.voxelise of two far-apart points (batch 1 bit + spans of 21, 21 and 20 bits = 63) is accepted; one
  more bit is refused."""
  from deepglobalregistration_b200 import _abi
  for b, ok in (((21, 21, 20), True), ((21, 21, 21), False), ((20, 22, 20), True), ((22, 22, 19), False)):
    span = [span_of(k) for k in b]
    assert [bits(s) for s in span] == list(b)
    x = np.array([[0.5, 0.5, 0.5], [span[0] + 0.5, span[1] + 0.5, span[2] + 0.5]]) - 1e6
    d = torch.from_numpy(x).cuda()
    if ok:
      assert _abi.voxelise(d, 1.0)[5] == 2
    else:
      with pytest.raises(_abi.DgrError, match=NOT_FINITE):
        _abi.voxelise(d, 1.0)


def box_cloud(vs, b, seed, n=60):
  """Cloud 0 of the 6-D extent pairs: the 8 corners of a box whose spans pack into bits b, plus n random points."""
  span = np.array([span_of(k) for k in b], np.float64)
  g = np.random.default_rng(seed)
  corners = np.stack(np.meshgrid(*[[0.0, 1.0]] * 3, indexing='ij'), -1).reshape(-1, 3) * span
  pts = np.vstack([corners, np.floor(g.uniform(0.0, 1.0, (n, 3)) * span)])
  return (pts + 0.5) * vs


def check_same_as_fresh(d, x0, x1):
  """The next pair on a context that just refused one equals the same pair on a fresh context: integer taps and rows
  bit for bit, features within 5e-5."""
  from deepglobalregistration_b200 import native
  res, ctx = run_pair(d, x0, x1)
  t = taps(ctx)
  fresh = native.Context(d.device)
  res_f, _ = run_pair(d, x0, x1, ctx=fresh)
  f = taps(fresh)
  fresh.close()
  assert res[40:42].tolist() == res_f[40:42].tolist()
  for k in ('coords', 'sel', 'xyz'):
    assert t[k].tobytes() == f[k].tobytes(), k
  assert np.abs(t['features'] - f['features']).max() <= 5e-5


def test_6d_key_extent_boundary():
  """Cloud 1 is a single voxel, so N1 = 1, every correspondence is row 0 and cloud 1's three 6-D columns take 7
  bits each; with the batch bit, cloud 0's spans may take 41 bits.  Spans of (14, 14, 13) bits register, (14, 14, 14)
  are refused at the 6-D read (the 3-D key of the same pair, 1 + 42 bits, fits), and the context then registers the
  next pair as a fresh one does."""
  from deepglobalregistration_b200 import _abi
  vs = 0.05
  d = dgr(vs)
  one = np.array([[1000.3 * vs, 1000.6 * vs, 100.2 * vs]])          # inside cloud 0's box: the 3-D spans do not grow
  small = syn.room_scan(7, 2000, (0.8, 0.6, 0.5))
  for k, (b, ok) in enumerate((((14, 14, 13), True), ((14, 14, 14), False), ((13, 14, 14), True),
                               ((15, 13, 14), False))):
    x0 = box_cloud(vs, b, k)
    if ok:
      res, ctx = run_pair(d, x0, one)
      assert int(res[40]) == len(x0) and int(res[41]) == 1
      assert int(ctx.tap('idx1').abs().sum()) == 0
    else:
      with pytest.raises(_abi.DgrError, match=EXTENT) as e:
        run_pair(d, x0, one)
      assert 'not finite' not in str(e.value)            # refused at the 6-D read, not at the 3-D one
      check_same_as_fresh(d, small, small[::-1] + 0.013)


# ---------------------------------------------------------------------------------------------------------------------
# shapes and state
# ---------------------------------------------------------------------------------------------------------------------
def test_single_voxel_and_single_point_clouds():
  """N0 = 1, N1 = 1 and both; single-point clouds and clouds whose points all share one voxel."""
  vs = 0.05
  d = dgr(vs)
  one = np.array([[0.31, -0.52, 1.07]])
  cluster = one + np.random.default_rng(0).uniform(0.0, 0.9 * vs, (50, 3)) - (one % vs)      # one voxel
  scan = syn.room_scan(8, 3000, (0.8, 0.6, 0.5))
  for x0, x1 in ((one, scan), (scan, one), (one, one + 0.2), (cluster, scan), (scan, cluster), (cluster, one)):
    for dt in (np.float64, np.float32):
      a, b = x0.astype(dt), x1.astype(dt)
      res, ctx = run_pair(d, a, b)
      check_rows(res, ctx, a, b, vs)


def test_identical_clouds():
  """xyz1 == xyz0: N0 == N1, the batch column keeps the clouds apart, sel1 = sel0 + n_raw0 and the rows are
  equal."""
  vs = 0.05
  d = dgr(vs)
  x = snap_to_boundaries(syn.room_scan(9, 8000, (1.2, 1.0, 0.8)), vs, 0.3, 3)
  for dt in (np.float64, np.float32):
    a = x.astype(dt)
    res, ctx = run_pair(d, a, a.copy())
    t, n0, _ = check_rows(res, ctx, a, a, vs)
    assert int(res[41]) == n0
    assert np.array_equal(t['coords'][n0:, 1:], t['coords'][:n0, 1:])
    assert np.array_equal(t['sel'][n0:], t['sel'][:n0] + len(a))
    assert t['xyz'][n0:].tobytes() == t['xyz'][:n0].tobytes()


def test_arena_reuse_keeps_results():
  """On one context, a 60k-point pair, a tiny pair, then the 60k pair again: the last run's integer taps and rows
  are bit-identical to the first's."""
  vs = 0.05
  d = dgr(vs)
  a, b, _ = syn.room_pair(3, n_raw=60000, extent=(2.4, 2.0, 1.6))
  res1, ctx = run_pair(d, a, b)
  t1 = taps(ctx)
  run_pair(d, a[:5], b[:3], ctx=ctx)
  res3, _ = run_pair(d, a, b, ctx=ctx)
  t3 = taps(ctx)
  assert res1[40:42].tolist() == res3[40:42].tolist()
  for k in ('coords', 'sel', 'xyz'):
    assert t1[k].tobytes() == t3[k].tobytes(), k


# ---------------------------------------------------------------------------------------------------------------------
# the rule's C entry through _abi.float32_in_cells
# ---------------------------------------------------------------------------------------------------------------------
def test_float32_in_cells_moves_only_boundary_rows():
  """_abi.float32_in_cells (dgr_float32_in_cells) over the hash-search test clouds: every row ends in its stored cell,
  a row whose float32 value is already there keeps its bits, no coordinate moves more than CELL_NUDGE_STEPS ulps,
  and every row equals rows_in_cells; keys from float64 (the stand-ins, multiway) and from a float32 division
  (preprocess() of float32 input), given contiguous and as the [:, 1:] view of raw coordinates."""
  from deepglobalregistration_b200 import _abi
  clouds = [(np.array([[-127.9000015258789, 0.0, 0.0], [-127.79999993771924, -0.0, 1e-30]]), 0.05)]
  clouds += [(straddling_pairs(cell, R).reshape(-1, 3), cell) for cell in (0.03, 0.05, 0.07) for R in (1, 2, 3, 6)]
  clouds += [(snapped_cloud(s, cell, off), cell) for s, cell in enumerate((0.05, 0.3, 0.0625, 0.02))
             for off in (0.0, -100.0, 1000.0)]
  moved_rows = 0
  for x64, cell in clouds:
    x32 = x64.astype(np.float32)
    for x, keys in ((x64, np.floor(x64 / cell)), (x32, np.floor(x32 / np.float32(cell)).astype(np.float64))):
      k32 = torch.from_numpy(keys.astype(np.int32)).cuda()
      raw = torch.cat([torch.zeros_like(k32[:, :1]), k32], 1)
      for cells in (k32, raw[:, 1:]):
        y = _abi.float32_in_cells(torch.from_numpy(x).cuda(), cells, cell)
        assert y.dtype == torch.float32 and y.is_contiguous() and y.is_cuda
        y = y.cpu().numpy()
        assert np.array_equal(np.floor(y.astype(np.float64) / cell), keys)
        agree = np.floor(x32.astype(np.float64) / cell) == keys
        assert y[agree].tobytes() == x32[agree].tobytes()
        assert np.abs(ordered(y) - ordered(x32)).max() <= _abi.CELL_NUDGE_STEPS
        assert y.tobytes() == rows_in_cells(x.astype(np.float64), cell, keys).tobytes()
      moved_rows += int((~agree).any(1).sum())
  assert moved_rows > 1000
