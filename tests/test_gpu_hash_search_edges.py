"""The voxel-hash searches (normals, colour gradients, FPFH, ICP, the information matrix) against fp64 references
evaluated on exactly the float32 rows the kernels read, at the edges where a hash search goes wrong: rows within
rounding of a cell boundary, neighbours at the radius +- 1 ulp, radius / cell ratios that round below an integer,
probe blocks with every live cell occupied, d^2 ties split by max_nn, and small or awkward shapes.

Every search assumes that a row stored under key k has floor(double(xyz32[row]) / cell) == k.  Tables keyed in float64
(the open3d stand-ins, multiway) or by a float32 division (preprocess() of float32 input) hold rows whose float32 value
lies across a boundary; _abi.float32_in_cells moves those rows back into their cells.  `rows_in_cells` below restates
it in numpy."""
import math
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import colored_icp as oc
from oracle import normals as onm
from oracle import pose_graph as opg
from test_gpu_colored_icp import PIVOT_EXCLUDE
from test_gpu_fpfh import check_parity
from test_gpu_icp_plane import _t, check_normals

pytestmark = pytest.mark.gpu

F32_UP, F32_DOWN = np.float32(np.inf), np.float32(-np.inf)


def rows_in_cells(x64, cell, keys=None):
  """float32 rows of x64 [n, 3] in the cells `keys` (default floor(x64 / cell)): each coordinate whose float32 value's
  cell differs is moved toward its cell one ulp at a time."""
  x64 = np.asarray(x64, np.float64).reshape(-1, 3)
  k = np.floor(x64 / cell) if keys is None else np.asarray(keys, np.float64)
  x32 = x64.astype(np.float32)
  for _ in range(8):
    c = np.floor(x32.astype(np.float64) / cell)
    x32 = np.where(c < k, np.nextafter(x32, F32_UP), np.where(c > k, np.nextafter(x32, F32_DOWN), x32))
  assert np.array_equal(np.floor(x32.astype(np.float64) / cell), k)
  return x32


def first_per_cell(x64, cell):
  """The first row of every cell floor(x64 / cell) (in float64, as the stand-ins key), rows in input order."""
  _, first = np.unique(np.floor(x64 / cell).astype(np.int64), axis=0, return_index=True)
  return x64[np.sort(first)]


def table(x64, cell):
  """(spec, table, rows) of the float64 cloud's own hash at `cell` (every row kept) and the float32 rows the searches
  read, from _abi.float32_in_cells; the rows are checked against rows_in_cells."""
  from deepglobalregistration_b200 import _abi
  d = _t(x64, torch.float64)
  raw, spec, tab, _, _, n = _abi.voxelise(d, cell)
  assert n == len(x64)
  rows = _abi.float32_in_cells(d, raw[:, 1:], cell)
  assert rows.dtype == torch.float32 and rows.is_contiguous()
  r = rows.cpu().numpy()
  assert r.tobytes() == rows_in_cells(x64, cell).tobytes()
  return spec, tab, rows, r.astype(np.float64)


def radius_of(R, cell):
  """The largest radius near R cells with ceil(radius / cell) == R (R * cell itself can round above R)."""
  r = R * cell
  while math.ceil(r / cell) > R:
    r = float(np.nextafter(r, 0.0))
  return r


def straddling_pairs(cell, R, lo=-4000, hi=4000, gap=None):
  """[m, 3, 3] triples (p, q, s) on the x axis, radius R cells.  p: the largest float32 of cell c.  q: the smallest
  float64 of cell c + R + 1, whose float32 rounding falls into cell c + R and within the radius of p (so a search from
  p's cell misses q's float32 row when it is keyed at q's float64 cell).  s: the smallest float32 at least the radius
  above float32(q) and less than the radius above q's row moved back into its cell (so s matches q only there).
  Triples are at least `gap` cells apart."""
  radius = radius_of(R, cell)
  r2 = radius * radius
  out, last = [], -10 ** 9
  gap = 2 * R + 6 if gap is None else gap
  for c in range(lo, hi):
    if c - last < gap:
      continue
    q = (c + R + 1) * cell
    while math.floor(q / cell) < c + R + 1:
      q = float(np.nextafter(q, np.inf))
    while math.floor(float(np.nextafter(q, -np.inf)) / cell) == c + R + 1:
      q = float(np.nextafter(q, -np.inf))
    q32 = float(np.float32(q))
    if math.floor(q32 / cell) != c + R:
      continue
    p = float(np.float32((c + 1) * cell))
    while math.floor(p / cell) > c:
      p = float(np.nextafter(np.float32(p), F32_DOWN))
    if not (q32 - p) ** 2 < r2:
      continue
    q_in = float(np.nextafter(np.float32(q32), F32_UP))
    s = float(np.float32(q32 + radius))
    while (s - q32) ** 2 < r2:
      s = float(np.nextafter(np.float32(s), F32_UP))
    while (float(np.nextafter(np.float32(s), F32_DOWN)) - q32) ** 2 >= r2:
      s = float(np.nextafter(np.float32(s), F32_DOWN))
    if not (s - q_in) ** 2 < r2:
      continue
    out.append([[p, 0.0, 0.0], [q, 0.0, 0.0], [s, 0.0, 0.0]])
    last = c
  return np.asarray(out, np.float64).reshape(-1, 3, 3)


def test_the_constructed_pair_is_what_it_claims():
  """cell 0.05, radius 2 cells: p = -127.9000015258789 (exact in float32, cell -2559) and q = -127.79999993771924
  (cell -2556, float32 -127.80000305175781 in cell -2557, 0.0999985 from p)."""
  cell, p, q = 0.05, -127.9000015258789, -127.79999993771924
  assert float(np.float32(p)) == p and math.floor(p / cell) == -2559 and math.floor(q / cell) == -2556
  q32 = float(np.float32(q))
  assert q32 == -127.80000305175781 and math.floor(q32 / cell) == -2557 and (q32 - p) ** 2 < 0.01
  t = straddling_pairs(cell, 2, -2560, -2558, gap=1)       # the same p, and q's cell's smallest float64
  assert len(t) == 1 and t[0, 0, 0] == p and math.floor(t[0, 1, 0] / cell) == -2556 and np.float32(t[0, 1, 0]) == q32


def self_search(x64, cell, radius, max_nn, batch=0, hashed=None):
  """Counts (normals, gradients, FPFH) and normals through the float64-keyed table, checked against the reference on
  the rows the kernels read."""
  from deepglobalregistration_b200 import _abi
  spec, tab, rows, r = hashed or table(x64, cell)
  want = onm.neighbours(r, radius, max_nn)[1]
  reach = math.ceil(radius / cell)
  if reach <= 4:
    nn = min(max_nn, _abi.MAX_NN)
    nrm, cnt = _abi.estimate_normals(rows, (spec, tab), cell, radius, nn, return_counts=True, batch=batch)
    assert np.array_equal(cnt.cpu().numpy(), want)
    check_normals(nrm.cpu().numpy().astype(np.float64), cnt.cpu().numpy(), r, radius, nn)
    inten = np.random.default_rng(len(r)).random(len(r))
    grad, gcnt = _abi.color_gradient(rows, nrm, _t(inten, torch.float32), (spec, tab), cell, radius, nn,
                                     return_counts=True, batch=batch)
    assert np.array_equal(gcnt.cpu().numpy(), want)
    g = grad.cpu().numpy()
    g_o, _, pivot = oc.color_gradient(r, nrm.cpu().numpy(), inten.astype(np.float32), radius, nn)
    ok, zero = pivot > PIVOT_EXCLUDE, np.minimum(want, nn) < 4
    assert not g[zero].any()
    err = np.linalg.norm(g - g_o.astype(np.float32), axis=1) / np.maximum(np.linalg.norm(g_o, axis=1), 1e-3)
    assert np.all(err[ok] <= 1e-9 + 2.0 ** -23), np.sort(err[ok])[-5:]
  nrm = _t(np.tile([[0.0, 0.0, 1.0]], (len(r), 1)), torch.float32)
  _, fcnt = _abi.compute_fpfh(rows, nrm, (spec, tab), cell, radius, min(max_nn, 128), return_counts=True, batch=batch)
  assert np.array_equal(fcnt.cpu().numpy(), onm.neighbours(r, radius, min(max_nn, 128))[1])
  return want


def nearest_counts(src32, tgt_rows, max_dist):
  j = opg.nearest_within(np.asarray(src32, np.float64), np.asarray(tgt_rows, np.float64), max_dist)
  return int((j >= 0).sum())


@pytest.mark.parametrize('cell', [0.03, 0.07])
@pytest.mark.parametrize('R', [1, 2, 3, 4, 5, 6])
def test_straddling_pairs_through_the_abi(R, cell):
  """Generated (p, q, s) triples in one cloud, searched through the float64-keyed table at radius R cells."""
  from deepglobalregistration_b200 import _abi
  radius = radius_of(R, cell)
  t = straddling_pairs(cell, R)
  assert len(t) >= 3, len(t)
  x64 = t.reshape(-1, 3)
  hashed = table(x64, cell)
  spec, tab, rows, r = hashed
  moved = r[:, 0] != x64.astype(np.float32)[:, 0]
  assert moved[1::3].all() and not moved[0::3].any() and not moved[2::3].any()   # only q moves, by one ulp
  self_search(x64, cell, radius, 64, hashed=hashed)
  if R > 4:
    return
  spec, tab, rows, r = table(t[:, 1], cell)            # the q rows alone are the target
  src = np.concatenate([t[:, 0], t[:, 2]]).astype(np.float32)
  want = nearest_counts(src, r, radius)
  assert want == len(t)                       # every s matches its q, no p does
  for fn in (_abi.icp_point_to_point, lambda *a, **k: _abi.icp_point_to_plane(a[0], a[1], torch.ones_like(a[1]),
                                                                               *a[2:], **k)):
    res = fn(_t(src, torch.float32), rows, (spec, tab), cell, radius, np.eye(4), max_iter=0).cpu().numpy()
    assert int(res[19]) == want and res[16] == want / len(src), res[16:]
  info = _abi.information_matrix(_t(src, torch.float32), rows, (spec, tab), cell, radius, np.eye(4)).cpu().numpy()
  L, n = opg.information_matrix(src, r, np.eye(4), radius)
  assert int(info[36]) == n == want and np.allclose(info[:36].reshape(6, 6), L, rtol=1e-12, atol=1e-9)


def test_straddling_pairs_through_the_stand_ins():
  """registration_icp (point-to-point and point-to-plane), the information matrix and FPFH of the open3d stand-ins on
  float64 clouds of (p, q, s) triples at the stand-ins' radius of 2 cells: every correspondence of s is found, none of
  p, and FPFH rows agree with the reference on the rows the search reads."""
  from deepglobalregistration_b200 import o3d_registration as reg
  cell = 0.05
  t = straddling_pairs(cell, 2)
  src, tgt = np.concatenate([t[:, 0], t[:, 2]]), t[:, 1]
  rows = rows_in_cells(tgt, cell).astype(np.float64)
  want = nearest_counts(src.astype(np.float32), rows, 2 * cell)
  assert want == len(t)
  crit = reg.ICPConvergenceCriteria(max_iteration=0)
  r = reg.registration_icp(src, tgt, 2 * cell, criteria=crit)
  assert len(r.correspondence_set) == want and r.fitness == want / len(src), r
  pl = types.SimpleNamespace(points=tgt, normals=np.tile([[1.0, 0.0, 0.0]], (len(tgt), 1)))
  r = reg.registration_icp(src, pl, 2 * cell, estimation_method=reg.TransformationEstimationPointToPlane(),
                           criteria=crit)
  assert len(r.correspondence_set) == want, r
  L = reg.get_information_matrix_from_point_clouds(src, tgt, 2 * cell, np.eye(4))
  assert L[5, 5] == want
  # FPFH of the whole cloud (radius 2 cells: the stand-in's cell is radius / 2): rows match the reference's
  x64 = t.reshape(-1, 3)
  nrm = np.tile([[0.0, 0.6, 0.8]], (len(x64), 1))
  f = reg.compute_fpfh_feature(types.SimpleNamespace(points=x64, normals=nrm),
                               reg.KDTreeSearchParamHybrid(radius=2 * cell, max_nn=30)).data.T
  _, f_rows = check_parity('straddling triples', rows_in_cells(x64, cell).astype(np.float64), cell, 2 * cell, 30,
                           nrm=_t(nrm, torch.float32))
  assert f.astype(np.float32).tobytes() == f_rows.tobytes()
  # a point with no neighbour but itself has an all-zero feature: only s and q see each other
  assert not f[0::3].any() and f[1::3].any() and f[2::3].any()


def snapped_cloud(seed, cell, offset, side=10, ulps=2):
  """One float64 point per cell of a side^3 block at `offset`, most coordinates within `ulps` float32 ulps (plus a
  sub-ulp float64 part) of a cell boundary."""
  g = np.random.default_rng(seed)
  c = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing='ij'), -1).reshape(-1, 3) + np.floor(offset / cell)
  c = c[g.permutation(len(c))[:int(0.7 * len(c))]]
  x = (c + g.uniform(0.0, 1.0, c.shape)) * cell
  b = c * cell
  ulp = np.spacing(np.abs(b).astype(np.float32) + np.float32(cell)).astype(np.float64)
  snap = b + (g.integers(-ulps, ulps + 1, c.shape) + g.uniform(-0.5, 0.5, c.shape)) * ulp
  x = np.where(g.random(c.shape) < 0.8, snap, x)
  return first_per_cell(x, cell)


@pytest.mark.parametrize('offset', [0.0, -100.0, 1000.0])
@pytest.mark.parametrize('R', [2, 3, 4, 6])
def test_boundary_snapped_clouds(offset, R):
  from deepglobalregistration_b200 import _abi
  cell = 0.05
  radius = radius_of(R, cell)
  x64 = snapped_cloud(R, cell, offset)
  hashed = table(x64, cell)
  spec, tab, rows, r = hashed
  assert (r != x64.astype(np.float32)).any()            # some rows moved back into their cells
  self_search(x64, cell, radius, 64 if R <= 4 else 128, hashed=hashed)
  if R <= 4:
    src = (x64 + np.random.default_rng(1).normal(0.0, cell, x64.shape)).astype(np.float32)
    res = _abi.icp_point_to_point(_t(src, torch.float32), rows, (spec, tab), cell, radius, np.eye(4),
                                  max_iter=0).cpu().numpy()
    assert int(res[19]) == nearest_counts(src, r, radius)


def test_snapped_clouds_through_the_stand_ins():
  from deepglobalregistration_b200 import o3d_registration as reg
  cell = 0.05
  for offset in (0.0, -100.0, 1000.0):
    tgt = snapped_cloud(7, cell, offset)
    src = tgt + np.random.default_rng(2).normal(0.0, cell, tgt.shape)
    r = reg.registration_icp(src, tgt, 2 * cell, criteria=reg.ICPConvergenceCriteria(max_iteration=0))
    want = nearest_counts(src.astype(np.float32), rows_in_cells(tgt, cell), 2 * cell)
    assert len(r.correspondence_set) == want, (offset, r, want)


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_pipeline_tables(dtype):
  """preprocess() keys in the input dtype (a float32 division for float32 input) and returns the rows the ICP refine
  and the baselines search that table with: on batch 1, the normals counts and the refine's correspondences agree with
  the reference on exactly those rows."""
  from deepglobalregistration_b200 import _abi
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  vs = 0.05
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=vs),
                                                   clip_weight_thresh=0.05, verbose=False))
  t = straddling_pairs(vs, 2)
  x1 = np.vstack([t.reshape(-1, 3), snapped_cloud(3, vs, -100.0)]).astype(dtype)
  if dtype == np.float32:                               # one row per cell of the float32 keys
    _, first = np.unique(np.floor(x1 / np.float32(vs)).astype(np.int64), axis=0, return_index=True)
    x1 = x1[np.sort(first)]
  with torch.no_grad():
    p1, c1, _ = d.preprocess(x1, 1, _batch=1)
  r1 = p1.cpu().numpy()
  assert len(r1) == len(x1)
  assert np.array_equal(np.floor(r1.astype(np.float64) / vs), c1[:, 1:].cpu().numpy())
  moved = np.abs(r1.view(np.int32).astype(np.int64) - x1.astype(np.float32).view(np.int32))
  assert moved.max() <= _abi.CELL_NUDGE_STEPS and moved.any()
  _, cnt = _abi.estimate_normals(p1, c1._dgr_manager, vs, 2 * vs, 30, return_counts=True, batch=1)
  assert np.array_equal(cnt.cpu().numpy(), onm.neighbours(r1.astype(np.float64), 2 * vs, 30)[1])
  # the refine's search: the p and s rows onto the q rows
  with torch.no_grad():
    p0, _, _ = d.preprocess(np.concatenate([t[:, 0], t[:, 2]]).astype(dtype), 0, _batch=0)
    p2, c2, _ = d.preprocess(t[:, 1].astype(dtype), 1, _batch=1)
  res = _abi.icp_point_to_point(p0, p2, c2._dgr_manager, vs, 2 * vs, np.eye(4), max_iter=0, batch=1).cpu().numpy()
  want = nearest_counts(p0.cpu().numpy(), p2.cpu().numpy(), 2 * vs)
  assert int(res[19]) == want and res[16] == want / len(p0)
  if dtype == np.float64:
    assert want == len(t)


def test_multiway_rows_agree_with_their_table():
  from deepglobalregistration_b200.core.multiway import MultiwayRegistration
  vs = 0.05
  m = MultiwayRegistration('dgr', voxel_size=vs)
  t = straddling_pairs(vs, 2)
  x = t[:, 1]                                           # the q rows
  from deepglobalregistration_b200 import _abi
  _abi.refresh_stream()
  rows, (spec, tab), n = m._voxelised(x, torch.device('cuda'))
  assert n == len(x) and rows.cpu().numpy().tobytes() == rows_in_cells(x, vs).tobytes()
  src = np.concatenate([t[:, 0], t[:, 2]]).astype(np.float32)
  info = _abi.information_matrix(_t(src, torch.float32), rows, (spec, tab), vs, m.info_radius, np.eye(4)).cpu().numpy()
  assert int(info[36]) == nearest_counts(src, rows.cpu().numpy(), m.info_radius) == len(t)


# ---------------------------------------------------------------------------------------------------------------------
# radius edges (float32-exact clouds: the rows are the clouds)
# ---------------------------------------------------------------------------------------------------------------------
def f32(x):
  return np.asarray(x, np.float32).astype(np.float64)


def shell_cloud(centre, radius, dirs, k):
  """centre plus one point along every direction at the radius, each of its nonzero coordinates then moved k float32
  ulps outward (k > 0) or inward (k < 0); one point per cell."""
  pts = [centre]
  for d in dirs:
    d = np.asarray(d, np.float64) / np.linalg.norm(d)
    q = np.asarray(centre + radius * d, np.float32)
    for a in range(3):
      if d[a] != 0.0:
        for _ in range(abs(k)):
          q[a] = np.nextafter(q[a], F32_UP if (k > 0) == (d[a] > 0) else F32_DOWN)
    pts.append(q.astype(np.float64))
  return np.asarray(pts)


AXES = [[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]]
DIAG = [[1, 1, 0], [-1, 1, -1], [1, -1, 1], [0, -1, -1], [-1, 0, 1], [1, 1, 1], [-1, -1, -1], [1, 0, -1]]


@pytest.mark.parametrize('cell,ratio', [(0.0625, 2.0), (0.0625, 3.0), (0.0625, 4.0), (0.05, 2.0), (0.05, 3.0),
                                        (0.05, 2.5), (0.05, 6.0), (0.3, 1.5)])
def test_neighbours_at_the_radius(cell, ratio):
  """Points at the radius - 2 .. + 2 ulps along the axes and diagonals: inside below, outside above, and at the
  radius itself as the float64 d^2 of the float32 rows decides."""
  radius = radius_of(ratio, cell) if ratio == int(ratio) else ratio * cell
  centre = f32([5.37 * cell, -2.39 * cell, 11.5 * cell])
  first = {}
  for k in (-2, -1, 0, 1, 2):
    P = first_per_cell(shell_cloud(centre, radius, AXES + DIAG, k), cell)
    first[k] = (self_search(P, cell, radius, 128 if ratio > 4 else 64)[0], len(P))
  assert first[-2][0] == first[-2][1] and first[2][0] == 1, first


def f32_in_cell(k, cell, top):
  """The largest (top) or smallest float32 x with floor(x / cell) == k."""
  x = np.float32((k + 1) * cell if top else k * cell)
  while math.floor(float(x) / cell) > k:
    x = np.nextafter(x, F32_DOWN)
  while math.floor(float(x) / cell) < k:
    x = np.nextafter(x, F32_UP)
  step = F32_UP if top else F32_DOWN
  while math.floor(float(np.nextafter(x, step)) / cell) == k:
    x = np.nextafter(x, step)
  return float(x)


def test_a_ratio_just_below_an_integer_keeps_its_corner_cells():
  """cell 0.05, radius 0.15: radius / cell = 2.9999999999999996 and radius^2 / cell^2 = 8.999999999999998, so the
  gap-9 cells such as (3, 3, 2) are live only through the 1e-6 margin; points sit at the corners of those cells
  nearest the query, beside gap-6 and gap-8 cells that hold in-radius points."""
  cell, radius = 0.05, 0.15
  assert radius / cell < 3.0 and radius * radius / (cell * cell) < 9.0 and math.ceil(radius / cell) == 3
  c = [f32_in_cell(0, cell, True)] * 3                      # the +++ corner of cell (0, 0, 0)
  pts = [c]
  for off in [(3, 3, 2), (3, 2, 3), (2, 3, 3), (3, 3, 1), (3, 2, 2), (2, 3, 2), (-3, 2, 2), (2, -3, -2), (-2, -2, -3)]:
    pts.append([f32_in_cell(o, cell, o < 0) for o in off])
  want = self_search(np.asarray(pts), cell, radius, 64)
  assert want[0] >= 4, want


@pytest.mark.parametrize('reach,max_nn', [(2, 1), (2, 64), (3, 64), (4, 1), (4, 64), (5, 128), (6, 1), (6, 128)])
def test_full_probe_blocks(reach, max_nn):
  """Every cell of a (2 reach + 3)^3 block occupied near its centre: the central points' lists hold every live
  cell's key, and max_nn cuts through them."""
  cell = 0.0625
  side = 2 * reach + 3
  c = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing='ij'), -1).reshape(-1, 3)
  g = np.random.default_rng(reach * 1000 + max_nn)
  P = f32((c + 0.5 + g.uniform(-0.02, 0.02, c.shape)) * cell - 7.0)
  radius = (reach - 0.01) * cell
  counts = self_search(P, cell, radius, max_nn)
  if reach >= 3 or max_nn == 1:
    assert counts.max() > max_nn


@pytest.mark.parametrize('max_nn', [1, 6, 7, 19, 64, 128])
def test_d2_ties_split_by_max_nn(max_nn):
  """A lattice at an exact binary spacing with rows permuted: the 6, 12, 8 neighbours at d^2 = 1, 2, 3 spacings tie
  exactly, and the row order decides which of a tied group max_nn keeps."""
  cell = 0.125
  side = 7
  c = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing='ij'), -1).reshape(-1, 3)
  P = (c[np.random.default_rng(max_nn).permutation(len(c))] - 3) * cell - 2.0
  radius = 2.5 * cell
  self_search(P, cell, radius, max_nn)
  o = check_parity(f'lattice ties max_nn {max_nn}', P, cell, radius, min(max_nn, 128))[0]
  assert o['counts'].max() > min(max_nn, 30)


@pytest.mark.parametrize('n', [1, 2, 5, 31, 33, 129, 1001])
def test_shapes(n):
  """n = 1, n not a multiple of 4 warps or 8 lanes, negative coordinates and an isolated point far from the rest."""
  from deepglobalregistration_b200 import _abi
  cell = 0.05
  g = np.random.default_rng(n)
  P = first_per_cell(f32(g.uniform(-0.6, -0.1, (n, 3))), cell)
  if n > 2:
    P[-1] = [-40.0, 25.0, -13.0]                    # isolated, far from the rest
  for reach, max_nn in ((2, 30), (4, 64), (6, 128)):
    counts = self_search(P, cell, radius_of(reach, cell), max_nn)
    assert n <= 2 or counts[-1] == 1
