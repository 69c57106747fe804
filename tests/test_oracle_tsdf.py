"""oracle/tsdf.py on its own (CPU): the marching-cubes tables, the mesh's structure, its accuracy against the analytic
room, the first-occurrence touch order and the no-op frame."""
from collections import Counter

import numpy as np
import pytest

from deepglobalregistration_b200 import synthetic as syn
from oracle import tsdf as ot

VL, TRUNC = 0.02, 0.06
W, H = 160, 120
# Vertices of the small sequence below lie within this distance of the analytic box faces (measured 7.6 mm away from
# box edges, 48 mm at the worst corner; 2 cm voxels, 1 mm depth quantisation).
FACE_BOUND_AWAY = 0.012


@pytest.fixture(scope='module')
def small_mesh():
  c, d, P, K = syn.rgbd_sequence(0, 6, W, H)
  ov = ot.Volume(VL, TRUNC, color=True)
  for k in range(len(P)):
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (W, H) + K, np.linalg.inv(P[k]), c[k])
  return ov, ov.extract_triangle_mesh()


def _edge_counts(T):
  e = Counter()
  for a, b, c in T.tolist():
    for x, y in ((a, b), (b, c), (c, a)):
      e[(min(x, y), max(x, y))] += 1
  return e


def test_tables():
  assert ot.TRI_TABLE.shape == (256, 16)
  assert ot.EDGE_TABLE[1] == 0x109 and ot.EDGE_TABLE[255] == 0 and ot.EDGE_TABLE[0] == 0
  for i in range(256):
    row = ot.TRI_TABLE[i][ot.TRI_TABLE[i] >= 0]
    assert len(row) % 3 == 0
    # a configuration's triangles use exactly its sign-changing edges
    assert set(row.tolist()) == {e for e in range(12) if (ot.EDGE_TABLE[i] >> e) & 1}, i
    assert ot.TRI_COUNT[i] == len(row) // 3


def test_mesh_structure(small_mesh):
  ov, (V, C, T) = small_mesh
  assert len(T) > 1000 and len(V) == len(C)
  assert T.min() >= 0 and T.max() < len(V)
  assert all(len(set(t)) == 3 for t in T.tolist())
  # every vertex has exactly one off-lattice coordinate: lattice points sit at (g + 0.5) voxel_length
  frac = np.abs(V / VL - 0.5 - np.round(V / VL - 0.5))
  off = (frac > 1e-9).sum(axis=1)
  assert (off <= 1).all()
  assert (off == 1).mean() > 0.95          # the rest lie exactly on an endpoint (|f0| == 0)
  assert max(_edge_counts(T).values()) <= 2
  assert ((C >= 0) & (C <= 1)).all()


def test_mesh_accuracy(small_mesh):
  _, (V, _, _) = small_mesh
  face, edge = syn.box_face_distance(V, syn.room_boxes(0))
  away = face[edge > 0.1]
  print(f'\n[oracle tsdf] face distance away from edges: p99 {np.percentile(away, 99) * 1e3:.2f} mm, '
        f'max {away.max() * 1e3:.2f} mm')
  assert away.max() <= FACE_BOUND_AWAY


def test_sphere_is_closed():
  # a smooth, fully observed field: the signed distance to a sphere, written straight into the slabs
  ov = ot.Volume(0.01, 0.05)
  R = ot.RES
  for u in [(x, y, z) for x in (-1, 0) for y in (-1, 0) for z in (-1, 0)]:
    ov.slot[u] = len(ov.keys)
    ov.keys = np.concatenate([ov.keys, np.array([u], np.int64)])
  loc = np.stack(np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing='ij'), -1).reshape(-1, 3)
  p = (ov.keys[:, None, :] * R + loc[None] + 0.5) * 0.01
  ov.tsdf = (np.linalg.norm(p, axis=2) - 0.093).astype(np.float32) / np.float32(0.05)
  ov.weight = np.ones_like(ov.tsdf)
  ov.rgb = np.zeros((len(ov.keys), 3, R ** 3), np.float32)
  V, C, T = ov.extract_triangle_mesh()
  assert C is None and len(T) > 500
  counts = _edge_counts(T)
  assert set(counts.values()) == {2}
  assert np.abs(np.linalg.norm(V, axis=1) - 0.093).max() < 0.002
  # outward winding: the normal of (v0, v1, v2) points away from the centre
  n = np.cross(V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]])
  assert (np.einsum('ij,ij->i', n, V[T].mean(axis=1)) > 0).all()


def test_touch_order_is_first_occurrence():
  c, d, P, K = syn.rgbd_sequence(1, 2, W, H)
  depth = ot.depth_from_raw(d[0], 1000.0, 4.5)
  pose = P[0]
  units = ot.touched_units(depth, (W, H) + K, pose, VL, TRUNC)
  # restate the rule with plain loops
  L = VL * ot.RES
  fx, fy, cx, cy = K
  seen, order = set(), []
  for i in range(0, H, 4):
    for j in range(0, W, 4):
      dd = float(depth[i, j])
      if dd <= 0:
        continue
      x, y = ((j - cx) * dd) / fx, ((i - cy) * dd) / fy
      p = [((pose[r, 0] * x + pose[r, 1] * y) + pose[r, 2] * dd) + pose[r, 3] for r in range(3)]
      lo = [int(np.floor((q - TRUNC) / L)) for q in p]
      hi = [int(np.floor((q + TRUNC) / L)) for q in p]
      for ux in range(lo[0], hi[0] + 1):
        for uy in range(lo[1], hi[1] + 1):
          for uz in range(lo[2], hi[2] + 1):
            if (ux, uy, uz) not in seen:
              seen.add((ux, uy, uz))
              order.append((ux, uy, uz))
  assert [tuple(u) for u in units.tolist()] == order
  ov = ot.Volume(VL, TRUNC)
  ov.integrate(depth, (W, H) + K, np.linalg.inv(pose))
  assert [tuple(u) for u in ov.keys.tolist()] == order
  assert ov.last_touched.tolist() == list(range(len(order)))
  # a second frame: known units keep their slots, new ones follow in first-touch order
  d2 = ot.depth_from_raw(d[1], 1000.0, 4.5)
  u2 = [tuple(u) for u in ot.touched_units(d2, (W, H) + K, P[1], VL, TRUNC).tolist()]
  ov.integrate(d2, (W, H) + K, np.linalg.inv(P[1]))
  new = [u for u in u2 if u not in set(order)]
  assert [tuple(u) for u in ov.keys.tolist()] == order + new
  assert ov.last_touched.tolist() == [ov.slot[u] for u in u2]


def test_zero_depth_changes_nothing():
  c, d, P, K = syn.rgbd_sequence(2, 1, W, H)
  ov = ot.Volume(VL, TRUNC, color=True)
  ov.integrate(ot.depth_from_raw(d[0], 1000.0, 4.5), (W, H) + K, np.linalg.inv(P[0]), c[0])
  before = (ov.keys.copy(), ov.tsdf.copy(), ov.weight.copy(), ov.rgb.copy())
  ov.integrate(np.zeros((H, W), np.float32), (W, H) + K, np.linalg.inv(P[0]), c[0])
  assert len(ov.last_touched) == 0
  for a, b in zip(before, (ov.keys, ov.tsdf, ov.weight, ov.rgb)):
    assert np.array_equal(a, b)
  fresh = ot.Volume(VL, TRUNC)
  fresh.integrate(np.zeros((H, W), np.float32), (W, H) + K, np.eye(4))
  V, C, T = fresh.extract_triangle_mesh()
  assert len(fresh.keys) == 0 and V.shape == (0, 3) and T.shape == (0, 3)


def test_argument_errors():
  with pytest.raises(ValueError):
    ot.Volume(VL, TRUNC, res=8)
  ov = ot.Volume(VL, TRUNC, color=True)
  with pytest.raises(ValueError):
    ov.integrate(np.zeros((H, W), np.float32), (W + 1, H, 100.0, 100.0, 80.0, 60.0), np.eye(4),
                 np.zeros((H, W, 3), np.uint8))
  with pytest.raises(ValueError):
    ov.integrate(np.zeros((H, W), np.float32), (W, H, 100.0, 100.0, 80.0, 60.0), np.eye(4),
                 np.zeros((H, W), np.float32))


def test_library_tables_equal_the_oracle():
  from deepglobalregistration_b200 import _abi
  edge, tri = _abi.tsdf_mc_tables()               # host copy: no device needed
  assert np.array_equal(edge, ot.EDGE_TABLE)
  assert np.array_equal(tri, ot.TRI_TABLE)
