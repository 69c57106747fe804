"""Readers for the on-disk formats either side of register() (SURVEY.md §8f rank 4) - host-side
numpy only, nothing here touches the GPU path:

* PLY point clouds (what ``o3d.io.read_point_cloud`` reads for demo.py:34-37): ascii,
  binary_little_endian and binary_big_endian, any scalar vertex properties, x/y/z picked by name;
* KITTI velodyne ``.bin``: float32 x, y, z, reflectance (dataloader/kitti_loader.py:132-136);
* 3DMatch fragments ``.npz`` with a ``pcd`` array (dataloader/threedmatch_loader.py:51-54);
* ``.npy`` / whitespace text ``.xyz`` / ``.txt`` / ``.pts`` arrays of [N, >=3];
* ``gt.log`` trajectory files: a line of integer metadata followed by a 4x4 matrix
  (util/file.py:69-90).

``PointCloud`` is the small part of ``open3d.geometry.PointCloud`` the reference's demo and
``DeepGlobalRegistration.preprocess`` (core/deep_global_registration.py:143-148) rely on:
``.points``, ``.normals``, ``.transform(T)`` and ``estimate_normals``.  With no argument
``estimate_normals()`` does nothing (demo.py calls it for display only); with
``KDTreeSearchParamHybrid(radius, max_nn)`` (util/pointcloud.py:60) it computes the normals on the GPU -
the one call here that leaves the host, through a lazy import of o3d_registration.
"""
import os
import re

import numpy as np

_PLY_TYPES = {
    'char': 'i1', 'int8': 'i1', 'uchar': 'u1', 'uint8': 'u1', 'short': 'i2', 'int16': 'i2',
    'ushort': 'u2', 'uint16': 'u2', 'int': 'i4', 'int32': 'i4', 'uint': 'u4', 'uint32': 'u4',
    'float': 'f4', 'float32': 'f4', 'double': 'f8', 'float64': 'f8',
}


class PointCloud:
  """Points [N, 3] float64 plus optional per-point attributes read alongside them."""

  def __init__(self, points=None, attributes=None, **more_attributes):
    self.points = np.zeros((0, 3)) if points is None else points
    # per-point extras as ONE dict (a PLY property may be called anything, 'points' included)
    self.attributes = dict(attributes or {}, **more_attributes)
    self.normals = None

  @property
  def points(self):
    return self._points

  @points.setter
  def points(self, value):
    value = np.asarray(value, dtype=np.float64)
    if value.ndim != 2 or value.shape[1] != 3:
      raise ValueError(f'points must be [N, 3], got {value.shape}')
    self._points = np.ascontiguousarray(value)

  def __len__(self):
    return len(self._points)

  def has_points(self):
    return len(self._points) > 0

  def transform(self, T):
    T = np.asarray(T, dtype=np.float64)
    if T.shape != (4, 4):
      raise ValueError('transform expects a 4x4 matrix')
    self._points = self._points @ T[:3, :3].T + T[:3, 3]
    if self.normals is not None:
      self.normals = np.asarray(self.normals, dtype=np.float64) @ T[:3, :3].T
    return self

  def has_normals(self):
    return self.normals is not None

  def estimate_normals(self, search_param=None, fast_normal_computation=True):
    """``estimate_normals()`` is a no-op (demo.py:35,37 calls it for display; open3d's default there is
    KDTreeSearchParamKNN(30), an unbounded search the voxel-hash kernel cannot do).
    ``estimate_normals(KDTreeSearchParamHybrid(radius, max_nn))`` computes the normals on the GPU
    (o3d_registration.estimate_normals; max_nn <= 64) into ``normals`` (float64 [N, 3]); existing normals orient
    the new ones, as in open3d.  KDTreeSearchParamKNN / KDTreeSearchParamRadius raise NotImplementedError."""
    if search_param is None:
      return self
    from .o3d_registration import estimate_normals
    self.normals = estimate_normals(self._points, search_param, prev=self.normals)
    return self

  def __repr__(self):
    return f'PointCloud with {len(self)} points.'


# ------------------------------------------------------------------------------------------
# PLY
# ------------------------------------------------------------------------------------------
def _ply_header(fh):
  if fh.readline().strip() != b'ply':
    raise ValueError('not a PLY file')
  fmt, elements = None, []
  while True:
    raw = fh.readline()
    if not raw:
      raise ValueError('PLY header without end_header')
    tok = raw.decode('ascii', 'replace').split()
    if not tok or tok[0] in ('comment', 'obj_info'):
      continue
    if tok[0] == 'format':
      fmt = tok[1]
    elif tok[0] == 'element':
      elements.append(dict(name=tok[1], count=int(tok[2]), props=[]))
    elif tok[0] == 'property':
      if not elements:
        raise ValueError('PLY property before any element')
      if tok[1] == 'list':
        elements[-1]['props'].append(('list', tok[2], tok[3], tok[4]))
      else:
        if tok[1] not in _PLY_TYPES:
          raise ValueError(f'unknown PLY type {tok[1]}')
        elements[-1]['props'].append(('scalar', tok[1], tok[2]))
    elif tok[0] == 'end_header':
      break
  if fmt not in ('ascii', 'binary_little_endian', 'binary_big_endian'):
    raise ValueError(f'unsupported PLY format {fmt}')
  return fmt, elements


def _skip_binary_element(fh, el, order):
  if all(p[0] == 'scalar' for p in el['props']):
    fh.seek(el['count'] * sum(np.dtype(_PLY_TYPES[p[1]]).itemsize for p in el['props']), os.SEEK_CUR)
    return
  for _ in range(el['count']):        # list properties: row sizes vary
    for p in el['props']:
      if p[0] == 'scalar':
        fh.seek(np.dtype(_PLY_TYPES[p[1]]).itemsize, os.SEEK_CUR)
      else:
        cnt_t, val_t = np.dtype(order + _PLY_TYPES[p[1]]), np.dtype(_PLY_TYPES[p[2]])
        n = int(np.frombuffer(fh.read(cnt_t.itemsize), dtype=cnt_t)[0])
        fh.seek(n * val_t.itemsize, os.SEEK_CUR)


def read_ply(path):
  """-> (points float64 [N, 3], {other scalar vertex properties: array [N]})."""
  with open(path, 'rb') as fh:
    fmt, elements = _ply_header(fh)
    order = {'ascii': '=', 'binary_little_endian': '<', 'binary_big_endian': '>'}[fmt]
    for el in elements:
      if el['name'] != 'vertex':
        if fmt == 'ascii':
          for _ in range(el['count']):
            fh.readline()
        else:
          _skip_binary_element(fh, el, order)
        continue
      if any(p[0] == 'list' for p in el['props']):
        raise ValueError('list properties on the vertex element are not supported')
      names = [p[2] for p in el['props']]
      if not all(a in names for a in 'xyz'):
        raise ValueError('PLY vertex element lacks x / y / z')
      if fmt == 'ascii':
        rows = [fh.readline().split() for _ in range(el['count'])]
        if any(len(r) < len(names) for r in rows):
          raise ValueError('truncated PLY vertex data')
        table = np.array([r[:len(names)] for r in rows], dtype=np.float64).reshape(el['count'], len(names))
        cols = {n: table[:, k] for k, n in enumerate(names)}
      else:
        dt = np.dtype([(p[2], order + _PLY_TYPES[p[1]]) for p in el['props']])
        buf = fh.read(dt.itemsize * el['count'])
        if len(buf) != dt.itemsize * el['count']:
          raise ValueError('truncated PLY vertex data')
        rec = np.frombuffer(buf, dtype=dt)
        cols = {n: rec[n] for n in names}
      pts = np.stack([np.asarray(cols[a], dtype=np.float64) for a in 'xyz'], axis=1)
      extra = {n: np.asarray(v) for n, v in cols.items() if n not in ('x', 'y', 'z')}
      return pts, extra
  raise ValueError('PLY file has no vertex element')


def write_ply(path, points, fmt='binary_little_endian', dtype='float', **props):
  """Minimal writer (tests, exporting registered clouds): x y z as `dtype` plus uchar / float extras."""
  points = np.asarray(points)
  tname = {'float': 'f4', 'double': 'f8'}[dtype]
  order = {'ascii': '=', 'binary_little_endian': '<', 'binary_big_endian': '>'}[fmt]
  fields = [('x', tname), ('y', tname), ('z', tname)]
  fields += [(k, 'u1' if np.asarray(v).dtype.kind in 'ui' else 'f4') for k, v in props.items()]
  rec = np.empty(len(points), dtype=[(n, order + t) for n, t in fields])
  for k, a in zip('xyz', points.T):
    rec[k] = a
  for k, v in props.items():
    rec[k] = v
  back = {'f4': 'float', 'f8': 'double', 'u1': 'uchar'}
  head = ['ply', f'format {fmt} 1.0', 'comment dgr-b200', f'element vertex {len(points)}']
  head += [f'property {back[t]} {n}' for n, t in fields] + ['end_header']
  with open(path, 'wb') as fh:
    fh.write(('\n'.join(head) + '\n').encode('ascii'))
    if fmt == 'ascii':
      for row in rec:
        fh.write((' '.join(repr(float(x)) if isinstance(x, (float, np.floating)) else str(int(x))
                           for x in row.tolist()) + '\n').encode('ascii'))
    else:
      fh.write(rec.tobytes())


# ------------------------------------------------------------------------------------------
# other point formats
# ------------------------------------------------------------------------------------------
def read_kitti_bin(path):
  """-> (xyz float32 [N, 3], reflectance float32 [N]); float32 stays float32 so that voxelisation
  divides in the caller's dtype exactly as the reference does for KITTI (scripts/test_kitti.py:76-80)."""
  raw = np.fromfile(path, dtype=np.float32)
  if raw.size % 4:
    raise ValueError(f'{path}: size is not a multiple of 4 float32 values')
  raw = raw.reshape(-1, 4)
  return np.ascontiguousarray(raw[:, :3]), np.ascontiguousarray(raw[:, 3])


def read_points(path):
  """Any supported file -> ndarray [N, 3] (float32 for KITTI .bin, the stored dtype for .npz /
  .npy, float64 otherwise)."""
  ext = os.path.splitext(path)[1].lower()
  if ext == '.ply':
    return read_ply(path)[0]
  if ext == '.bin':
    return read_kitti_bin(path)[0]
  if ext == '.npz':
    with np.load(path) as data:
      if 'pcd' not in data:
        raise ValueError(f"{path}: no 'pcd' array (3DMatch fragment layout)")
      pts = np.asarray(data['pcd'])
  elif ext == '.npy':
    pts = np.load(path)
  elif ext in ('.xyz', '.txt', '.pts', '.csv'):
    pts = np.loadtxt(path, delimiter=',' if ext == '.csv' else None, ndmin=2)
  else:
    raise ValueError(f'unsupported point-cloud file type {ext!r}')
  if pts.ndim != 2 or pts.shape[1] < 3:
    raise ValueError(f'{path}: expected [N, >=3] points, got {pts.shape}')
  return np.ascontiguousarray(pts[:, :3])


def read_point_cloud(path):
  """``o3d.io.read_point_cloud`` for the formats above -> PointCloud (points as float64, which is
  what open3d holds and why the reference voxelises PLY input in float64)."""
  if os.path.splitext(path)[1].lower() == '.ply':
    pts, extra = read_ply(path)
    return PointCloud(pts, attributes=extra)
  return PointCloud(read_points(path))


# ------------------------------------------------------------------------------------------
# trajectories (gt.log)
# ------------------------------------------------------------------------------------------
class CameraPose:
  def __init__(self, metadata, pose):
    self.metadata = list(metadata)
    self.pose = pose

  def __repr__(self):
    return f'CameraPose(metadata={self.metadata}, pose=\n{self.pose})'


def read_trajectory(filename, dim=4):
  """util/file.py:69-90: [CameraPose(metadata ints, dim x dim float64 pose)]."""
  poses = []
  with open(filename, 'r') as fh:
    lines = [ln for ln in fh.read().splitlines() if ln.strip()]
  if len(lines) % (dim + 1):
    raise ValueError(f'{filename}: {len(lines)} non-empty lines is not a multiple of {dim + 1}')
  for k in range(0, len(lines), dim + 1):
    meta = [int(x) for x in lines[k].split()]
    mat = np.array([[float(x) for x in re.split(r'[ \t]+', ln.strip())] for ln in lines[k + 1:k + 1 + dim]])
    if mat.shape != (dim, dim):
      raise ValueError(f'{filename}: pose block {k // (dim + 1)} is not {dim}x{dim}')
    poses.append(CameraPose(meta, mat))
  return poses


def write_trajectory(filename, poses):
  """poses: iterable of CameraPose or (metadata, 4x4)."""
  with open(filename, 'w') as fh:
    for p in poses:
      meta, mat = (p.metadata, p.pose) if isinstance(p, CameraPose) else p
      fh.write(' '.join(str(int(m)) for m in meta) + '\n')
      for row in np.asarray(mat, dtype=np.float64):
        fh.write(' '.join(f'{x:.17g}' for x in row) + '\n')
