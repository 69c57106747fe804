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
``.points``, ``.normals``, ``.colors`` (what colored ICP registers), ``.transform(T)`` and ``estimate_normals``.  With no argument
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
  """Points [N, 3] float64, optional colours [N, 3] float64 in [0, 1], plus optional per-point attributes read
  alongside them."""

  def __init__(self, points=None, attributes=None, **more_attributes):
    self.points = np.zeros((0, 3)) if points is None else points
    # per-point extras as ONE dict (a PLY property may be called anything, 'points' included)
    self.attributes = dict(attributes or {}, **more_attributes)
    self.normals = None
    self.colors = None
    self.covariances = None

  @property
  def points(self):
    return self._points

  @points.setter
  def points(self, value):
    value = np.asarray(value, dtype=np.float64)
    if value.ndim != 2 or value.shape[1] != 3:
      raise ValueError(f'points must be [N, 3], got {value.shape}')
    self._points = np.ascontiguousarray(value)

  @property
  def colors(self):
    return self._colors

  @colors.setter
  def colors(self, value):
    if value is not None:
      value = np.asarray(value, dtype=np.float64)
      if value.ndim != 2 or value.shape[1] != 3:
        raise ValueError(f'colors must be [N, 3], got {value.shape}')
      value = np.ascontiguousarray(value)
    self._colors = value

  def has_colors(self):
    """open3d's rule: one colour per point of a non-empty cloud."""
    return self._colors is not None and len(self._colors) == len(self._points) > 0

  @property
  def covariances(self):
    return self._covariances

  @covariances.setter
  def covariances(self, value):
    if value is not None:
      value = np.asarray(value, dtype=np.float64)
      if value.ndim != 3 or value.shape[1:] != (3, 3):
        raise ValueError(f'covariances must be [N, 3, 3], got {value.shape}')
      value = np.ascontiguousarray(value)
    self._covariances = value

  def has_covariances(self):
    """open3d's rule: one covariance per point of a non-empty cloud."""
    return self._covariances is not None and len(self._covariances) == len(self._points) > 0

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
    if self._covariances is not None:
      R = T[:3, :3]
      self._covariances = np.ascontiguousarray(np.einsum('ab,nbc,dc->nad', R, self._covariances, R))
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

  def estimate_covariances(self, search_param=None):
    """``estimate_covariances(KDTreeSearchParamHybrid(radius, max_nn))`` computes per-point covariances on the GPU
    (o3d_registration.estimate_covariances; max_nn <= 64) into ``covariances`` (float64 [N, 3, 3]).  Without an
    argument it raises NotImplementedError: open3d's default there is KDTreeSearchParamKNN(30), an unbounded search
    the voxel-hash kernel cannot do."""
    if search_param is None:
      raise NotImplementedError('estimate_covariances() defaults to KDTreeSearchParamKNN(30), which is not built: pass '
                                'KDTreeSearchParamHybrid(radius, max_nn)')
    from .o3d_registration import estimate_covariances
    self.covariances = estimate_covariances(self._points, search_param)
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
  return _read_ply(path)[:2]


def _read_ply(path):
  """read_ply plus {vertex property name: its PLY type}."""
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
      return pts, extra, {p[2]: p[1] for p in el['props']}
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


def _ply_colors(extra, types):
  """Colours [N, 3] in [0, 1] from PLY red / green / blue (uchar divided by 255, floating point kept), else None."""
  names = ('red', 'green', 'blue')
  if not all(n in extra for n in names):
    return None
  kinds = {np.dtype(_PLY_TYPES[types[n]]).kind for n in names}
  rgb = np.stack([np.asarray(extra[n], np.float64) for n in names], axis=1)
  if kinds == {'f'}:
    return rgb
  if {types[n] for n in names} <= {'uchar', 'uint8'}:
    return rgb / 255.0
  return None                                           # other integer widths: left in attributes only


def read_point_cloud(path):
  """``o3d.io.read_point_cloud`` for the formats above -> PointCloud (points as float64, which is
  what open3d holds and why the reference voxelises PLY input in float64).  PLY red / green / blue also fill
  ``colors`` (and stay in ``attributes``); a mesh PLY reads as its coloured vertices."""
  if os.path.splitext(path)[1].lower() == '.ply':
    pts, extra, types = _read_ply(path)
    pcd = PointCloud(pts, attributes=extra)
    pcd.colors = _ply_colors(extra, types)
    return pcd
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


# ------------------------------------------------------------------------------------------
# PNG (3DMatch raw RGB-D frames) and triangle meshes (fragments fused from them)
# ------------------------------------------------------------------------------------------
_PNG_SIG = b'\x89PNG\r\n\x1a\n'
_PNG_KINDS = {(8, 2): (np.dtype('u1'), 3), (16, 0): (np.dtype('>u2'), 1)}   # (bit depth, colour type) -> (dtype, C)


def _png_paeth_row(line, prev, bpp):
  out, prev = bytearray(line), bytes(prev)
  for i in range(len(out)):
    a = out[i - bpp] if i >= bpp else 0
    b = prev[i]
    c = prev[i - bpp] if i >= bpp else 0
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    out[i] = (out[i] + (a if pa <= pb and pa <= pc else b if pb <= pc else c)) & 0xFF
  return np.frombuffer(bytes(out), np.uint8)


def _png_average_row(line, prev, bpp):
  out, prev = bytearray(line), bytes(prev)
  for i in range(len(out)):
    a = out[i - bpp] if i >= bpp else 0
    out[i] = (out[i] + ((a + prev[i]) >> 1)) & 0xFF
  return np.frombuffer(bytes(out), np.uint8)


def read_png(path):
  """A non-interlaced 8-bit RGB ([H, W, 3] uint8) or 16-bit greyscale ([H, W] uint16) PNG, the two kinds 3DMatch's
  raw colour and depth frames use; filters 0-4.  Anything else, a bad CRC or truncated data raises ValueError."""
  import zlib
  with open(path, 'rb') as fh:
    buf = fh.read()
  if buf[:8] != _PNG_SIG:
    raise ValueError(f'{path}: not a PNG file')
  pos, ihdr, idat, ended = 8, None, [], False
  while pos + 12 <= len(buf):
    n = int.from_bytes(buf[pos:pos + 4], 'big')
    kind, data = buf[pos + 4:pos + 8], buf[pos + 8:pos + 8 + n]
    if len(data) != n or pos + 12 + n > len(buf):
      raise ValueError(f'{path}: truncated {kind!r} chunk')
    if zlib.crc32(kind + data) != int.from_bytes(buf[pos + 8 + n:pos + 12 + n], 'big'):
      raise ValueError(f'{path}: CRC mismatch in {kind!r} chunk')
    pos += 12 + n
    if kind == b'IHDR':
      if n != 13:
        raise ValueError(f'{path}: bad IHDR')
      ihdr = data
    elif kind == b'IDAT':
      idat.append(data)
    elif kind == b'IEND':
      ended = True
      break
  if ihdr is None or not ended:
    raise ValueError(f'{path}: missing IHDR or IEND')
  W, H = int.from_bytes(ihdr[0:4], 'big'), int.from_bytes(ihdr[4:8], 'big')
  depth, ctype, comp, filt, interlace = ihdr[8], ihdr[9], ihdr[10], ihdr[11], ihdr[12]
  if (depth, ctype) not in _PNG_KINDS:
    raise ValueError(f'{path}: unsupported PNG kind (bit depth {depth}, colour type {ctype}); '
                     'only 8-bit RGB and 16-bit greyscale are read')
  if comp != 0 or filt != 0 or interlace != 0 or W == 0 or H == 0:
    raise ValueError(f'{path}: unsupported PNG (compression {comp}, filter method {filt}, interlace {interlace})')
  dt, ch = _PNG_KINDS[(depth, ctype)]
  bpp = ch * dt.itemsize
  stride = W * bpp
  try:
    raw = zlib.decompress(b''.join(idat))
  except zlib.error as e:
    raise ValueError(f'{path}: corrupt image data ({e})') from None
  if len(raw) != H * (stride + 1):
    raise ValueError(f'{path}: image data has {len(raw)} bytes, expected {H * (stride + 1)}')
  rows = np.frombuffer(raw, np.uint8).reshape(H, stride + 1)
  out = np.zeros((H, stride), np.uint8)
  prev = np.zeros(stride, np.uint8)
  for r in range(H):
    f, line = rows[r, 0], rows[r, 1:]
    if f == 0:
      cur = line
    elif f == 1:
      cur = (np.cumsum(line.reshape(W, bpp), axis=0, dtype=np.uint64) & 0xFF).astype(np.uint8).reshape(-1)
    elif f == 2:
      cur = line + prev
    elif f == 3:
      cur = _png_average_row(line, prev, bpp)
    elif f == 4:
      cur = _png_paeth_row(line, prev, bpp)
    else:
      raise ValueError(f'{path}: bad filter type {f} on row {r}')
    out[r] = cur
    prev = out[r]
  img = out.view(dt).reshape(H, W, ch) if ch > 1 else out.view(dt).reshape(H, W)
  return img.astype(dt.newbyteorder('='))


def write_png(path, img, filter_type=1):
  """Write [H, W, 3] uint8 as 8-bit RGB or [H, W] uint16 as 16-bit greyscale; every row uses `filter_type` (0-4)."""
  import zlib
  img = np.asarray(img)
  if img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3:
    depth, ctype, data = 8, 2, img
  elif img.dtype == np.uint16 and img.ndim == 2:
    depth, ctype, data = 16, 0, img.astype('>u2')
  else:
    raise ValueError(f'write_png takes [H, W, 3] uint8 or [H, W] uint16, got {img.dtype} {img.shape}')
  if filter_type not in range(5):
    raise ValueError(f'filter_type must be 0..4, got {filter_type}')
  H, W = img.shape[:2]
  bpp = data.dtype.itemsize * (3 if ctype == 2 else 1)
  x = np.ascontiguousarray(data).view(np.uint8).reshape(H, W * bpp).astype(np.int32)
  a = np.zeros_like(x)
  a[:, bpp:] = x[:, :-bpp]
  b = np.zeros_like(x)
  b[1:] = x[:-1]
  c = np.zeros_like(x)
  c[1:, bpp:] = x[:-1, :-bpp]
  if filter_type == 0:
    pred = np.zeros_like(x)
  elif filter_type == 1:
    pred = a
  elif filter_type == 2:
    pred = b
  elif filter_type == 3:
    pred = (a + b) >> 1
  else:
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
  rows = np.empty((H, W * bpp + 1), np.uint8)
  rows[:, 0] = filter_type
  rows[:, 1:] = ((x - pred) & 0xFF).astype(np.uint8)

  def chunk(kind, payload):
    return len(payload).to_bytes(4, 'big') + kind + payload + zlib.crc32(kind + payload).to_bytes(4, 'big')
  ihdr = W.to_bytes(4, 'big') + H.to_bytes(4, 'big') + bytes([depth, ctype, 0, 0, 0])
  with open(path, 'wb') as fh:
    fh.write(_PNG_SIG + chunk(b'IHDR', ihdr) + chunk(b'IDAT', zlib.compress(rows.tobytes(), 6)) + chunk(b'IEND', b''))


class Image:
  """``open3d.geometry.Image``: an [H, W] or [H, W, C] array; ``np.asarray(img)`` returns it."""

  def __init__(self, data=None):
    self.data = np.ascontiguousarray(np.zeros((0, 0), np.uint8) if data is None else np.asarray(data))

  def __array__(self, dtype=None, copy=None):
    return self.data if dtype is None else self.data.astype(dtype)

  @property
  def width(self):
    return self.data.shape[1]

  @property
  def height(self):
    return self.data.shape[0]

  def get_min_bound(self):
    return np.zeros(2)

  def get_max_bound(self):
    """(width, height), as open3d returns it (util/integration.py:92)."""
    return np.array([self.data.shape[1], self.data.shape[0]], dtype=np.float64)

  def is_empty(self):
    return self.data.size == 0

  def __repr__(self):
    return f'Image of size {self.width}x{self.height}, with {1 if self.data.ndim == 2 else self.data.shape[2]} channels.'


def read_image(path):
  """``o3d.io.read_image`` for PNG -> Image."""
  return Image(read_png(path))


class TriangleMesh:
  """``open3d.geometry.TriangleMesh``: vertices [N, 3] float64, triangles [M, 3] int32, vertex_colors [N, 3] in
  [0, 1] (empty when the mesh has none)."""

  def __init__(self, vertices=None, triangles=None, vertex_colors=None):
    self.vertices = np.zeros((0, 3)) if vertices is None else np.asarray(vertices, np.float64).reshape(-1, 3)
    self.triangles = (np.zeros((0, 3), np.int32) if triangles is None
                      else np.asarray(triangles, np.int32).reshape(-1, 3))
    self.vertex_colors = (np.zeros((0, 3)) if vertex_colors is None
                          else np.asarray(vertex_colors, np.float64).reshape(-1, 3))

  def has_vertex_colors(self):
    return len(self.vertex_colors) > 0 and len(self.vertex_colors) == len(self.vertices)

  def is_empty(self):
    return len(self.vertices) == 0

  def __repr__(self):
    return f'TriangleMesh with {len(self.vertices)} points and {len(self.triangles)} triangles.'


def write_triangle_mesh(path, mesh, **kwargs):
  """Binary little-endian PLY: the vertex element first (float x y z, uchar red green blue when the mesh has
  colours, round(255 c) clipped), then ``face`` with ``list uchar int vertex_indices``.  read_point_cloud of the file
  returns the vertices.  -> True (open3d's return)."""
  V = np.asarray(mesh.vertices, np.float64).reshape(-1, 3)
  T = np.asarray(mesh.triangles, np.int64).reshape(-1, 3)
  cols = np.asarray(getattr(mesh, 'vertex_colors', np.zeros((0, 3))), np.float64).reshape(-1, 3)
  has_c = len(cols) == len(V) and len(V) > 0
  if len(T) and (T.min() < 0 or T.max() >= len(V)):
    raise ValueError('triangle index out of range')
  fields = [('x', '<f4'), ('y', '<f4'), ('z', '<f4')]
  if has_c:
    fields += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1')]
  rec = np.empty(len(V), dtype=fields)
  for k, a in zip('xyz', V.T):
    rec[k] = a
  if has_c:
    c8 = np.clip(np.round(cols * 255.0), 0, 255).astype(np.uint8)
    for k, n in enumerate(('red', 'green', 'blue')):
      rec[n] = c8[:, k]
  face = np.empty(len(T), dtype=[('n', 'u1'), ('v', '<i4', (3,))])
  face['n'] = 3
  face['v'] = T
  head = ['ply', 'format binary_little_endian 1.0', 'comment dgr-b200', f'element vertex {len(V)}',
          'property float x', 'property float y', 'property float z']
  if has_c:
    head += ['property uchar red', 'property uchar green', 'property uchar blue']
  head += [f'element face {len(T)}', 'property list uchar int vertex_indices', 'end_header']
  with open(path, 'wb') as fh:
    fh.write(('\n'.join(head) + '\n').encode('ascii'))
    fh.write(rec.tobytes())
    fh.write(face.tobytes())
  return True
