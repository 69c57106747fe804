"""open3d's RGB-D integration objects, backed by libdgr_b200 (csrc/tsdf.cu): ``pipelines.integration`` (``integration``
before 0.12) ScalableTSDFVolume / TSDFVolumeColorType, ``camera.PinholeCameraIntrinsic`` and ``geometry.Image`` /
``RGBDImage`` / ``TriangleMesh`` - what util/integration.py:13-105 calls to fuse 3DMatch RGB-D frames into fragments.

The volume's arithmetic is oracle/tsdf.py's, bit for bit; its mesh comes in a canonical order (vertices by unit slot,
voxel, axis; triangles by unit slot, voxel, table order) where open3d's follows its hash map.
"""
import numpy as np
import torch

from . import _abi
from .io import Image, TriangleMesh  # noqa: F401  (open3d.geometry's names)


class TSDFVolumeColorType:
  NoColor = 0
  RGB8 = 1
  Gray32 = 2


class PinholeCameraIntrinsic:
  def __init__(self, width=-1, height=-1, fx=0.0, fy=0.0, cx=0.0, cy=0.0):
    self.width, self.height = int(width), int(height)
    self.intrinsic_matrix = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=np.float64)

  def set_intrinsics(self, width, height, fx, fy, cx, cy):
    self.__init__(width, height, fx, fy, cx, cy)

  def get_focal_length(self):
    return float(self.intrinsic_matrix[0, 0]), float(self.intrinsic_matrix[1, 1])

  def get_principal_point(self):
    return float(self.intrinsic_matrix[0, 2]), float(self.intrinsic_matrix[1, 2])

  def _params(self):
    K = self.intrinsic_matrix
    return np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], dtype=np.float64)

  def __repr__(self):
    return f'PinholeCameraIntrinsic with width = {self.width} and height = {self.height}.'


def _raycast_max_steps(W, H, intr, pose, voxel_length, depth_max):
  """dgr_tsdf_raycast's step bound, ceil(((2 s_max) depth_max) / voxel_length) + 1: s = |R (a, b, 1)| is the ray's
  world length per unit of t, convex in (a, b), so its largest value s_max is at a corner pixel."""
  fx, fy, cx, cy = intr
  s_max = 0.0
  for c in range(4):
    a = (float(W - 1 if c & 1 else 0) - cx) / fx
    b = (float(H - 1 if c & 2 else 0) - cy) / fy
    d = [(pose[r, 0] * a + pose[r, 1] * b) + pose[r, 2] for r in range(3)]
    s = float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
    s_max = s if s > s_max else s_max
  return float(np.ceil(((2.0 * s_max) * depth_max) / voxel_length) + 1.0)


class RGBDImage:
  def __init__(self, color=None, depth=None):
    self.color = color if color is not None else Image()
    self.depth = depth if depth is not None else Image()

  @staticmethod
  def create_from_color_and_depth(color, depth, depth_scale=1000.0, depth_trunc=3.0, convert_rgb_to_intensity=True):
    """Depth in metres: float32(raw) / float32(depth_scale), 0 where >= depth_trunc.  Colour stays as given, or
    becomes float32 intensity (0.299 R + 0.587 G + 0.114 B) / 255 with convert_rgb_to_intensity."""
    raw = np.asarray(depth)
    if raw.ndim != 2:
      raise ValueError(f'depth image must have one channel, got shape {raw.shape}')
    d = raw.astype(np.float32) / np.float32(depth_scale)
    d[d >= np.float32(depth_trunc)] = 0
    c = np.asarray(color)
    if convert_rgb_to_intensity and c.ndim == 3:
      cf = c.astype(np.float32)
      c = ((cf[..., 0] * np.float32(0.299) + cf[..., 1] * np.float32(0.587) + cf[..., 2] * np.float32(0.114))
           / np.float32(255.0)).astype(np.float32)
    if c.shape[:2] != d.shape:
      raise ValueError(f'colour {c.shape[:2]} and depth {d.shape} sizes differ')
    return RGBDImage(Image(c), Image(d))


class ScalableTSDFVolume:
  """A sparse TSDF volume of 16^3-voxel units on the GPU.  It owns its device tensors: the unit table (rebuilt
  larger before a frame could take its load past 1/2), the unit keys in slot order and the tsdf / weight / colour
  slabs, grown by reallocation and copy."""

  def __init__(self, voxel_length, sdf_trunc, color_type=TSDFVolumeColorType.NoColor, volume_unit_resolution=16,
               depth_sampling_stride=4, device='cuda'):
    if not voxel_length > 0:
      raise ValueError(f'voxel_length must be positive, got {voxel_length}')
    if not sdf_trunc > 0:
      raise ValueError(f'sdf_trunc must be positive, got {sdf_trunc}')
    if volume_unit_resolution != _abi.TSDF_RES:
      raise ValueError(f'volume_unit_resolution must be {_abi.TSDF_RES}, got {volume_unit_resolution}')
    if int(depth_sampling_stride) != depth_sampling_stride or depth_sampling_stride < 1:
      raise ValueError(f'depth_sampling_stride must be an integer >= 1, got {depth_sampling_stride}')
    if color_type == TSDFVolumeColorType.Gray32:
      raise NotImplementedError('Gray32 colour is not supported (NoColor and RGB8 are)')
    if color_type not in (TSDFVolumeColorType.NoColor, TSDFVolumeColorType.RGB8):
      raise ValueError(f'unknown color_type {color_type}')
    self.voxel_length, self.sdf_trunc = float(voxel_length), float(sdf_trunc)
    self.color_type = color_type
    self.volume_unit_resolution = int(volume_unit_resolution)
    self.depth_sampling_stride = int(depth_sampling_stride)
    self.device = _abi.require_device(device)
    self.reset()

  @property
  def _color(self):
    return self.color_type == TSDFVolumeColorType.RGB8

  def reset(self):
    dev = self.device
    self.n_units = 0
    self.n_touched = 0
    self._keys = torch.empty(0, dtype=torch.int64, device=dev)
    self._vals = torch.empty(0, dtype=torch.int32, device=dev)
    self._unit_keys = torch.empty(0, 3, dtype=torch.int32, device=dev)
    self._tsdf = torch.zeros(0, 4096, dtype=torch.float32, device=dev)
    self._weight = torch.zeros(0, 4096, dtype=torch.float32, device=dev)
    self._rgb = torch.zeros(0, 3, 4096, dtype=torch.float32, device=dev) if self._color else None
    self._touched = torch.empty(0, dtype=torch.int32, device=dev)

  def _reserve(self, n_cand):
    need = self.n_units + n_cand
    if self._unit_keys.shape[0] < need:
      uk = torch.empty(max(need, 2 * self._unit_keys.shape[0]), 3, dtype=torch.int32, device=self.device)
      uk[:self.n_units] = self._unit_keys[:self.n_units]
      self._unit_keys = uk
    if self._keys.numel() < 2 * need:
      cap = _abi.table_cap(need)
      self._keys = torch.empty(cap, dtype=torch.int64, device=self.device)
      self._vals = torch.empty(cap, dtype=torch.int32, device=self.device)
      _abi.tsdf_rehash(self._unit_keys, self.n_units, self._keys, self._vals)

  def _grow_slabs(self, n):
    cap = self._tsdf.shape[0]
    if n <= cap:
      return
    new = max(n, 2 * cap)
    for name in ('_tsdf', '_weight', '_rgb'):
      old = getattr(self, name)
      if old is None:
        continue
      t = torch.zeros((new,) + tuple(old.shape[1:]), dtype=old.dtype, device=self.device)
      t[:cap] = old
      setattr(self, name, t)

  def integrate(self, image, intrinsic, extrinsic):
    """Fuse one RGBDImage seen by `intrinsic` from `extrinsic` (4x4 world to camera).  One host read."""
    depth = np.asarray(image.depth)
    W, H = intrinsic.width, intrinsic.height
    if depth.dtype != np.float32 or depth.shape != (H, W):
      raise ValueError(f'depth must be float32 [{H}, {W}] (the intrinsic\'s size), got {depth.dtype} {depth.shape}')
    color = None
    if self._color:
      color = np.asarray(image.color)
      if color.dtype != np.uint8 or color.shape != (H, W, 3):
        raise ValueError('an RGB8 volume needs 3-channel uint8 colour of the depth\'s size '
                         f'(convert_rgb_to_intensity=False), got {color.dtype} {color.shape}')
    ext = np.asarray(extrinsic, dtype=np.float64)
    if ext.shape != (4, 4) or not np.isfinite(ext).all():
      raise ValueError(f'extrinsic must be a finite 4x4 matrix, got shape {ext.shape}')
    intr = intrinsic._params()
    if not (intr[0] > 0 and intr[1] > 0):
      raise ValueError('focal lengths must be positive')
    pose = np.linalg.inv(ext)
    n_cand, words = _abi.tsdf_touch_ws(W, H, self.depth_sampling_stride, self.voxel_length, self.sdf_trunc)
    _abi.refresh_stream()
    self._reserve(n_cand)
    if self._touched.numel() < n_cand:
      self._touched = torch.empty(n_cand, dtype=torch.int32, device=self.device)
    dev = self.device
    d_dev = torch.from_numpy(np.ascontiguousarray(depth)).to(dev)
    c_dev = torch.from_numpy(np.ascontiguousarray(color)).to(dev) if color is not None else None
    ws = _abi.scratch('tsdf_touch', words, torch.int64, dev)
    counts = torch.empty(3, dtype=torch.int32, device=dev)
    _abi.tsdf_touch(d_dev, intr, pose, self.voxel_length, self.sdf_trunc, self.depth_sampling_stride, self._keys,
                    self._vals, self._unit_keys, self.n_units, self._touched, counts, ws)
    n_touched, n_units, bad = (int(v) for v in counts.cpu())
    self.n_units, self.n_touched = n_units, n_touched
    if bad:
      raise ValueError('a touched unit lies outside the volume\'s coordinate range '
                       f'(|unit| <= 2^20 units of {16 * self.voxel_length} m); the frame was not integrated')
    if n_touched == 0:                                 # no depth: nothing to integrate
      return
    self._grow_slabs(n_units)
    _abi.tsdf_integrate(d_dev, c_dev, intr, ext, self.voxel_length, self.sdf_trunc, self._unit_keys, self._touched,
                        n_touched, self._tsdf, self._weight, self._rgb)

  def extract_triangle_mesh(self):
    """Marching cubes over every unit -> TriangleMesh (vertex colours in [0, 1] for RGB8)."""
    _abi.refresh_stream()
    self._grow_slabs(self.n_units)
    v, c, t = self.extract_triangle_mesh_tensors()
    return TriangleMesh(v.cpu().numpy(), t.cpu().numpy(), None if c is None else c.cpu().numpy())

  def extract_triangle_mesh_tensors(self):
    """-> (vertices [nv, 3] f64, colours [nv, 3] f64 or None, triangles [nt, 3] int32) on the device."""
    return _abi.tsdf_extract(self._unit_keys, self.n_units, self._keys if self._keys.numel() else
                             torch.full((1,), -1, dtype=torch.int64, device=self.device), self._vals if
                             self._vals.numel() else torch.zeros(1, dtype=torch.int32, device=self.device),
                             self._tsdf, self._weight, self._rgb, self.voxel_length)

  def raycast(self, intrinsic, extrinsic, depth_min=0.1, depth_max=3.0, weight_threshold=3.0,
              convert_rgb_to_intensity=True):
    """Render the volume seen by `intrinsic` from `extrinsic` (4x4 world to camera) - a project extension; legacy
    open3d has no ray cast, and the defaults follow open3d's VoxelBlockGrid.ray_cast.  -> RGBDImage of float32 depth
    in metres (0 where the ray meets no surface) and float32 colour: the intensity, or RGB in [0, 1] with
    convert_rgb_to_intensity=False.  A NoColor volume renders depth only (its colour image is empty).  One host read:
    the outputs share one device buffer, copied once."""
    want = 'intensity' if convert_rgb_to_intensity else 'colour'
    flat, out = self._raycast(intrinsic, extrinsic, depth_min, depth_max, weight_threshold,
                              ('depth', want) if self._color else ('depth',))
    host = flat.cpu().numpy()
    H, W = out['depth'].shape
    depth = host[:H * W].reshape(H, W)
    color = Image(host[H * W:].reshape(out[want].shape)) if self._color else Image()
    return RGBDImage(color, Image(depth))

  def raycast_tensors(self, intrinsic, extrinsic, depth_min=0.1, depth_max=3.0, weight_threshold=3.0,
                      outputs=('depth', 'intensity', 'colour')):
    """raycast() on the device, without a host read: -> {name: CUDA float32 tensor} for the requested outputs of
    'depth' [H, W], 'intensity' [H, W] and 'colour' [H, W, 3] (the last two RGB8 volumes only), views of one buffer
    in that order.  One launch."""
    return self._raycast(intrinsic, extrinsic, depth_min, depth_max, weight_threshold, tuple(outputs))[1]

  def _raycast(self, intrinsic, extrinsic, depth_min, depth_max, weight_threshold, outputs):
    """Check every argument, then launch dgr_tsdf_raycast -> (the flat device buffer, {name: view of it})."""
    if 'depth' not in outputs or any(o not in ('depth', 'intensity', 'colour') for o in outputs):
      raise ValueError(f"outputs must include 'depth' and name only depth / intensity / colour, got {outputs}")
    if not self._color and len(outputs) > 1:
      raise ValueError('a NoColor volume renders depth only')
    W, H = intrinsic.width, intrinsic.height
    if W < 1 or H < 1:
      raise ValueError(f'image size must be positive, got {W} x {H}')
    intr = intrinsic._params()
    if not (intr[0] > 0 and intr[1] > 0 and np.isfinite(intr).all()):
      raise ValueError('focal lengths must be finite and positive, the principal point finite')
    ext = np.asarray(extrinsic, dtype=np.float64)
    if ext.shape != (4, 4) or not np.isfinite(ext).all():
      raise ValueError(f'extrinsic must be a finite 4x4 matrix, got shape {ext.shape}')
    try:
      pose = np.linalg.inv(ext)
    except np.linalg.LinAlgError:
      raise ValueError('extrinsic must be invertible') from None
    if not np.isfinite(pose).all():
      raise ValueError('extrinsic must be invertible')
    if not (0.0 <= depth_min < depth_max < np.inf):
      raise ValueError(f'need 0 <= depth_min < depth_max < inf, got {depth_min}, {depth_max}')
    if not 0.0 < weight_threshold < np.inf:
      raise ValueError(f'weight_threshold must be finite and positive, got {weight_threshold}')
    steps = _raycast_max_steps(W, H, intr, pose, self.voxel_length, depth_max)
    if not steps <= _abi.TSDF_RAYCAST_MAX_STEPS:
      raise ValueError(f'a ray could take {steps:g} steps, more than {_abi.TSDF_RAYCAST_MAX_STEPS}: the focal '
                       'length, principal point, extrinsic scale, depth_max or voxel_length is out of range')
    _abi.refresh_stream()
    self._grow_slabs(self.n_units)
    sizes = {'depth': (H, W), 'intensity': (H, W), 'colour': (H, W, 3)}
    names = [o for o in ('depth', 'intensity', 'colour') if o in outputs]
    flat = torch.empty(sum(int(np.prod(sizes[o])) for o in names), dtype=torch.float32, device=self.device)
    out, at = {}, 0
    for o in names:
      n = int(np.prod(sizes[o]))
      out[o] = flat[at:at + n].view(sizes[o])
      at += n
    empty = self.n_units == 0
    _abi.tsdf_raycast(None if empty else self._keys, None if empty else self._vals, self._tsdf, self._weight,
                      self._rgb, W, H, intr, pose, self.voxel_length, self.sdf_trunc, depth_min, depth_max,
                      weight_threshold, out['depth'], out.get('intensity'), out.get('colour'))
    return flat, out

  def extract_point_cloud(self):
    raise NotImplementedError('ScalableTSDFVolume.extract_point_cloud is not implemented')

  def extract_voxel_point_cloud(self):
    raise NotImplementedError('ScalableTSDFVolume.extract_voxel_point_cloud is not implemented')

  def voxel_state(self):
    """Host copy of the volume: unit keys [n, 3] int32 in slot order, the slots the last frame touched (in
    first-touch order) and the slabs tsdf / weight [n, 4096], rgb [n, 3, 4096] (None for NoColor)."""
    n = self.n_units
    return {'unit_keys': self._unit_keys[:n].cpu(), 'touched': self._touched[:self.n_touched].cpu(),
            'tsdf': self._tsdf[:n].cpu(), 'weight': self._weight[:n].cpu(),
            'rgb': None if self._rgb is None else self._rgb[:n].cpu()}
