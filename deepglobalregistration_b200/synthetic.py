"""Deterministic synthetic scans and checkpoints (SURVEY.md §8d).

There is no network in the build environment, so neither the 3DMatch / KITTI
datasets nor the released DGR weights (downloaded by the reference at
``demo.py:14-26``) are available.  Everything measured or tested in this repo
therefore runs on seeded synthetic scans with the *shape* of the reference's
data and on seeded random-init checkpoints written in the reference's
checkpoint layout (``core/trainer.py:527-549`` as read back by
``core/deep_global_registration.py:88-129``).

numpy / torch-CPU only: this module is imported by the product (bench, tests)
and by the oracle alike, so it must not depend on either.
"""
import math

import numpy as np
import torch

# ResUNetBN2C hyper-parameters (reference model/resunet.py:419-426,662-665)
CHANNELS = [None, 32, 64, 128, 256]
TR_CHANNELS = [None, 64, 64, 64, 128]


class AttrDict(dict):
  """dict with attribute access: the reference reads its checkpoint config both
  as ``cfg.voxel_size`` and ``cfg['feat_model']``
  (core/deep_global_registration.py:89-127)."""

  def __getattr__(self, k):
    try:
      return self[k]
    except KeyError as e:
      raise AttributeError(k) from e

  def __setattr__(self, k, v):
    self[k] = v


# --------------------------------------------------------------------------- #
# rigid motions
# --------------------------------------------------------------------------- #
def random_se3(rng, max_angle_deg=45.0, max_trans=0.5):
  axis = rng.normal(size=3)
  axis /= np.linalg.norm(axis)
  ang = math.radians(max_angle_deg) * rng.uniform(0.2, 1.0)
  K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
  R = np.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * (K @ K)
  t = rng.uniform(-max_trans, max_trans, size=3)
  T = np.eye(4)
  T[:3, :3] = R
  T[:3, 3] = t
  return T


def apply_se3(T, xyz):
  return xyz @ T[:3, :3].T + T[:3, 3]


def rte_rre(T_pred, T_gt):
  """Translation error [m] and rotation error [rad]; the reference's metric
  definition (scripts/test_3dmatch.py:38-46) without its degree conversion."""
  rte = float(np.linalg.norm(T_pred[:3, 3] - T_gt[:3, 3]))
  c = (np.trace(T_pred[:3, :3].T @ T_gt[:3, :3]) - 1) / 2
  rre = float(np.arccos(np.clip(c, -1 + 1e-16, 1 - 1e-16)))
  return rte, rre


# --------------------------------------------------------------------------- #
# scans
# --------------------------------------------------------------------------- #
def _box_faces(lo, hi):
  lo, hi = np.asarray(lo, float), np.asarray(hi, float)
  faces = []
  for ax in range(3):
    o = [a for a in range(3) if a != ax]
    area = (hi[o[0]] - lo[o[0]]) * (hi[o[1]] - lo[o[1]])
    for v in (lo[ax], hi[ax]):
      faces.append((ax, v, o, area))
  return lo, hi, faces


def _sample_boxes(boxes, n, rng, noise):
  """Area-uniform samples on the faces of axis-aligned boxes."""
  allf = []
  for lo, hi in boxes:
    lo, hi, faces = _box_faces(lo, hi)
    for f in faces:
      allf.append((lo, hi) + f)
  areas = np.array([f[5] for f in allf])
  counts = rng.multinomial(n, areas / areas.sum())
  out = []
  for (lo, hi, ax, v, o, _), c in zip(allf, counts):
    p = np.empty((c, 3))
    p[:, ax] = v
    p[:, o[0]] = rng.uniform(lo[o[0]], hi[o[0]], c)
    p[:, o[1]] = rng.uniform(lo[o[1]], hi[o[1]], c)
    out.append(p)
  p = np.concatenate(out)
  p += rng.normal(scale=noise, size=p.shape)
  return p[rng.permutation(len(p))]


def room_boxes(seed, extent=(3.6, 3.0, 2.5), n_furniture=6):
  rng = np.random.default_rng(10_000 + seed)
  ex = np.asarray(extent, float)
  boxes = [(np.zeros(3), ex)]
  for _ in range(n_furniture):
    size = rng.uniform(0.4, 1.5, size=3) * np.minimum(1.0, ex / 3.0)
    lo = rng.uniform(0, 1, size=3) * (ex - size)
    lo[2] = 0.0
    boxes.append((lo, lo + size))
  return boxes


def room_scan(seed, n_raw=250_000, extent=(3.6, 3.0, 2.5), scene_seed=None, noise=0.005):
  """3DMatch-shape scan: a box room with furniture boxes, area-uniform surface
  samples with 5 mm noise.  n_raw=250k gives ~52k voxels at 0.05 m (SURVEY §8d
  config 2).  ``scene_seed`` fixes the geometry; ``seed`` the sampling."""
  boxes = room_boxes(seed if scene_seed is None else scene_seed, extent)
  rng = np.random.default_rng(seed)
  return _sample_boxes(boxes, n_raw, rng, noise)


def room_pair(seed, n_raw=250_000, extent=(3.6, 3.0, 2.5), rigid_copy=False, voxel_size=0.0625):
  """(xyz0, xyz1, T_gt) float64 with T_gt mapping cloud 0 into cloud 1's frame.

  rigid_copy=False: the same surfaces re-sampled with another seed, then moved by
  a random SE(3) (<=45 deg, <=0.5 m).  rigid_copy=True: cloud 1 is cloud 0
  translated by a multiple of 8 voxels (the network's coarsest tensor stride, so the
  strided lattices of both clouds align; use a power-of-two voxel size so the shift is
  exact in binary) - the known-answer case in which identical neighbourhoods yield
  identical features, exact correspondences and therefore the exact transform."""
  xyz0 = room_scan(2 * seed, n_raw, extent, scene_seed=seed)
  rng = np.random.default_rng(777 + seed)
  if rigid_copy:
    T = np.eye(4)
    T[:3, 3] = voxel_size * 8 * rng.integers(-3, 4, size=3)
    return xyz0, apply_se3(T, xyz0), T
  T = random_se3(rng)
  xyz1 = apply_se3(T, room_scan(2 * seed + 1, n_raw, extent, scene_seed=seed))
  return xyz0, xyz1, T


def lidar_scan(seed, pose_xy=(0.0, 0.0), n_beams=64, n_azimuth=1900, noise=0.02, scan_id=0):
  """KITTI-shape scan: 64 beams x 1900 azimuth steps over a ground plane, two street walls and
  ~40 box obstacles (parked cars, poles) fixed in the WORLD frame, seen from a sensor at
  pose_xy - so two poses along the street give genuinely different scans of one scene.
  ~120k returns, ~16-18k voxels at 0.3 m (SURVEY §8d config 3).  Points are in the sensor frame."""
  rng = np.random.default_rng(20_000 + seed)
  wall_l, wall_r = rng.uniform(6, 14), -rng.uniform(6, 14)
  h = 1.73
  n_obj = 40
  cx = rng.uniform(-40, 60, n_obj)
  cy = rng.uniform(wall_r + 1.0, wall_l - 1.0, n_obj)
  sx, sy = rng.uniform(0.2, 2.2, n_obj), rng.uniform(0.2, 1.0, n_obj)
  sz = rng.uniform(1.0, 3.0, n_obj)
  lo = np.stack([cx - sx, cy - sy, np.full(n_obj, -h)], 1)
  hi = np.stack([cx + sx, cy + sy, sz - h], 1)
  keep_obj = (np.abs(cx - pose_xy[0]) > 3.0) | (np.abs(cy - pose_xy[1]) > 2.0)   # none on top of the sensor
  lo, hi = lo[keep_obj], hi[keep_obj]
  elev = np.radians(np.linspace(-24.8, 2.0, n_beams))
  azim = np.linspace(-math.pi, math.pi, n_azimuth, endpoint=False)
  e, a = np.meshgrid(elev, azim, indexing='ij')
  d = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], -1).reshape(-1, 3)
  x0, y0 = pose_xy
  with np.errstate(divide='ignore', invalid='ignore'):
    tg = np.where(d[:, 2] < 0, -h / d[:, 2], np.inf)
    tl = np.where(d[:, 1] > 0, (wall_l - y0) / d[:, 1], np.inf)
    tr = np.where(d[:, 1] < 0, (wall_r - y0) / d[:, 1], np.inf)
    t = np.minimum(np.minimum(tg, tl), tr)
    org = np.array([x0, y0, 0.0])
    inv = 1.0 / d
    for blo, bhi in zip(lo, hi):                      # slab test against every box
      t1, t2 = (blo - org) * inv, (bhi - org) * inv
      tn = np.nanmax(np.minimum(t1, t2), axis=1)
      tf = np.nanmin(np.maximum(t1, t2), axis=1)
      hit = (tn <= tf) & (tf > 0) & (tn > 0)
      t = np.where(hit, np.minimum(t, tn), t)
  keep = t < 80.0
  p = d[keep] * t[keep, None]
  p += np.random.default_rng(1000 * seed + scan_id).normal(scale=noise, size=p.shape)
  return p


def lidar_pair(seed, advance=10.0):
  xyz0 = lidar_scan(seed, (0.0, 0.0), scan_id=0)
  xyz1 = lidar_scan(seed, (advance, 0.0), scan_id=1)
  T = np.eye(4)
  T[0, 3] = -advance  # a point at x in frame 0 sits at x-advance in frame 1
  return xyz0, xyz1, T


# --------------------------------------------------------------------------- #
# checkpoints
# --------------------------------------------------------------------------- #
def _bn_entries(prefix, c, g, sd):
  u = lambda: torch.rand(c, generator=g) * 0.2 - 0.1
  sd[prefix + '.bn.weight'] = 1.0 + u()
  sd[prefix + '.bn.bias'] = u()
  sd[prefix + '.bn.running_mean'] = u()
  sd[prefix + '.bn.running_var'] = 1.0 + u()
  sd[prefix + '.bn.num_batches_tracked'] = torch.tensor(1, dtype=torch.long)


def _kernel(g, kvol, cin, cout, gain=1.0):
  bound = gain / math.sqrt(kvol * cin)
  shape = (kvol, cin, cout) if kvol > 1 else (cin, cout)
  return (torch.rand(shape, generator=g) * 2 - 1) * bound


def resunet_state_dict(seed, in_channels, out_channels, conv1_kernel_size, D,
                       channels=CHANNELS, tr_channels=TR_CHANNELS, gain=3.0):
  """Seeded random-init state dict with MinkowskiEngine parameter names/shapes
  for the reference's ResUNet2 family (model/resunet.py:442-596,
  model/residual_block.py:98-115, model/common.py:13): ``*.kernel`` is
  [K, Cin, Cout] ([Cin, Cout] for 1x1), ``final.bias`` is [1, Cout]."""
  g = torch.Generator().manual_seed(seed)
  sd = {}
  C, T = channels, tr_channels
  k3 = 3 ** D

  def block(name, c):
    for i in (1, 2):
      sd[f'{name}.conv{i}.kernel'] = _kernel(g, k3, c, c, gain)
      _bn_entries(f'{name}.norm{i}', c, g, sd)

  sd['conv1.kernel'] = _kernel(g, conv1_kernel_size ** D, in_channels, C[1], gain)
  _bn_entries('norm1', C[1], g, sd)
  block('block1', C[1])
  for lvl in (2, 3, 4):
    sd[f'conv{lvl}.kernel'] = _kernel(g, k3, C[lvl - 1], C[lvl], gain)
    _bn_entries(f'norm{lvl}', C[lvl], g, sd)
    block(f'block{lvl}', C[lvl])
  tr_in = {4: C[4], 3: C[3] + T[4], 2: C[2] + T[3]}
  for lvl in (4, 3, 2):
    sd[f'conv{lvl}_tr.kernel'] = _kernel(g, k3, tr_in[lvl], T[lvl], gain)
    _bn_entries(f'norm{lvl}_tr', T[lvl], g, sd)
    block(f'block{lvl}_tr', T[lvl])
  sd['conv1_tr.kernel'] = _kernel(g, 1, C[1] + T[2], T[1], gain)
  sd['final.kernel'] = _kernel(g, 1, T[1], out_channels, gain)
  sd['final.bias'] = (torch.rand(1, out_channels, generator=g) * 2 - 1) * 0.1
  return sd


POINTNET_WIDTHS = ((3, 64), (64, 64), (64, 64), (64, 128), (128, 1024))
POINTNET_MODULES = (('h1.0', 'h1.1'), ('h1.3', 'h1.4'), ('h2.0', 'h2.1'), ('h2.3', 'h2.4'), ('h2.6', 'h2.7'))


def _pointnet_layer(sd, conv, bn, W, b, gamma, beta, mean, var):
  cout, cin = W.shape
  sd[conv + '.weight'] = torch.as_tensor(W, dtype=torch.float32).reshape(cout, cin, 1)
  sd[conv + '.bias'] = torch.as_tensor(b, dtype=torch.float32)
  sd[bn + '.weight'] = torch.as_tensor(gamma, dtype=torch.float32)
  sd[bn + '.bias'] = torch.as_tensor(beta, dtype=torch.float32)
  sd[bn + '.running_mean'] = torch.as_tensor(mean, dtype=torch.float32)
  sd[bn + '.running_var'] = torch.as_tensor(var, dtype=torch.float32)
  sd[bn + '.num_batches_tracked'] = torch.tensor(1, dtype=torch.long)


def pointnetlk_state_dict(seed):
  """Seeded PointNet_features state dict in the published PointNetLK layout (Conv1d weights [cout, cin, 1]):
  torch's default Conv1d init (uniform within 1 / sqrt(cin)) and BatchNorm statistics perturbed by up to 0.1, as
  ``resunet_state_dict`` does.  A random network: no trained weights exist offline."""
  g = torch.Generator().manual_seed(seed)
  sd = {}
  for (conv, bn), (cin, cout) in zip(POINTNET_MODULES, POINTNET_WIDTHS):
    bound = 1.0 / math.sqrt(cin)
    u = lambda: torch.rand(cout, generator=g) * 0.2 - 0.1
    W = (torch.rand(cout, cin, generator=g) * 2 - 1) * bound
    b = (torch.rand(cout, generator=g) * 2 - 1) * bound
    _pointnet_layer(sd, conv, bn, W, b, 1.0 + u(), u(), u(), 1.0 + u())
  return sd


def fibonacci_sphere(n):
  """n unit directions spread evenly over the sphere (the golden-angle spiral)."""
  k = np.arange(n) + 0.5
  z = 1.0 - 2.0 * k / n
  r = np.sqrt(1.0 - z * z)
  phi = math.pi * (3.0 - math.sqrt(5.0)) * k
  return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)


def pointnetlk_support_state_dict(carry=8.0, offset=10.0):
  """PointNet_features state dict whose features are the support function of the (centred) cloud, shifted:
  phi_k(P) = max_p a_k . p + offset for the 1024 Fibonacci-sphere directions a_k, up to the fp32 rounding of the
  weights (the BatchNorms are identities: gamma = sqrt(1 + eps), beta = mean = 0, var = 1).  Layers 1-4 carry x + carry, y + carry, z + carry through three identity channels (carry larger
  than any |coordinate|, so no ReLU clips them; the other channels are 0); layer 5 maps them to a_k . q + offset
  (offset larger than any |q|, so no ReLU clips).  A pose-sensitive descriptor with a known meaning."""
  sd = {}
  for l, ((conv, bn), (cin, cout)) in enumerate(zip(POINTNET_MODULES, POINTNET_WIDTHS)):
    W = np.zeros((cout, cin))
    b = np.zeros(cout)
    if l < 4:
      W[:3, :3] = np.eye(3)
      b[:3] = carry if l == 0 else 0.0
    else:
      A = fibonacci_sphere(cout)
      W[:, :3] = A
      b[:] = offset - carry * A.sum(1)
    _pointnet_layer(sd, conv, bn, W, b, np.full(cout, math.sqrt(1.0 + 1e-5)), np.zeros(cout), np.zeros(cout),
                    np.ones(cout))
  return sd


def make_checkpoint(seed=0, voxel_size=0.05, feat_conv1_kernel_size=7, feat_model_n_out=32,
                    inlier_conv1_kernel_size=3, inlier_feature_type='ones',
                    channels=CHANNELS, tr_channels=TR_CHANNELS, with_inlier=True):
  """dict(state_dict, state_dict_inlier, config) as DeepGlobalRegistration loads
  it (core/deep_global_registration.py:88-129)."""
  cfg = AttrDict(
      voxel_size=voxel_size, feat_model='ResUNetBN2C', feat_model_n_out=feat_model_n_out,
      bn_momentum=0.05, feat_conv1_kernel_size=feat_conv1_kernel_size, normalize_feature=True,
      inlier_model='ResUNetBN2C', inlier_conv1_kernel_size=inlier_conv1_kernel_size,
      inlier_feature_type=inlier_feature_type, nn_max_n=250)
  state = dict(config=cfg,
               state_dict=resunet_state_dict(seed, 1, feat_model_n_out, feat_conv1_kernel_size, 3,
                                             channels, tr_channels))
  if with_inlier:
    nin = 6 if inlier_feature_type == 'coords' else 1
    state['state_dict_inlier'] = resunet_state_dict(seed + 1, nin, 1, inlier_conv1_kernel_size, 6,
                                                    channels, tr_channels)
  return state


def correspondence_set(seed, n=1500, inlier_frac=0.3, noise=0.004):
  """Putative correspondences for the safeguard (RANSAC) tests: source points in a 3 m cube, a
  random pose (<= 40 deg, <= 0.5 m), `inlier_frac` of the targets = pose(source) + N(0, noise),
  the rest uniform clutter; target rows shuffled so idx1 is a real gather.
  -> (src f32 [n,3], tgt f32 [n,3], idx0, idx1, T_gt, inlier mask)."""
  g = np.random.default_rng(seed)
  P = g.uniform(-1.5, 1.5, size=(n, 3)).astype(np.float32)
  T = random_se3(g, 40.0, 0.5)
  Q = apply_se3(T, P.astype(np.float64)) + g.normal(0, noise, size=(n, 3))
  out = g.random(n) >= inlier_frac
  Q[out] = g.uniform(-2.0, 2.0, size=(int(out.sum()), 3))
  perm = g.permutation(n)
  tgt = np.empty_like(Q)
  tgt[perm] = Q
  return P, tgt.astype(np.float32), np.arange(n), perm, T, ~out


def feature_matching_pair(seed, n=2000, match_frac=0.3, spacing=0.1, noise=0.003, dim=16):
  """Clouds and features for the feature-matching RANSAC tests.  Source = n jittered points of a lattice
  of pitch `spacing` (so no two share a cell of a voxel hash finer than spacing / 2); target = a random pose
  (<= 40 deg, <= 0.5 m) of the source plus N(0, noise), rows shuffled.  Features: random unit vectors on the
  target; a source point's feature is its true partner's feature for `match_frac` of the points and a
  random other target row's otherwise (plus 1e-3 noise, far from any near-tie).
  -> (src f32 [n,3], tgt f32 [n,3], feat_src f32 [n,dim], feat_tgt f32 [n,dim], T_gt, partner [n],
  identified mask [n])."""
  g = np.random.default_rng(seed)
  side = int(np.ceil(n ** (1 / 3))) + 2
  lattice = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing='ij'), -1).reshape(-1, 3)
  P = (lattice[g.choice(len(lattice), n, replace=False)] - side / 2) * spacing
  P = (P + g.uniform(-0.1, 0.1, size=P.shape) * spacing).astype(np.float32)
  T = random_se3(g, 40.0, 0.5)
  Q = apply_se3(T, P.astype(np.float64)) + g.normal(0, noise, size=(n, 3))
  perm = g.permutation(n)                          # source i <-> target row perm[i]
  tgt = np.empty_like(Q)
  tgt[perm] = Q
  ft = g.normal(size=(n, dim))
  ft /= np.linalg.norm(ft, axis=1, keepdims=True)
  ident = g.random(n) < match_frac
  wrong = (perm + g.integers(1, n, size=n)) % n
  fs = ft[np.where(ident, perm, wrong)] + g.normal(0, 1e-3, size=(n, dim))
  return P, tgt.astype(np.float32), fs.astype(np.float32), ft.astype(np.float32), T, perm, ident
