"""Ray casting the TSDF volume on the GPU (dgr_tsdf_raycast through ScalableTSDFVolume.raycast / raycast_tensors)
against oracle/tsdf_raycast.py bit for bit, its launch count and argument checks, its depth against the
synthetic renderer at full size, and frame-to-model tracking (integration.track_model, --poses model)."""
import contextlib
import io as pyio
import json
import os

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import _abi
from deepglobalregistration_b200 import integration
from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import o3d_integration as integ
from deepglobalregistration_b200 import synthetic as syn
from deepglobalregistration_b200.core.multiway import absolute_trajectory_error
from oracle import tsdf as ot
from oracle import tsdf_raycast as orc

pytestmark = pytest.mark.gpu

VL, TRUNC = 0.02, 0.06
W, H = 160, 120


def _rgbd(color, depth_raw, max_depth=4.5):
  return integ.RGBDImage.create_from_color_and_depth(integ.Image(color), integ.Image(depth_raw), depth_trunc=max_depth,
                                                     convert_rgb_to_intensity=False)


@pytest.fixture(scope='module')
def small():
  c, d, P, K = syn.rgbd_sequence(3, 12, width=W, height=H, turn=0.05, radius=0.05)
  intr = integ.PinholeCameraIntrinsic(W, H, *K)
  vols = {True: integ.ScalableTSDFVolume(VL, TRUNC, integ.TSDFVolumeColorType.RGB8),
          False: integ.ScalableTSDFVolume(VL, TRUNC, integ.TSDFVolumeColorType.NoColor)}
  ov = ot.Volume(VL, TRUNC, color=True)
  for k in range(len(P)):
    for v in vols.values():
      v.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(P[k]))
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (W, H) + tuple(K), np.linalg.inv(P[k]), c[k])
  gray = ot.Volume(VL, TRUNC, color=False)          # integration of tsdf / weight does not depend on the colour
  gray.keys, gray.slot, gray.tsdf, gray.weight = ov.keys, ov.slot, ov.tsdf, ov.weight
  assert torch.equal(vols[True].voxel_state()['tsdf'], torch.from_numpy(ov.tsdf))
  assert torch.equal(vols[False].voxel_state()['weight'], torch.from_numpy(ov.weight))
  return c, d, P, K, intr, vols, {True: ov, False: gray}


@pytest.fixture(scope='module')
def around():
  """A volume whose 12 frames turn half a revolution, so the room is observed on both sides of the camera path."""
  c, d, P, K = syn.rgbd_sequence(3, 12, width=W, height=H)
  intr = integ.PinholeCameraIntrinsic(W, H, *K)
  vols = {True: integ.ScalableTSDFVolume(VL, TRUNC, integ.TSDFVolumeColorType.RGB8),
          False: integ.ScalableTSDFVolume(VL, TRUNC, integ.TSDFVolumeColorType.NoColor)}
  ov = ot.Volume(VL, TRUNC, color=True)
  for k in range(len(P)):
    for v in vols.values():
      v.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(P[k]))
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (W, H) + tuple(K), np.linalg.inv(P[k]), c[k])
  gray = ot.Volume(VL, TRUNC, color=False)
  gray.keys, gray.slot, gray.tsdf, gray.weight = ov.keys, ov.slot, ov.tsdf, ov.weight
  return c, d, P, K, intr, vols, {True: ov, False: gray}


def _behind_surface(P, d, k=9, back=0.03):
  """3 cm behind the surface frame k's centre pixel sees, looking back across the room."""
  R, C = P[k][:3, :3], P[k][:3, 3]
  X = C + (d[k][H // 2, W // 2] / 1000.0) * R[:, 2]
  pose = np.eye(4)
  pose[:3, :3] = R @ np.diag([-1.0, 1.0, -1.0])
  pose[:3, 3] = X + back * R[:, 2]
  return pose


def _voxel_at(ov, p):
  """(tsdf, weight) of the oracle voxel holding world point p, or None in a missing unit."""
  g = np.floor(p / VL)
  U = np.floor(g / 16)
  s = ov.slot.get(tuple(int(x) for x in U), -1)
  if s < 0:
    return None
  lo = (g - 16 * U).astype(int)
  lv = (lo[0] * 16 + lo[1]) * 16 + lo[2]
  return float(ov.tsdf[s, lv]), float(ov.weight[s, lv])


def _case(name, P, ov):
  """-> (camera-to-world pose, depth_min, depth_max, weight_threshold) of a named bit-exactness case."""
  pose = P[4].copy()
  if name == 'between':                              # halfway between two fused positions, frame 5's rotation
    pose = P[5].copy()
    pose[:3, 3] = 0.5 * (P[5][:3, 3] + P[6][:3, 3])
  elif name == 'outside':                            # 6 m behind frame 0, outside every unit
    pose = P[0].copy()
    pose[:3, 3] -= 6.0 * pose[:3, 2]
    return pose, 0.1, 9.0, 3.0
  elif name == 'unit_boundaries':                    # optical axis (pixel (cx, cy)) along two unit planes
    L = 16 * VL
    pose = np.eye(4)
    pose[:3, :3] = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])     # camera z -> world +x
    pose[:3, 3] = (3 * L, 5 * L, 4 * L)
  elif name == 'depth_cut':
    return pose, 0.1, 1.5, 3.0
  elif name == 'threshold_above_all':
    return pose, 0.1, 3.0, float(ov.weight.max()) + 1.0
  return pose, 0.1, 3.0, 3.0


CASES = ['fused', 'between', 'outside', 'behind_surface', 'unit_boundaries', 'depth_cut', 'threshold_above_all']


@pytest.mark.parametrize('color', [True, False])
@pytest.mark.parametrize('name', CASES)
def test_bit_exact_against_oracle(request, name, color):
  if name == 'behind_surface':
    # Every ray starts at the camera centre, in a known voxel behind a surface (tsdf < 0), so it must pass a positive
    # sample before it may hit.  Measured (oracle): hit share 0.287; most hits are the next crossing within 6 cm of
    # that surface, 178 rays reach surfaces beyond 0.5 m.
    c, d, P, K, intr, vols, ovs = request.getfixturevalue('around')
    pose, dmin, dmax, wthr = _behind_surface(P, d), 0.0, 6.0, 3.0
    start = _voxel_at(ovs[True], pose[:3, 3])
    assert start is not None and start[0] < 0 and start[1] >= wthr
  else:
    c, d, P, K, intr, vols, ovs = request.getfixturevalue('small')
    pose, dmin, dmax, wthr = _case(name, P, ovs[True])
  ext = np.linalg.inv(pose)
  outs = ('depth', 'intensity', 'colour') if color else ('depth',)
  got = vols[color].raycast_tensors(intr, ext, dmin, dmax, wthr, outputs=outs)
  D, I, Col = orc.raycast(ovs[color], (W, H) + tuple(K), ext, dmin, dmax, wthr)
  hits = float((D > 0).mean())
  print(f'\n[raycast exact] {name} colour {color}: hit share {hits:.3f}')
  assert torch.equal(got['depth'].cpu(), torch.from_numpy(D))
  if color:
    assert torch.equal(got['intensity'].cpu(), torch.from_numpy(I))
    assert torch.equal(got['colour'].cpu(), torch.from_numpy(Col))
  else:
    assert I is None and Col is None
  if name == 'threshold_above_all':
    assert hits == 0.0 and not got['depth'].any()
  elif name in ('fused', 'between', 'depth_cut'):
    assert hits > 0.3
  if name == 'depth_cut':
    assert D.max() <= 1.5
  if name == 'behind_surface':
    assert hits >= 0.2 and (D > 0.5).sum() >= 100


@pytest.mark.parametrize('color', [True, False])
def test_empty_volume(small, color):
  c, d, P, K, intr, _, _ = small
  vol = integ.ScalableTSDFVolume(VL, TRUNC, integ.TSDFVolumeColorType.RGB8 if color else
                                 integ.TSDFVolumeColorType.NoColor)
  outs = ('depth', 'intensity', 'colour') if color else ('depth',)
  got = vol.raycast_tensors(intr, np.linalg.inv(P[0]), outputs=outs)
  D, I, Col = orc.raycast(ot.Volume(VL, TRUNC, color=color), (W, H) + tuple(K), np.linalg.inv(P[0]))
  assert not D.any()
  for name, ref in zip(outs, (D, I, Col)):
    assert torch.equal(got[name].cpu(), torch.from_numpy(ref))


def test_deterministic_one_launch_and_argument_checks(small):
  c, d, P, K, intr, vols, _ = small
  ext = np.linalg.inv(P[3])
  vol = vols[True]
  a = vol.raycast_tensors(intr, ext)
  torch.cuda.synchronize()
  before = _abi.lib().dgr_launch_count()
  b = vol.raycast_tensors(intr, ext)
  assert _abi.lib().dgr_launch_count() == before + 1          # one kernel, no workspace, no host read
  for k in a:
    assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes()
  img = vol.raycast(intr, ext)
  assert np.array_equal(np.asarray(img.depth), a['depth'].cpu().numpy())
  assert np.array_equal(np.asarray(img.color), a['intensity'].cpu().numpy())
  rgb = vol.raycast(intr, ext, convert_rgb_to_intensity=False)
  assert np.array_equal(np.asarray(rgb.color), a['colour'].cpu().numpy())
  gray = vols[False].raycast(intr, ext)
  assert np.array_equal(np.asarray(gray.depth), a['depth'].cpu().numpy()) and np.asarray(gray.color).size == 0
  torch.cuda.synchronize()
  before = _abi.lib().dgr_launch_count()
  bad = [dict(depth_min=-0.1), dict(depth_min=2.0, depth_max=1.0), dict(depth_max=np.inf), dict(depth_max=1e6),
         dict(weight_threshold=0.0), dict(weight_threshold=np.nan), dict(extrinsic=np.full((4, 4), np.nan)),
         dict(extrinsic=np.zeros((4, 4))), dict(extrinsic=np.eye(3)), dict(outputs=('intensity',)),
         dict(intrinsic=integ.PinholeCameraIntrinsic(W, H, 0.0, 100.0, 80.0, 60.0)),
         # rays whose world length per unit of t is unbounded: the march could stall or run for ever
         dict(intrinsic=integ.PinholeCameraIntrinsic(W, H, 1e-30, 1e-30, 80.0, 60.0)),
         dict(intrinsic=integ.PinholeCameraIntrinsic(W, H, 1e-3, 1e-3, 80.0, 60.0)),
         dict(intrinsic=integ.PinholeCameraIntrinsic(W, H, 100.0, 100.0, 1e9, 60.0)),
         dict(extrinsic=np.diag([1e-4, 1e-4, 1e-4, 1.0]) @ ext),
         dict(depth_max=600.0)]                                   # 72 600 steps at 2 cm
  for kw in bad:
    args = dict(intrinsic=intr, extrinsic=ext)
    args.update(kw)
    with pytest.raises(ValueError):
      vol.raycast_tensors(**args)
  with pytest.raises(ValueError):
    vols[False].raycast_tensors(intr, ext, outputs=('depth', 'intensity'))
  g = vols[False]
  dep = torch.empty(H, W, device=g.device)
  inten = torch.empty(H, W, device=g.device)
  common = (intr._params(), P[3], VL, TRUNC)
  with pytest.raises(_abi.DgrError):                           # colour output from a NoColor volume
    _abi.tsdf_raycast(g._keys, g._vals, g._tsdf, g._weight, None, W, H, *common, 0.1, 3.0, 3.0, dep, inten)
  nan_pose = P[3].copy()
  nan_pose[0, 3] = np.nan
  with pytest.raises(_abi.DgrError):                           # the library checks the pose itself
    _abi.tsdf_raycast(g._keys, g._vals, g._tsdf, g._weight, None, W, H, intr._params(), nan_pose, VL, TRUNC, 0.1,
                      3.0, 3.0, dep)
  with pytest.raises(_abi.DgrError):
    _abi.tsdf_raycast(g._keys, g._vals, g._tsdf, g._weight, None, W, H, *common, 0.5, 0.5, 3.0, dep)
  with pytest.raises(_abi.DgrError):                           # the library bounds the steps itself
    _abi.tsdf_raycast(g._keys, g._vals, g._tsdf, g._weight, None, W, H, (1e-30, 1e-30, 80.0, 60.0), P[3], VL, TRUNC,
                      0.1, 3.0, 3.0, dep)
  with pytest.raises(_abi.DgrError):
    _abi.tsdf_raycast(None, None, None, None, None, 640, 480, (1e-30, 1e-30, 320.0, 240.0), np.eye(4), VL, TRUNC,
                      0.1, 3.0, 3.0, torch.empty(480, 640, device=g.device))
  assert _abi.lib().dgr_launch_count() == before


@pytest.fixture(scope='module')
def vga():
  c, d, P, K = syn.rgbd_sequence(0, 50, 640, 480)
  intr = integ.PinholeCameraIntrinsic(640, 480, *K)
  vol = integ.ScalableTSDFVolume(0.008, 0.04, integ.TSDFVolumeColorType.RGB8)
  for k in range(50):
    vol.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(P[k]))
  return c, d, P, K, intr, vol


def test_geometry_full_size(vga):
  # 640 x 480, 50 frames fused at 8 mm / 4 cm, rendered at the frames' own poses against the renderer's depth.
  # Measured on an H100: hit share (frames 0, 10, 25, 40, 49) 0.816 / 1.000 / 0.999 / 0.999 / 0.884 (the path's ends
  # see view edges fewer than 3 frames saw); |depth error| median 1.78 mm, 95th percentile 3.97 mm (the sample is the
  # voxel holding p, so a crossing is off by up to half a voxel).
  c, d, P, K, intr, vol = vga
  errs, shares = [], []
  for k in (0, 10, 25, 40, 49):
    D = vol.raycast_tensors(intr, np.linalg.inv(P[k]), outputs=('depth',))['depth'].cpu().numpy()
    gt = d[k].astype(np.float32) / np.float32(1000.0)
    gt[gt > 3.0] = 0
    both = (D > 0) & (gt > 0)
    errs.append(np.abs(D - gt)[both])
    shares.append(both.sum() / (gt > 0).sum())
  err = np.concatenate(errs)
  med, p95 = float(np.median(err)), float(np.percentile(err, 95))
  print(f'\n[raycast vga] hit share per frame {np.round(shares, 4).tolist()}, |depth error| median {med * 1e3:.3f} mm, '
        f'p95 {p95 * 1e3:.3f} mm')
  assert min(shares) >= 0.75
  assert med <= 0.0025 and p95 <= 0.006


def _gt_relative(P):
  return np.linalg.inv(P[0]) @ P


def test_tracking_accuracy_and_determinism():
  # syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05): 0.72 degrees and 6 mm per frame, 640 x 480.  Measured on an
  # H100: ATE 2.97 mm, no failure (--poses odometry with its pose graph: 1.2 mm on the same frames).
  c, d, P, K = syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05)
  intr = integ.PinholeCameraIntrinsic(640, 480, *K)
  runs = []
  for _ in range(2):
    poses, vol, st = integration.track_model(zip(c, d), intr)
    runs.append(poses)
  ate = float(absolute_trajectory_error(runs[0], _gt_relative(P)))
  print(f'\n[model tracking] 50 frames: ATE {ate * 1e3:.3f} mm, {st}, {vol.n_units} units')
  assert runs[0].tobytes() == runs[1].tobytes()
  assert st == dict(tracked_frames=49, tracking_failures=0)
  assert ate <= 4.5e-3


def _noisy(d, seed):
  """Depth noise growing with z^2 (0.0012 + 0.0019 (z - 0.4)^2 m, an axial Kinect noise model), quantised to mm."""
  rng = np.random.default_rng(seed)
  z = d.astype(np.float64) / 1000.0
  sigma = 0.0012 + 0.0019 * (z - 0.4) ** 2
  mm = np.round((z + rng.standard_normal(z.shape) * sigma) * 1000.0)
  return np.where(d > 0, np.clip(mm, 1, 65535), 0).astype(np.uint16)


def test_tracking_on_noisy_frames(tmp_path):
  # Measured on an H100: ATE --poses odometry 1.20 mm, --poses model 2.99 mm.  Frame-to-model tracking is not better
  # than the odometry chain plus pose graph here: both errors stay at their noise-free values, so the model's error
  # is set by the rendering (nearest-voxel samples), not by the depth noise.  DESIGN.md records the finding.
  c, d, P, K = syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05)
  dn = _noisy(d, 11)
  seq = syn.write_rgbd_sequence(str(tmp_path), 'room', c, dn, P, K)
  frames = integration.sequence_frames(seq, need_poses=False)
  intr = integ.PinholeCameraIntrinsic(640, 480, *K)
  gt = _gt_relative(P)
  P_odo, _ = integration.odometry_poses(seq, frames, intr, 0, 50)
  P_model, _, st = integration.model_poses(seq, frames, intr, 0, 50)
  ate_odo = float(absolute_trajectory_error(P_odo, gt))
  ate_model = float(absolute_trajectory_error(P_model, gt))
  print(f'\n[noisy tracking] ATE --poses odometry {ate_odo * 1e3:.3f} mm, --poses model {ate_model * 1e3:.3f} mm, {st}')
  assert st['tracking_failures'] == 0
  assert ate_model <= 4.5e-3 and ate_odo <= 2.5e-3


def _cli(argv):
  buf = pyio.StringIO()
  with contextlib.redirect_stdout(buf):
    code = integration.main(argv)
  return code, (json.loads(buf.getvalue().strip().splitlines()[-1]) if code == 0 else None)


def test_integration_cli_model(tmp_path):
  cols, deps, poses, intr = syn.rgbd_sequence(5, 12, turn=0.02, radius=0.02)    # 0.65 degrees, 1 cm per frame
  syn.write_rgbd_sequence(str(tmp_path / 'raw'), 'room', cols, deps, poses, intr)
  code, summary = _cli([str(tmp_path / 'raw' / 'room'), str(tmp_path / 'out'), '--frames_per_fragment', '12',
                        '--poses', 'model'])
  print('\nintegration --poses model:', summary)
  assert code == 0 and summary['fragments'] == 1 and summary['frames'] == 12
  assert summary['tracked_frames'] == 11 and summary['tracking_failures'] == 0
  assert summary['fragment_ate'][0] <= 2.5e-3                  # measured on an H100: 1.25 mm
  assert 'odometry_pairs' not in summary
  seq_out = tmp_path / 'out' / 'room' / 'seq-01'
  assert sorted(os.listdir(seq_out)) == ['fragment-0.log', 'fragment-0.ply']
  assert len(dio.read_trajectory(str(seq_out / 'fragment-0.log'))) == 12
  v = np.asarray(dio.read_point_cloud(str(seq_out / 'fragment-0.ply')).points)
  vw = v @ poses[0][:3, :3].T + poses[0][:3, 3]                # first camera -> world
  face, _ = syn.box_face_distance(vw, syn.room_boxes(5, (3.6, 3.0, 2.5)))
  print('model fragment: median / 95% vertex-face distance', np.median(face), np.quantile(face, 0.95))
  assert len(v) > 1000
  assert np.median(face) <= 1e-3 and np.quantile(face, 0.95) <= 3e-3    # measured: 0.23 mm, 0.59 mm
  n = _abi.POSE_GRAPH_MAX_NODES + 1                            # no pose graph: the fragment length is not capped
  code, s2 = _cli([str(tmp_path / 'raw' / 'room'), str(tmp_path / 'out2'), '--frames_per_fragment', str(n),
                   '--poses', 'model'])
  assert code == 0 and s2['fragments'] == 1 and s2['tracked_frames'] == 11
  with pytest.raises(SystemExit):
    _cli([str(tmp_path / 'raw' / 'room'), str(tmp_path / 'out3'), '--frames_per_fragment', str(n),
          '--poses', 'odometry'])
