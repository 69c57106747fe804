"""RGB-D fusion on the GPU (csrc/tsdf.cu through o3d_integration.ScalableTSDFVolume) against oracle/tsdf.py: the
volume state and the mesh bit for bit, determinism, accuracy against the analytic room, a fuse-then-register loop,
the open3d stand-in, the CLI and the edge cases."""
import json
import os
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import io as dio
from deepglobalregistration_b200 import o3d_integration as integ
from deepglobalregistration_b200 import synthetic as syn
from oracle import tsdf as ot

pytestmark = pytest.mark.gpu

SMALL = dict(width=160, height=120)
# Vertices of a 50-frame 640 x 480 fragment at 8 mm, away (> 2 cm) from box edges, against the analytic faces.
# Measured on an H100: p50 / p90 / p99 / p99.9 / max = 0.08 / 0.26 / 0.77 / 25.9 / 31.0 mm.  The tail past p99 is the
# spurious surface TSDF fusion leaves along depth discontinuities (furniture silhouettes seen at grazing angles); it
# cannot reach past the truncation distance.
# 0.59 % of the vertices lie farther than 5 mm.
FACE_P99_BOUND = 0.0015
FACE_TAIL_SHARE = 0.01
# FPFH + FGR + ICP recovers the known motion between two fused fragments within these bounds (measured on an H100:
# RTE 1.35 cm, RRE 0.11 deg); the success criterion of evaluate.py is 0.3 m / 15 deg.
LOOP_RTE_BOUND, LOOP_RRE_BOUND = 0.05, 1.0


def _frames(seed, n, **kw):
  c, d, P, K = syn.rgbd_sequence(seed, n, **{**SMALL, **kw})
  return c, d, P, K


def _rgbd(color, depth_raw, max_depth=4.5):
  return integ.RGBDImage.create_from_color_and_depth(integ.Image(color), integ.Image(depth_raw), depth_trunc=max_depth,
                                                     convert_rgb_to_intensity=False)


def _intr(c, K):
  return integ.PinholeCameraIntrinsic(c.shape[2], c.shape[1], *K)


def _gpu_volume(c, d, P, K, vl, trunc, color=True, frames=None, vol=None):
  vol = vol or integ.ScalableTSDFVolume(vl, trunc, integ.TSDFVolumeColorType.RGB8 if color else
                                        integ.TSDFVolumeColorType.NoColor)
  intr = _intr(c, K)
  for k in (range(len(P)) if frames is None else frames):
    vol.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(P[k]))
  return vol


def _oracle_volume(c, d, P, K, vl, trunc, color=True, frames=None, check=None):
  ov = ot.Volume(vl, trunc, color=color)
  W, H = c.shape[2], c.shape[1]
  for k in (range(len(P)) if frames is None else frames):
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (W, H) + tuple(K), np.linalg.inv(P[k]),
                 c[k] if color else None)
    if check is not None:
      check(k, ov)
  return ov


def _assert_state_equal(vol, ov):
  s = vol.voxel_state()
  assert torch.equal(s['unit_keys'], torch.from_numpy(ov.keys.astype(np.int32)))
  assert torch.equal(s['tsdf'], torch.from_numpy(ov.tsdf))
  assert torch.equal(s['weight'], torch.from_numpy(ov.weight))
  if ov.color:
    assert torch.equal(s['rgb'], torch.from_numpy(ov.rgb))
  else:
    assert s['rgb'] is None


def _assert_mesh_equal(v, c, t, V, C, T):
  assert torch.equal(v.cpu(), torch.from_numpy(V))
  assert torch.equal(t.cpu(), torch.from_numpy(T))
  if C is None:
    assert c is None
  else:
    assert torch.equal(c.cpu(), torch.from_numpy(C))


@pytest.mark.parametrize('color', [True, False])
def test_state_and_mesh_bit_exact(color):
  c, d, P, K = _frames(3, 20)
  vol = integ.ScalableTSDFVolume(0.02, 0.06, integ.TSDFVolumeColorType.RGB8 if color else
                                 integ.TSDFVolumeColorType.NoColor)
  intr = _intr(c, K)
  ov = ot.Volume(0.02, 0.06, color=color)
  for k in range(len(P)):
    vol.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(P[k]))
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (160, 120) + tuple(K), np.linalg.inv(P[k]),
                 c[k] if color else None)
    assert torch.equal(vol.voxel_state()['touched'], torch.from_numpy(ov.last_touched.astype(np.int32))), k
  _assert_state_equal(vol, ov)
  print(f'\n[tsdf state] colour {color}: {len(ov.keys)} units, last frame touched {len(ov.last_touched)}')
  v, cc, t = vol.extract_triangle_mesh_tensors()
  V, C, T = ov.extract_triangle_mesh()
  print(f'[tsdf mesh] {len(V)} vertices, {len(T)} triangles')
  assert len(T) > 1000
  _assert_mesh_equal(v, cc, t, V, C, T)
  mesh = vol.extract_triangle_mesh()
  assert np.array_equal(mesh.vertices, V) and np.array_equal(mesh.triangles, T)
  assert mesh.has_vertex_colors() == color


def test_determinism():
  c, d, P, K = _frames(5, 12)
  outs = []
  for _ in range(2):
    vol = _gpu_volume(c, d, P, K, 0.015, 0.05)
    s = vol.voxel_state()
    v, cc, t = vol.extract_triangle_mesh_tensors()
    outs.append([s['unit_keys'], s['tsdf'], s['weight'], s['rgb'], v.cpu(), cc.cpu(), t.cpu()])
  for a, b in zip(*outs):
    assert a.dtype == b.dtype and a.shape == b.shape
    assert a.numpy().tobytes() == b.numpy().tobytes()


@pytest.fixture(scope='module')
def vga_sequence():
  return syn.rgbd_sequence(0, 75, 640, 480)


def test_full_size_fragment_accuracy(vga_sequence):
  c, d, P, K = vga_sequence
  vol = _gpu_volume(c, d, P, K, 0.008, 0.04, frames=range(50))
  mesh = vol.extract_triangle_mesh()
  face, edge = syn.box_face_distance(mesh.vertices, syn.room_boxes(0))
  away = face[edge > 0.02]
  q = np.percentile(away, [50, 90, 99, 99.9, 100])
  print(f'\n[tsdf accuracy] {vol.n_units} units, {len(mesh.vertices)} vertices, {len(mesh.triangles)} triangles; '
        f'face distance away from edges p50/p90/p99/p99.9/max = ' + ' / '.join(f'{x * 1e3:.2f}' for x in q) + ' mm')
  tail = float((away > 0.005).mean())
  print(f'[tsdf accuracy] share farther than 5 mm: {tail:.5f}')
  assert len(away) > 100_000
  assert np.percentile(away, 99) <= FACE_P99_BOUND
  assert tail <= FACE_TAIL_SHARE
  assert away.max() <= 0.04                         # sdf_trunc


def test_fused_fragments_register(vga_sequence):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.core.fpfh_baseline import FPFHFastGlobal
  c, d, P, K = vga_sequence
  A = _gpu_volume(c, d, P, K, 0.008, 0.04, frames=range(0, 50)).extract_triangle_mesh().vertices
  B = _gpu_volume(c, d, P, K, 0.008, 0.04, frames=range(25, 75)).extract_triangle_mesh().vertices
  rng = np.random.default_rng(7)
  T_gt = syn.random_se3(rng, max_angle_deg=30.0, max_trans=0.5)
  dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=syn.make_checkpoint(0, voxel_size=0.05),
                                                     clip_weight_thresh=0.05, verbose=False))
  dgr.use_icp = True
  T = FPFHFastGlobal(dgr).register(B, syn.apply_se3(T_gt, A))
  ok, rte, rre = ev.rte_rre(T, T_gt, 0.3, 15.0)
  print(f'\n[tsdf loop] fragments of {len(A)} / {len(B)} vertices: RTE {rte:.4f} m, RRE {rre:.3f} deg')
  assert ok == 1.0
  assert rte <= LOOP_RTE_BOUND and rre <= LOOP_RRE_BOUND


def test_open3d_stand_in_matches_direct_api(tmp_path):
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  c, d, P, K = _frames(2, 6)
  seq = syn.write_rgbd_sequence(str(tmp_path), 'scene', c, d, P, K)
  files = sorted(os.listdir(seq))
  colors = [f for f in files if f.endswith('.color.png')]
  depths = [f for f in files if f.endswith('.depth.png')]
  poses = [f for f in files if f.endswith('.pose.txt')]
  Kf = np.loadtxt(os.path.join(seq, '..', 'camera-intrinsics.txt'))
  width, height = o3d.io.read_image(os.path.join(seq, colors[0])).get_max_bound()
  intrinsic = o3d.camera.PinholeCameraIntrinsic(int(width), int(height), Kf[0, 0], Kf[1, 1], Kf[0, 2], Kf[1, 2])
  volume = o3d.integration.ScalableTSDFVolume(voxel_length=0.02, sdf_trunc=0.06,
                                              color_type=o3d.integration.TSDFVolumeColorType.RGB8)
  for i in range(len(colors)):
    rgbd = o3d.geometry.RGBDImage.create_from_color_and_depth(
        o3d.io.read_image(os.path.join(seq, colors[i])), o3d.io.read_image(os.path.join(seq, depths[i])),
        depth_trunc=4.5, convert_rgb_to_intensity=False)
    volume.integrate(rgbd, intrinsic, np.linalg.inv(np.loadtxt(os.path.join(seq, poses[i]))))
  mesh = volume.extract_triangle_mesh()
  assert o3d.io.write_triangle_mesh(str(tmp_path / 'fragment-0.ply'), mesh)
  direct = _gpu_volume(c, d, P, K, 0.02, 0.06).extract_triangle_mesh()
  assert len(mesh.triangles) > 100
  assert np.array_equal(mesh.vertices, direct.vertices) and np.array_equal(mesh.triangles, direct.triangles)
  assert np.array_equal(mesh.vertex_colors, direct.vertex_colors)
  back = dio.read_point_cloud(str(tmp_path / 'fragment-0.ply')).points
  assert np.array_equal(back, direct.vertices.astype(np.float32).astype(np.float64))


def test_cli_writes_fragments(tmp_path, capsys):
  from deepglobalregistration_b200 import integration as cli
  c, d, P, K = _frames(4, 7)
  syn.write_rgbd_sequence(str(tmp_path / 'raw'), 'scene', c, d, P, K)
  argv = [str(tmp_path / 'raw' / 'scene'), str(tmp_path / 'out'), '--frames_per_fragment', '3',
          '--voxel_length', '0.02', '--sdf_trunc', '0.06']
  assert cli.main(argv) == 0
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  assert summary['fragments'] == 3 and summary['frames'] == 7
  for k, frames in enumerate((range(0, 3), range(3, 6), range(6, 7))):
    path = tmp_path / 'out' / 'scene' / 'seq-01' / f'fragment-{k}.ply'
    direct = _gpu_volume(c, d, P, K, 0.02, 0.06, frames=frames).extract_triangle_mesh()
    got = dio.read_point_cloud(str(path)).points
    assert np.array_equal(got, direct.vertices.astype(np.float32).astype(np.float64)), k
  assert cli.main(argv) == 2                          # the scene directory exists now
  assert 'overwrite' in capsys.readouterr().err
  assert cli.main(argv + ['--overwrite']) == 0


def test_edge_cases():
  c, d, P, K = _frames(6, 4)
  intr = _intr(c, K)
  empty = integ.ScalableTSDFVolume(0.02, 0.06, integ.TSDFVolumeColorType.RGB8)
  m = empty.extract_triangle_mesh()                   # empty extract
  assert m.vertices.shape == (0, 3) and m.triangles.shape == (0, 3)
  zero = np.zeros_like(d[0])
  empty.integrate(_rgbd(c[0], zero), intr, np.linalg.inv(P[0]))   # all-zero frame: nothing touched
  assert empty.n_units == 0 and empty.n_touched == 0
  # extract, integrate more, extract == integrate everything, extract
  vol = _gpu_volume(c, d, P, K, 0.02, 0.06, frames=range(2))
  vol.extract_triangle_mesh()
  vol.integrate(_rgbd(c[0], zero), intr, np.linalg.inv(P[1]))      # an all-zero frame changes nothing
  _gpu_volume(c, d, P, K, 0.02, 0.06, frames=range(2, 4), vol=vol)
  ref = _gpu_volume(c, d, P, K, 0.02, 0.06)
  a, b = vol.extract_triangle_mesh(), ref.extract_triangle_mesh()
  assert np.array_equal(a.vertices, b.vertices) and np.array_equal(a.triangles, b.triangles)
  # a frame whose depth was seen from the opposite direction: voxels behind the camera are skipped as the oracle does
  flip = P[0].copy()
  flip[:3, :3] = flip[:3, :3] @ np.diag([-1.0, 1.0, -1.0])
  ov = _oracle_volume(c, d, P, K, 0.02, 0.06, frames=[0])
  ov.integrate(ot.depth_from_raw(d[1], 1000.0, 4.5), (160, 120) + tuple(K), np.linalg.inv(flip), c[1])
  gv = _gpu_volume(c, d, P, K, 0.02, 0.06, frames=[0])
  gv.integrate(_rgbd(c[1], d[1]), intr, np.linalg.inv(flip))
  _assert_state_equal(gv, ov)
  # reset
  vol.reset()
  assert vol.n_units == 0 and vol.extract_triangle_mesh().is_empty()
  _gpu_volume(c, d, P, K, 0.02, 0.06, vol=vol)
  a = vol.extract_triangle_mesh()
  assert np.array_equal(a.vertices, b.vertices) and np.array_equal(a.triangles, b.triangles)


def test_host_argument_errors():
  c, d, P, K = _frames(6, 1)
  intr = _intr(c, K)
  with pytest.raises(ValueError):
    integ.ScalableTSDFVolume(0.02, 0.06, volume_unit_resolution=8)
  with pytest.raises(ValueError):
    integ.ScalableTSDFVolume(0.02, 0.06, depth_sampling_stride=0)
  with pytest.raises(ValueError):
    integ.ScalableTSDFVolume(0.02, 0.0)
  with pytest.raises(ValueError):
    integ.ScalableTSDFVolume(-0.02, 0.06)
  with pytest.raises(NotImplementedError):
    integ.ScalableTSDFVolume(0.02, 0.06, integ.TSDFVolumeColorType.Gray32)
  vol = integ.ScalableTSDFVolume(0.02, 0.06, integ.TSDFVolumeColorType.RGB8)
  gray = integ.RGBDImage.create_from_color_and_depth(integ.Image(c[0]), integ.Image(d[0]), depth_trunc=4.5)
  with pytest.raises(ValueError):
    vol.integrate(gray, intr, np.linalg.inv(P[0]))                 # intensity colour into an RGB8 volume
  with pytest.raises(ValueError):
    vol.integrate(_rgbd(c[0], d[0]), integ.PinholeCameraIntrinsic(320, 240, *K), np.linalg.inv(P[0]))
  with pytest.raises(ValueError):
    vol.integrate(_rgbd(c[0], d[0]), intr, np.eye(3))
  with pytest.raises(NotImplementedError):
    vol.extract_point_cloud()
  assert vol.n_units == 0
  from deepglobalregistration_b200 import _abi
  with pytest.raises(_abi.DgrError):
    _abi.tsdf_touch_ws(160, 120, 0, 0.02, 0.06)
