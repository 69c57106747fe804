"""RGB-D odometry on the GPU (csrc/odometry.cu through o3d_odometry) against oracle/rgbd_odometry.py: the images and
correspondence sets bit for bit, the per-step correspondence counts, the pose and the information matrix, determinism,
a dirty workspace, failures and argument checks, accuracy against the ray-cast ground truth, the integration CLI with
--poses odometry and the open3d stand-in."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import _abi
from deepglobalregistration_b200 import o3d_integration as integ
from deepglobalregistration_b200 import o3d_odometry as odo
from deepglobalregistration_b200 import synthetic as syn
from oracle import rgbd_odometry as ro

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _intensity(c):
  c = c.astype(np.float32)
  return ((c[..., 0] * np.float32(0.299) + c[..., 1] * np.float32(0.587) + c[..., 2] * np.float32(0.114))
          / np.float32(255.0)).astype(np.float32)


@pytest.fixture(scope='module')
def small():
  cols, deps, poses, intr = syn.rgbd_sequence(0, 50, width=160, height=120)
  frames = [(_intensity(cols[k]), deps[k].astype(np.float32) / np.float32(1000.0)) for k in range(50)]
  return frames, poses, intr


def _run(Is, Ds, It, Dt, intr, init=np.eye(4), jac='hybrid', its=(20, 10, 5), ws=None, **kw):
  t = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (Is, Ds, It, Dt)]
  r = _abi.rgbd_odometry(*t, intr, init, jac, its, ws=ws, **kw)
  return r.cpu().numpy()


def _ws(W, H, L):
  n = C.c_int64(0)
  _abi.call('dgr_rgbd_odometry_ws_elems', W, H, L, C.byref(n))
  return torch.empty(n.value, dtype=torch.int64, device=DEV)


def _bits(a):
  """float32 bits with every NaN made the same NaN (a NaN's payload carries no value)"""
  a = np.array(a, np.float32)
  a[np.isnan(a)] = np.nan
  return torch.from_numpy(a).view(torch.int32)


def _images(ws, W, H, L):
  """float images of the workspace as host arrays: per level 8, then the filtered intensities; the z-buffer."""
  off = _abi.rgbd_odometry_ws_layout(W, H, L)
  flat = ws.view(torch.float32)
  out = []
  for l in range(L):
    w, h = W >> l, H >> l
    out.append([flat[2 * off[8 * l + k]: 2 * off[8 * l + k] + w * h].reshape(h, w).cpu().numpy() for k in range(8)])
  Gs = flat[2 * off[8 * L]: 2 * off[8 * L] + W * H].reshape(H, W).cpu().numpy()
  Gt = flat[2 * off[8 * L + 1]: 2 * off[8 * L + 1] + W * H].reshape(H, W).cpu().numpy()
  z = ws[off[8 * L + 2]: off[8 * L + 2] + W * H].cpu().numpy().view(np.uint64)
  return out, Gs, Gt, z


def test_stage_images_bit_exact(small):
  frames, _, intr = small
  (Is, Ds), (It, Dt) = frames[10], frames[11]
  H, W = Ds.shape
  L = 3
  ws = _ws(W, H, L)
  _run(Is, Ds, It, Dt, intr, its=(0, 0, 0), ws=ws, min_depth=1.0, max_depth=2.0)     # holes where out of range
  lv, Gs, Gt, _ = _images(ws, W, H, L)
  prep = ro.prepare(Is, Ds, It, Dt, intr, np.eye(4), L, 0.03, 1.0, 2.0)
  assert torch.equal(_bits(Gs), _bits(prep['Gs'])) and torch.equal(_bits(Gt), _bits(prep['Gt']))
  names = ('Is', 'Ds', 'It', 'Dt', 'dIx', 'dIy', 'dDx', 'dDy')
  for l in range(L):
    for k, name in enumerate(names):
      assert torch.equal(_bits(lv[l][k]), _bits(prep['levels'][l][name])), (l, name)
  assert np.isnan(prep['levels'][0]['Ds']).any()        # the depth holes went through the filters


def test_correspondence_set_at_pose(small):
  frames, poses, intr = small
  (Is, Ds), (It, Dt) = frames[10], frames[13]
  H, W = Ds.shape
  T = np.linalg.inv(poses[13]) @ poses[10]
  ws = _ws(W, H, 1)
  r = _run(Is, Ds, It, Dt, intr, init=T, its=(0,), ws=ws)
  _, _, _, z = _images(ws, W, H, 1)
  tgt = np.flatnonzero(z != np.uint64(2 ** 64 - 1))
  src = (z[tgt] & np.uint64(0xFFFFFFFF)).astype(np.int64)
  prep = ro.prepare(Is, Ds, It, Dt, intr, T, 1, 0.03, 0.0, 4.0)
  s_o, t_o = ro.correspondences(prep['Ds0'], prep['Dt0'], ro.level_camera(intr, 0), T, 0.03)
  assert len(t_o) > 1000
  np.testing.assert_array_equal(tgt, t_o)
  np.testing.assert_array_equal(src, s_o)
  assert r[16] == 1.0 and r[54] == len(t_o)


@pytest.mark.parametrize('jac', ['hybrid', 'color'])
@pytest.mark.parametrize('its', [(6,), (5, 4), (4, 3, 3, 2)])
def test_against_oracle(small, jac, its):
  frames, _, intr = small
  (Is, Ds), (It, Dt) = frames[10], frames[11]
  r = _run(Is, Ds, It, Dt, intr, jac=jac, its=its)
  ok, T, info, tr = ro.compute_rgbd_odometry(Is, Ds, It, Dt, intr, hybrid=jac == 'hybrid', iterations=its)
  n = len(tr['counts'])
  assert bool(r[16]) == ok and int(r[17]) == n
  np.testing.assert_array_equal(r[55:55 + n], tr['counts'])
  assert np.abs(r[:16].reshape(4, 4) - T).max() <= 1e-7
  info_d = r[18:54].reshape(6, 6)
  assert np.abs(info_d - info).max() <= 1e-9 * np.abs(info).max()


def test_identical_frames_and_determinism(small):
  frames, _, intr = small
  Is, Ds = frames[20]
  r = _run(Is, Ds, Is, Ds, intr)
  assert r[16] == 1.0
  np.testing.assert_array_equal(r[:16].reshape(4, 4), np.eye(4))
  (It, Dt) = frames[21]
  a, b = _run(Is, Ds, It, Dt, intr), _run(Is, Ds, It, Dt, intr)
  assert a.tobytes() == b.tobytes()


def test_dirty_workspace(small):
  frames, _, intr = small
  (Is, Ds), (It, Dt) = frames[30], frames[31]
  H, W = Ds.shape
  clean = _run(Is, Ds, It, Dt, intr)
  for fill in (float('nan'), -1.0e30):
    ws = _ws(W, H, 3)
    ws.view(torch.float64).fill_(fill)
    assert _run(Is, Ds, It, Dt, intr, ws=ws).tobytes() == clean.tobytes()
  ws = _ws(W, H, 3)
  ws.copy_(torch.randint(-2 ** 62, 2 ** 62, ws.shape, device=DEV))
  assert _run(Is, Ds, It, Dt, intr, ws=ws).tobytes() == clean.tobytes()


def test_failures_and_argument_checks(small):
  frames, _, intr = small
  (Is, Ds), (It, Dt) = frames[0], frames[1]
  r = _run(Is, Ds, It, np.zeros_like(Dt), intr)              # no target depth: nothing corresponds
  assert r[16] == 0.0
  np.testing.assert_array_equal(r[:16].reshape(4, 4), np.eye(4))
  np.testing.assert_array_equal(r[18:54].reshape(6, 6), np.eye(6))
  far = np.eye(4)
  far[0, 3] = 50.0                                            # the source moved out of the target's view
  assert _run(Is, Ds, It, Dt, intr, init=far)[16] == 0.0
  torch.cuda.synchronize()
  before = _abi.lib().dgr_launch_count()
  bad = [dict(its=()), dict(its=(101,)), dict(its=(1,) * 7), dict(min_depth=2.0, max_depth=1.0),
         dict(max_depth_diff=0.0), dict(init=np.full((4, 4), np.nan)), dict(intr=(0.0, 1.0, 1.0, 1.0))]
  for kw in bad:
    intr_k = kw.pop('intr', intr)
    with pytest.raises(_abi.DgrError):
      _run(Is, Ds, It, Dt, intr_k, **kw)
  with pytest.raises(_abi.DgrError):
    _abi.rgbd_odometry(*(torch.zeros(4, 4, device=DEV) for _ in range(4)), intr, np.eye(4), 'hybrid', (1,) * 4)
  assert _abi.lib().dgr_launch_count() == before


def _rel_errors(T, gt):
  E = np.linalg.inv(gt) @ T
  return float(np.linalg.norm(E[:3, 3])), float(np.degrees(np.arccos(np.clip((np.trace(E[:3, :3]) - 1) / 2, -1, 1))))


def test_accuracy_full_size():
  # 640 x 480, 0.72 degrees and 6 mm per frame.  Consecutive pairs start from the identity; pairs 5 frames apart from
  # the chain of consecutive results, as integration --poses odometry starts its loop closures (from the identity
  # one of five such pairs diverged: 7.5 cm, 8.7 degrees).  Measured on an H100: consecutive worst 0.54 mm / 0.052 deg,
  # 5 apart 0.22 mm / 0.012 deg.
  cols, deps, poses, intr = syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05)
  cam = integ.PinholeCameraIntrinsic(640, 480, *intr)
  rgbd = {}

  def frame(k):
    if k not in rgbd:
      rgbd[k] = integ.RGBDImage.create_from_color_and_depth(cols[k], deps[k], depth_trunc=4.0)
    return rgbd[k]

  step = {}
  for s in range(0, 45):
    ok, T, _ = odo.compute_rgbd_odometry(frame(s), frame(s + 1), cam)
    assert ok
    step[s] = T
  out = {}
  for gap in (1, 5):
    te, re = [], []
    for s in range(0, 40, 8):
      t = s + gap
      init = np.eye(4)
      for k in range(s, t):
        init = step[k] @ init
      T = step[s] if gap == 1 else odo.compute_rgbd_odometry(frame(s), frame(t), cam, init)[1]
      e = _rel_errors(T, np.linalg.inv(poses[t]) @ poses[s])
      te.append(e[0])
      re.append(e[1])
    out[gap] = (max(te), max(re))
  print('rgbd odometry 640x480 worst (m, deg): consecutive', out[1], '5 apart', out[5])
  assert out[1][0] <= 2e-3 and out[1][1] <= 0.2
  assert out[5][0] <= 2e-3 and out[5][1] <= 0.1


def test_open3d_stand_in(small):
  from deepglobalregistration_b200 import shims
  o3d = shims._open3d_stub()
  frames, _, intr = small
  (Is, Ds), (It, Dt) = frames[10], frames[11]
  src = integ.RGBDImage(integ.Image(Is), integ.Image(Ds))
  tgt = integ.RGBDImage(integ.Image(It), integ.Image(Dt))
  cam = o3d.camera.PinholeCameraIntrinsic(160, 120, *intr)
  ok, T, info = o3d.pipelines.odometry.compute_rgbd_odometry(
      src, tgt, cam, np.eye(4), o3d.pipelines.odometry.RGBDOdometryJacobianFromHybridTerm(),
      o3d.pipelines.odometry.OdometryOption())
  r = _run(Is, Ds, It, Dt, intr)
  assert ok and np.array_equal(T, r[:16].reshape(4, 4)) and np.array_equal(info, r[18:54].reshape(6, 6))
  assert o3d.odometry.compute_rgbd_odometry is odo.compute_rgbd_odometry
  with pytest.raises(ValueError):
    odo.compute_rgbd_odometry(integ.RGBDImage(integ.Image(np.zeros((120, 160, 3), np.uint8)), integ.Image(Ds)),
                              tgt, cam)


def test_integration_cli_odometry(tmp_path):
  from deepglobalregistration_b200 import integration
  cols, deps, poses, intr = syn.rgbd_sequence(5, 12, turn=0.02, radius=0.02)    # 0.65 degrees, 1 cm per frame
  seq = syn.write_rgbd_sequence(str(tmp_path / 'raw'), 'room', cols, deps, poses, intr)
  out = tmp_path / 'out'
  import contextlib
  import io as pyio
  buf = pyio.StringIO()
  with contextlib.redirect_stdout(buf):
    assert integration.main([str(tmp_path / 'raw' / 'room'), str(out), '--frames_per_fragment', '12',
                             '--poses', 'odometry']) == 0
  summary = json.loads(buf.getvalue().strip().splitlines()[-1])
  print('integration --poses odometry:', summary)
  assert summary['fragments'] == 1 and summary['odometry_pairs'] == 11 + 3   # consecutive, and keyframes (0, 5), (0, 10), (5, 10)
  ate = summary['fragment_ate'][0]
  assert ate <= 2e-3                                           # measured on an H100: 0.32 mm
  log = out / 'room' / 'seq-01' / 'fragment-0.log'
  from deepglobalregistration_b200 import io as dio
  traj = dio.read_trajectory(str(log))
  assert len(traj) == 12
  for f in os.listdir(seq):
    if f.endswith('.pose.txt'):
      os.remove(os.path.join(seq, f))
  buf = pyio.StringIO()
  with contextlib.redirect_stdout(buf):
    assert integration.main([str(tmp_path / 'raw' / 'room'), str(tmp_path / 'out2'), '--frames_per_fragment', '12',
                             '--poses', 'odometry']) == 0
  s2 = json.loads(buf.getvalue().strip().splitlines()[-1])
  assert 'fragment_ate' not in s2 and s2['vertices'] > 1000
  v = np.asarray(dio.read_point_cloud(str(tmp_path / 'out2' / 'room' / 'seq-01' / 'fragment-0.ply')).points)
  vw = v @ poses[0][:3, :3].T + poses[0][:3, 3]                # first camera -> world
  face, _ = syn.box_face_distance(vw, syn.room_boxes(5, (3.6, 3.0, 2.5)))
  print('odometry fragment: median / 95% vertex-face distance', np.median(face), np.quantile(face, 0.95))
  assert np.median(face) <= 1e-3 and np.quantile(face, 0.95) <= 3e-3    # measured: 0.10 mm, 0.35 mm
