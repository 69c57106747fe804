"""oracle/rgbd_odometry.py on the CPU: the Jacobian rows against finite differences, the filters, pyramid and Sobel
images on hand-checkable inputs, the identical-frame and no-overlap cases, pose recovery on ray-cast frames, and the
open3d stand-in's argument checks (which need no device)."""
import numpy as np
import pytest

from deepglobalregistration_b200 import o3d_integration as integ
from deepglobalregistration_b200 import o3d_odometry as odo
from deepglobalregistration_b200 import synthetic as syn
from oracle import rgbd_odometry as ro


def _intensity(c):
  c = c.astype(np.float32)
  return ((c[..., 0] * np.float32(0.299) + c[..., 1] * np.float32(0.587) + c[..., 2] * np.float32(0.114))
          / np.float32(255.0)).astype(np.float32)


@pytest.mark.parametrize('hybrid', [True, False])
def test_jacobian_rows_match_finite_differences(hybrid):
  # linear target images in pixel coordinates: I = a0 + a u + b v, D = e0 + c u + d v; their Sobel * 0.125 is exact
  a, b, c, d = 0.013, -0.007, 0.002, 0.0035
  cam = (500.0, 480.0, 320.0, 240.0)
  fx, fy, cx, cy = cam
  rng = np.random.default_rng(0)
  for _ in range(20):
    p = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), rng.uniform(1.0, 3.0)])
    I_s = 0.3

    def residual(x):
      q = ro.move(ro.zyx(x), p[None])[0]
      u, v = fx * q[0] / q[2] + cx, fy * q[1] / q[2] + cy
      r_photo = (0.2 + a * u + b * v) - I_s
      r_geo = (1.5 + c * u + d * v) - q[2]
      if not hybrid:
        return np.array([r_photo])
      return np.array([np.sqrt(1 - ro.LAMBDA_HYBRID_DEPTH) * r_photo, np.sqrt(ro.LAMBDA_HYBRID_DEPTH) * r_geo])

    q = p[None]
    r, J = ro.jacobian_rows(q, [a / 0.125], [b / 0.125], [c / 0.125], [d / 0.125], [0.0], [0.0], [0.0], cam, hybrid)
    J = J[0]
    h = 1e-6
    fd = np.stack([(residual(h * e) - residual(-h * e)) / (2 * h) for e in np.eye(6)], 1)
    for k in range(J.shape[0]):
      assert np.linalg.norm(J[k] - fd[k]) <= 1e-6 * np.linalg.norm(fd[k]), (k, J[k], fd[k])


def test_gaussian_pyramid_sobel_by_hand():
  ramp = np.tile(np.arange(5, dtype=np.float32), (4, 1))      # I = u
  g = ro.gaussian3(ramp)
  np.testing.assert_array_equal(g[:, 1:4], ramp[:, 1:4])      # a linear ramp is kept inside
  np.testing.assert_array_equal(g[:, 0], np.float32(0.25))    # replicated border: 0.75 * 0 + 0.25 * 1
  np.testing.assert_array_equal(g[:, 4], np.float32(3.75))
  dx, dy = ro.sobel_dx(ramp) * 0.125, ro.sobel_dy(ramp) * 0.125
  np.testing.assert_array_equal(dx[:, 1:4], 1.0)              # slope 1: (-1, 0, 1) x (1, 2, 1) = 8, times 1/8
  np.testing.assert_array_equal(dx[:, 0], 0.5)                # border: (1 - 0) x (1 + 2 + 1) / 8
  np.testing.assert_array_equal(dy, 0.0)
  hole = np.ones((5, 5), np.float32)
  hole[2, 2] = np.nan
  gh = ro.gaussian3(hole)
  assert np.isnan(gh[1:4, 1:4]).all() and np.isfinite(gh[[0, 4], :]).all() and np.isfinite(gh[:, [0, 4]]).all()
  np.testing.assert_array_equal(gh[0], 1.0)
  pyr = ro.downsample(np.arange(20, dtype=np.float32).reshape(4, 5))
  np.testing.assert_array_equal(pyr, np.array([[3.0, 5.0], [13.0, 15.0]], np.float32))   # (0 + 1 + 5 + 6) / 4, ...
  d = ro.preprocess_depth(np.array([[0.0, 0.2, 1.0, 4.0, 4.5]], np.float32), 0.3, 4.0)
  np.testing.assert_array_equal(np.isnan(d), [[True, True, False, False, True]])


def _frames(n=50, w=160, h=120, seed=0):
  cols, deps, poses, intr = syn.rgbd_sequence(seed, n, width=w, height=h)
  return [(_intensity(cols[k]), deps[k].astype(np.float32) / np.float32(1000.0)) for k in range(n)], poses, intr


def test_identical_frames_and_no_overlap():
  frames, _, intr = _frames()
  Is, Ds = frames[10]
  ok, T, info, tr = ro.compute_rgbd_odometry(Is, Ds, Is, Ds, intr)
  assert ok
  np.testing.assert_array_equal(T, np.eye(4))
  assert not np.any(tr['steps'][0])                           # the first step is exactly zero
  assert info[5, 5] == len(tr['info_tgt']) > 1000
  It, Dt = frames[11]
  ok, T, info, _ = ro.compute_rgbd_odometry(Is, Ds, It, np.zeros_like(Dt), intr)
  assert not ok
  np.testing.assert_array_equal(T, np.eye(4))
  np.testing.assert_array_equal(info, np.eye(6))


def test_recovers_relative_pose():
  frames, poses, intr = _frames()
  (Is, Ds), (It, Dt) = frames[10], frames[11]
  ok, T, _, _ = ro.compute_rgbd_odometry(Is, Ds, It, Dt, intr)
  gt = np.linalg.inv(poses[11]) @ poses[10]
  E = np.linalg.inv(gt) @ T
  ang = np.degrees(np.arccos(np.clip((np.trace(E[:3, :3]) - 1) / 2, -1, 1)))
  # 160 x 120 frames 3.6 degrees and 3.8 cm apart; measured: 0.2 mm and 0.018 degrees
  assert ok and np.linalg.norm(E[:3, 3]) <= 2e-3 and ang <= 0.1


def test_stand_in_argument_checks():
  frames, _, intr = _frames(2, 32, 24)
  (Is, Ds), (It, Dt) = frames
  cam = integ.PinholeCameraIntrinsic(32, 24, *intr)
  src = integ.RGBDImage(integ.Image(Is), integ.Image(Ds))
  tgt = integ.RGBDImage(integ.Image(It), integ.Image(Dt))
  rgb = integ.RGBDImage(integ.Image(np.zeros((24, 32, 3), np.uint8)), integ.Image(Ds))
  bad_nan = integ.RGBDImage(integ.Image(np.full_like(Is, np.nan)), integ.Image(Ds))
  cases = [((rgb, tgt, cam), {}), ((src, tgt, integ.PinholeCameraIntrinsic(16, 24, *intr)), {}),
           ((bad_nan, tgt, cam), {}), ((src, tgt, cam), dict(odo_init=np.full((4, 4), np.inf))),
           ((src, tgt, cam), dict(option=odo.OdometryOption(max_depth_diff=0.0))),
           ((src, tgt, cam), dict(option=odo.OdometryOption(min_depth=2.0, max_depth=1.0))),
           ((src, tgt, cam), dict(option=odo.OdometryOption([1] * 7)))]
  for args, kw in cases:
    with pytest.raises(ValueError):
      odo.compute_rgbd_odometry(*args, **kw)
  with pytest.raises(TypeError):
    odo.compute_rgbd_odometry(src, tgt, cam, jacobian=object())
