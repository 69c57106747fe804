"""open3d's legacy RGB-D odometry, backed by libdgr_b200 (csrc/odometry.cu): ``pipelines.odometry`` (``odometry``
before 0.12) OdometryOption, RGBDOdometryJacobianFromHybridTerm / FromColorTerm and compute_rgbd_odometry - what
open3d's reconstruction system (make_fragments) poses the frames of a raw RGB-D sequence with.

oracle/rgbd_odometry.py states every reading of open3d and every departure (notably: one correspondence per target
pixel, kept by a z-buffer; a Cholesky solve; no correspondence at odo_init is a failure).
"""
import numpy as np
import torch

from . import _abi


class OdometryOption:
  def __init__(self, iteration_number_per_pyramid_level=(20, 10, 5), max_depth_diff=0.03, min_depth=0.0,
               max_depth=4.0):
    self.iteration_number_per_pyramid_level = [int(v) for v in iteration_number_per_pyramid_level]
    self.max_depth_diff = float(max_depth_diff)
    self.min_depth = float(min_depth)
    self.max_depth = float(max_depth)

  def __repr__(self):
    return (f'OdometryOption class.\niteration_number_per_pyramid_level = {self.iteration_number_per_pyramid_level}\n'
            f'max_depth_diff = {self.max_depth_diff}\nmin_depth = {self.min_depth}\nmax_depth = {self.max_depth}')


class RGBDOdometryJacobian:
  _name = None


class RGBDOdometryJacobianFromHybridTerm(RGBDOdometryJacobian):
  """Park, Zhou & Koltun (ICCV 2017): a photometric row scaled by sqrt(1 - 0.968) and a geometric one by sqrt(0.968)."""
  _name = 'hybrid'


class RGBDOdometryJacobianFromColorTerm(RGBDOdometryJacobian):
  """Steinbruecker, Sturm & Cremers (ICCVW 2011): the photometric row alone."""
  _name = 'color'


def _check_option(option):
  its = option.iteration_number_per_pyramid_level
  if not 1 <= len(its) <= _abi.ODOMETRY_MAX_LEVELS:
    raise ValueError(f'iteration_number_per_pyramid_level must list 1 to {_abi.ODOMETRY_MAX_LEVELS} levels, got {its}')
  if any(not 0 <= v <= _abi.ODOMETRY_MAX_ITERATIONS for v in its):
    raise ValueError(f'iterations per level must lie in [0, {_abi.ODOMETRY_MAX_ITERATIONS}], got {its}')
  if not (0.0 <= option.min_depth < option.max_depth < np.inf):
    raise ValueError(f'need 0 <= min_depth < max_depth < inf, got {option.min_depth}, {option.max_depth}')
  if not 0.0 < option.max_depth_diff < np.inf:
    raise ValueError(f'max_depth_diff must be finite and positive, got {option.max_depth_diff}')


def _frame(rgbd, which, W, H):
  color, depth = np.asarray(rgbd.color), np.asarray(rgbd.depth)
  if color.ndim != 2 or color.dtype != np.float32:
    raise ValueError(f'{which}: colour must be float32 intensity (convert_rgb_to_intensity=True), got {color.dtype} '
                     f'{color.shape}')
  if depth.dtype != np.float32 or depth.shape != (H, W) or color.shape != (H, W):
    raise ValueError(f'{which}: intensity {color.shape} and float32 depth {depth.shape} must match the intrinsic\'s '
                     f'[{H}, {W}]')
  if not (np.isfinite(color).all() and np.isfinite(depth).all()):
    raise ValueError(f'{which}: intensity and depth must be finite')
  return color, depth


def odometry_arguments(rgbd_source, rgbd_target, pinhole_camera_intrinsic, odo_init, jacobian, option):
  """Every argument checked as the library checks it, before a device is needed -> (host images, intrinsic (4,),
  odo_init [4, 4], jacobian name, option)."""
  option = OdometryOption() if option is None else option
  jacobian = RGBDOdometryJacobianFromHybridTerm() if jacobian is None else jacobian
  if not isinstance(jacobian, RGBDOdometryJacobian) or jacobian._name is None:
    raise TypeError(f'expected RGBDOdometryJacobianFromHybridTerm or FromColorTerm, got {type(jacobian).__name__}')
  _check_option(option)
  W, H = pinhole_camera_intrinsic.width, pinhole_camera_intrinsic.height
  intr = pinhole_camera_intrinsic._params()
  if not (intr[0] > 0 and intr[1] > 0 and np.isfinite(intr).all()):
    raise ValueError('focal lengths must be finite and positive, the principal point finite')
  L = len(option.iteration_number_per_pyramid_level)
  if W < 1 or H < 1 or (W >> (L - 1)) < 1 or (H >> (L - 1)) < 1:
    raise ValueError(f'a {W} x {H} image has no pixel at pyramid level {L - 1}')
  imgs = _frame(rgbd_source, 'source', W, H) + _frame(rgbd_target, 'target', W, H)
  init = np.asarray(odo_init, dtype=np.float64)
  if init.shape != (4, 4) or not np.isfinite(init).all():
    raise ValueError(f'odo_init must be a finite 4x4 matrix, got shape {init.shape}')
  return imgs, intr, init, jacobian._name, option


def enqueue_rgbd_odometry(imgs, intr, init, jacobian, option, device, result=None):
  """Upload the four host images and enqueue one pair (no host read) -> the device result block."""
  Is, Ds, It, Dt = (torch.from_numpy(np.ascontiguousarray(a)).to(device) for a in imgs)
  return _abi.rgbd_odometry(Is, Ds, It, Dt, intr, init, jacobian, option.iteration_number_per_pyramid_level,
                            option.max_depth_diff, option.min_depth, option.max_depth, result=result)


def unpack_result(r):
  """Host result block -> (success, trans [4, 4], info [6, 6])."""
  r = np.asarray(r, dtype=np.float64)
  return bool(r[16] != 0.0), r[:16].reshape(4, 4).copy(), r[18:54].reshape(6, 6).copy()


def compute_rgbd_odometry(rgbd_source, rgbd_target, pinhole_camera_intrinsic=None, odo_init=np.eye(4), jacobian=None,
                          option=None):
  """open3d's ``compute_rgbd_odometry`` on the GPU: the pose mapping the source camera into the target camera, from
  RGBDImages made with convert_rgb_to_intensity=True.  -> (success, trans [4, 4], info [6, 6]); (False, I4, I6) when a
  solve fails or no pixel corresponds at odo_init.  One host read."""
  if pinhole_camera_intrinsic is None:
    raise ValueError('a PinholeCameraIntrinsic is required')
  args = odometry_arguments(rgbd_source, rgbd_target, pinhole_camera_intrinsic, odo_init, jacobian, option)
  dev = _abi.require_device('cuda')
  _abi.refresh_stream()
  return unpack_result(enqueue_rgbd_odometry(*args, dev).cpu().numpy())
