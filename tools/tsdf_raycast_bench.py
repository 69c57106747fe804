"""Time the TSDF ray caster (dgr_tsdf_raycast, csrc/tsdf.cu) and frame-to-model tracking: CUDA-event medians of the
kernel and wall-clock medians of a whole ScalableTSDFVolume.raycast() call (host read included) at 640 x 480 on a
fused 50-frame synthetic volume (8 mm / 4 cm) at several poses; unit probes per ray counted by the fp64 oracle at
160 x 120; the per-frame split of a tracked frame (ray cast, odometry with its result read, integration with its
read); and one 50-frame fragment under ``integration --poses model`` against ``--poses odometry``.  Prints one JSON
line; numbers belong with the card's name and power limit, read in the same run.

    python tools/tsdf_raycast_bench.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepglobalregistration_b200 import _abi  # noqa: E402
from deepglobalregistration_b200 import integration  # noqa: E402
from deepglobalregistration_b200 import o3d_integration as integ  # noqa: E402
from deepglobalregistration_b200 import o3d_odometry as odo  # noqa: E402
from deepglobalregistration_b200 import synthetic as syn  # noqa: E402
from oracle import tsdf as ot  # noqa: E402
from oracle import tsdf_raycast as orc  # noqa: E402


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return out or torch.cuda.get_device_name(0)


def events(fn, reps):
  ts = []
  for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
  return float(np.median(ts))


def wall(fn, reps):
  ts = []
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    ts.append((time.perf_counter() - t0) * 1e3)
  return float(np.median(ts))


def _rgbd(c, d, trunc=4.5, intensity=False):
  return integ.RGBDImage.create_from_color_and_depth(c, d, depth_trunc=trunc, convert_rgb_to_intensity=intensity)


def raycast_times(reps):
  c, d, P, K = syn.rgbd_sequence(0, 50, 640, 480)
  intr = integ.PinholeCameraIntrinsic(640, 480, *K)
  vol = integ.ScalableTSDFVolume(0.008, 0.04, integ.TSDFVolumeColorType.RGB8)
  for k in range(50):
    vol.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(P[k]))
  between = P[24].copy()
  between[:3, 3] = 0.5 * (P[24][:3, 3] + P[25][:3, 3])
  out = {'units': vol.n_units}
  for name, pose in (('frame0', P[0]), ('frame25', P[25]), ('frame49', P[49]), ('between24_25', between)):
    ext = np.linalg.inv(pose)
    dep = torch.empty(480, 640, dtype=torch.float32, device=vol.device)
    inten = torch.empty_like(dep)
    col = torch.empty(480, 640, 3, dtype=torch.float32, device=vol.device)
    pose_h = np.linalg.inv(ext)

    def kernel(outs):
      _abi.tsdf_raycast(vol._keys, vol._vals, vol._tsdf, vol._weight, vol._rgb, 640, 480, intr._params(), pose_h,
                        vol.voxel_length, vol.sdf_trunc, 0.1, 3.0, 3.0, *outs)

    for _ in range(5):
      kernel((dep, inten, col))
      vol.raycast(intr, ext)
    hit = float((vol.raycast_tensors(intr, ext, outputs=('depth',))['depth'] > 0).float().mean())
    out[name] = {'kernel_depth_ms': round(events(lambda: kernel((dep,)), reps), 4),
                 'kernel_depth_intensity_colour_ms': round(events(lambda: kernel((dep, inten, col)), reps), 4),
                 'raycast_call_ms': round(wall(lambda: vol.raycast(intr, ext), reps), 4),
                 'hit_share': round(hit, 4)}
  return out


def oracle_probes(n_frames):
  c, d, P, K = syn.rgbd_sequence(0, n_frames, 160, 120)
  ov = ot.Volume(0.008, 0.04, color=True)
  for k in range(n_frames):
    ov.integrate(ot.depth_from_raw(d[k], 1000.0, 4.5), (160, 120) + tuple(K), np.linalg.inv(P[k]), c[k])
  out = {}
  for k in (0, n_frames // 2):
    tr = {}
    orc.raycast(ov, (160, 120) + tuple(K), np.linalg.inv(P[k]), trace=tr)
    steps = np.zeros(160 * 120, np.int64)
    kinds = np.zeros(3, np.int64)
    for ray, _, _, kind in tr['steps']:
      steps[ray] += 1
      kinds += np.bincount(kind, minlength=3)
    out[f'frame{k}'] = {'probes_per_ray_mean': round(float(tr['probes'].mean()), 2),
                        'probes_per_ray_max': int(tr['probes'].max()),
                        'steps_missing_unknown_known_per_ray': [round(float(x) / (160 * 120), 2) for x in kinds]}
  return out


def tracked_frame_split():
  c, d, P, K = syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05)
  intr = integ.PinholeCameraIntrinsic(640, 480, *K)
  opt = odo.OdometryOption(**integration.ODOMETRY_OPTION)
  its = opt.iteration_number_per_pyramid_level
  vol = integ.ScalableTSDFVolume(0.008, 0.04, integ.TSDFVolumeColorType.RGB8)
  dev = vol.device
  vol.integrate(_rgbd(c[0], d[0]), intr, np.eye(4))
  poses = [np.eye(4)]
  split = {'raycast_ms': [], 'odometry_and_read_ms': [], 'integrate_and_read_ms': []}
  for k in range(1, 50):
    src = _rgbd(c[k], d[k], opt.max_depth, True)
    Is, Ds = (torch.from_numpy(np.ascontiguousarray(np.asarray(a))).to(dev) for a in (src.color, src.depth))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model = vol.raycast_tensors(intr, np.linalg.inv(poses[-1]), opt.min_depth, opt.max_depth, float(min(k, 3)),
                                outputs=('depth', 'intensity'))
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    r = _abi.rgbd_odometry(Is, Ds, model['intensity'], model['depth'], intr._params(), np.eye(4), 'hybrid', its,
                           opt.max_depth_diff, opt.min_depth, opt.max_depth)
    ok, T, _ = odo.unpack_result(r.cpu().numpy())
    t2 = time.perf_counter()
    poses.append(poses[-1] @ T if ok else poses[-1])
    if ok:
      vol.integrate(_rgbd(c[k], d[k]), intr, np.linalg.inv(poses[-1]))
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    if k >= 5:
      split['raycast_ms'].append((t1 - t0) * 1e3)
      split['odometry_and_read_ms'].append((t2 - t1) * 1e3)
      split['integrate_and_read_ms'].append((t3 - t2) * 1e3)
  return {k: round(float(np.median(v)), 3) for k, v in split.items()}


def fragment_times():
  c, d, P, K = syn.rgbd_sequence(3, 50, turn=0.1, radius=0.05)
  cam = integ.PinholeCameraIntrinsic(640, 480, *K)
  out = {}
  with tempfile.TemporaryDirectory() as tmp:
    seq = syn.write_rgbd_sequence(tmp, 'room', c, d, P, K)
    frames = integration.sequence_frames(seq, need_poses=False)
    integration.model_poses(seq, frames, cam, 0, 5)                  # warm-up of every shape
    integration.odometry_poses(seq, frames, cam, 0, 5)
    for _ in range(2):                                               # the second pass is reported
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      _, vol, st = integration.model_poses(seq, frames, cam, 0, 50)
      vol.extract_triangle_mesh()
      torch.cuda.synchronize()
      t1 = time.perf_counter()
      P_odo, _ = integration.odometry_poses(seq, frames, cam, 0, 50)
      torch.cuda.synchronize()
      t2 = time.perf_counter()
      integration.integrate_fragment(seq, frames, cam, 0, 50, poses=P_odo)
      torch.cuda.synchronize()
      t3 = time.perf_counter()
    out = {'frames': 50, 'model_track_fuse_mesh_s': round(t1 - t0, 3), 'odometry_pairs_and_pose_graph_s':
           round(t2 - t1, 3), 'odometry_integration_and_mesh_s': round(t3 - t2, 3),
           'odometry_total_s': round(t3 - t1, 3), 'model_stats': st}
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=50)
  ap.add_argument('--oracle_frames', type=int, default=20)
  args = ap.parse_args()
  _abi.require_device('cuda')
  out = {'card': card(), 'raycast_640x480': raycast_times(args.reps),
         'oracle_160x120': oracle_probes(args.oracle_frames), 'tracked_frame_median': tracked_frame_split(),
         'fragment': fragment_times()}
  print(json.dumps(out))


if __name__ == '__main__':
  main()
